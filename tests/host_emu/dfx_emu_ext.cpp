// dfx_emu_ext.cpp -- HOST EMULATION of the external-wrench kernels (include/dfx.h DfxExternalWrench: the _ex entries), for
// CPU-side unit tests only.  The whole host emulation (dfx_emu.cpp) plus two entries, built into a library of its own
// (tests/wrench_util.py): the library the other tests load keeps its code -- with the wrench instantiations in the same
// translation unit the compiler inlines, and in the builds with FMA contraction contracts, differently.
#include "dfx_emu.cpp"

extern "C" {

// f_ext [n, L, 6] (torque, force at the centre of mass, world axes), held over the substeps
int emu_step_forward_ext(const EmuPack* p, int n, int substeps, int mm_freq, double dt,
                         const float* q, const float* qd, const float* act, const float* musc,
                         float* q_out, float* qd_out, float* tape, const DfxDerived* derived, const float* f_ext) {
    StepArgs a;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.q = q; a.qd = qd; a.act = act; a.musc = musc; a.q_out = q_out; a.qd_out = qd_out; a.tape = tape;
    if (derived) { a.derived = *derived; a.has_derived = 1; }
    a.tape_bf16 = g_tape_bf16;
    a.hinv_base = tape_geom(p->pack.L, p->pack.Q, p->pack.D, n, substeps, mm_freq).hinv_base;
    // (filled with NaN, as emu_step_forward: a field read before it is written shows up)
    std::vector<float> scratch((size_t)(wrench_scratch_end(p->host.layout, p->pack.L, false) + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    const DfxExternalWrench w{f_ext, nullptr};
    for (int env = 0; env < n; ++env) env_step_forward<true>(p->pack, p->host.layout, SP{scratch.data()}, g, env, a, w);
    return 0;
}

// the same f_ext as the forward call; its cotangent -> g_f_ext [n, L, 6] (NULL: skip)
int emu_step_backward_ext(const EmuPack* p, int n, int substeps, int mm_freq, double dt,
                          const float* act, const float* musc, const float* tape,
                          const float* gq_out, const float* gqd_out,
                          float* gq, float* gqd, float* gact, float* gmusc, const float* f_ext, float* g_f_ext) {
    StepArgs a;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.act = act; a.musc = musc; a.tape_in = tape; a.gq_out = gq_out; a.gqd_out = gqd_out;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc;
    a.tape_bf16 = g_tape_bf16;
    a.hinv_base = tape_geom(p->pack.L, p->pack.Q, p->pack.D, n, substeps, mm_freq).hinv_base;
    std::vector<float> scratch((size_t)(wrench_scratch_end(p->host.layout_bwd, p->pack.L, true) + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    const DfxExternalWrench w{f_ext, g_f_ext};
    for (int env = 0; env < n; ++env) env_step_backward<true>(p->pack, p->host.layout_bwd, SP{scratch.data()}, g, env, a, w);
    return 0;
}

}  // extern "C"
