// dfx_emu_dynamics.cpp -- HOST EMULATION of the dynamics-state kernels (include/dfx.h dfx_dynamics_state_forward / _backward), for
// CPU-side unit tests only.  The host emulation with the external-wrench entries (dfx_emu_ext.cpp, unchanged) plus two entries,
// built into a library of its own (tests/dynamics_util.py), so the libraries the other tests load keep their code.  The backward
// goes through a one-substep tape of its own, as the kernels' workspace: the tile kernel's forward (env_step_forward<true, true>,
// a NULL wrench reading as zero; substeps = mm_freq = 1, fp32 rows), then the seeded adjoint.  The _ext step entries of this same library give the derived dumps
// and the step adjoint of the convention check.
#include "dfx_emu_ext.cpp"

extern "C" {

// (q, qd, act, musc, f_ext (NULL: zero)) -> joint_qdd [n*D], joint_tau [n*D], H [n*D*D] (any NULL: skip)
int emu_dynamics_state_forward(const EmuPack* p, int n, const float* q, const float* qd, const float* act, const float* musc,
                               const float* f_ext, float* joint_qdd, float* joint_tau, float* H) {
    DynamicsStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.act = act; a.musc = musc; a.f_ext = f_ext;
    a.joint_qdd = joint_qdd; a.joint_tau = joint_tau; a.H = H;
    // (filled with NaN, as emu_step_forward: a field read before it is written shows up)
    std::vector<float> scratch((size_t)(wrench_scratch_end(p->host.layout, p->pack.L, false) + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) dynamics_state_forward(p->pack, p->host.layout, SP{scratch.data()}, g, env, a);
    return 0;
}

// cotangents (NULL == 0) -> gq [n*Q], gqd [n*D], gact [n*D], gmusc [n*M], g_f_ext [n*L*6] (NULL: skip)
int emu_dynamics_state_backward(const EmuPack* p, int n, const float* q, const float* qd, const float* act, const float* musc,
                                const float* f_ext, const float* g_qdd, const float* g_tau, const float* g_H,
                                float* gq, float* gqd, float* gact, float* gmusc, float* g_f_ext) {
    const TapeGeom t = tape_geom(p->pack.L, p->pack.Q, p->pack.D, n, 1, 1);
    std::vector<float> tape((size_t)t.total), q_end((size_t)n * p->pack.Q + 1), qd_end((size_t)n * p->pack.D + 1);
    StepArgs ta;
    memset(&ta, 0, sizeof ta);
    ta.N = n; ta.substeps = 1; ta.mm_freq = 1; ta.dt_sub = 0.0f;
    ta.q = q; ta.qd = qd; ta.act = act; ta.musc = musc; ta.q_out = q_end.data(); ta.qd_out = qd_end.data();
    ta.tape = tape.data(); ta.tape_in = tape.data(); ta.hinv_base = t.hinv_base;
    {
        std::vector<float> scratch((size_t)(wrench_scratch_end(p->host.layout, p->pack.L, false) + 16) * DFX_ES, nanf(""));
        GroupSerial g{0};
        const DfxExternalWrench w{f_ext, nullptr};      // (NULL reads as zero, as in dfx_tile_dynamics_backward_kernel)
        for (int env = 0; env < n; ++env) env_step_forward<true, true>(p->pack, p->host.layout, SP{scratch.data()}, g, env, ta, w);
    }
    DynamicsStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.act = act; a.musc = musc; a.f_ext = f_ext;
    a.g_qdd = g_qdd; a.g_tau = g_tau; a.g_H = g_H;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc; a.g_f_ext = g_f_ext;
    std::vector<float> scratch((size_t)(wrench_scratch_end(p->host.layout_bwd, p->pack.L, true) + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) dynamics_state_backward(p->pack, p->host.layout_bwd, SP{scratch.data()}, g, env, ta, a);
    return 0;
}

}  // extern "C"
