// dfx_emu_link.cpp -- HOST EMULATION of the link-state kernels (include/dfx.h dfx_link_state_forward / _backward), for CPU-side
// unit tests only.  The whole host emulation (dfx_emu.cpp, unchanged) plus two entries, built into a library of its own
// (tests/link_util.py), so the library the other tests load keeps its code.  The step entries of this same library give the
// derived dumps the link state is compared with bit for bit.
#include "dfx_emu.cpp"

extern "C" {

// q [n*Q], qd [n*D] -> body_X_sc, body_X_sm [n*L*7], body_v_s [n*L*6] (any NULL: skip)
int emu_link_state_forward(const EmuPack* p, int n, const float* q, const float* qd, float* X_sc, float* X_sm, float* v_s) {
    LinkStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.X_sc = X_sc; a.X_sm = X_sm; a.v_s = v_s;
    // (filled with NaN, as emu_step_forward: a field read before it is written shows up)
    std::vector<float> scratch((size_t)(p->host.layout.fwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) link_state_forward(p->pack, p->host.layout, SP{scratch.data()}, g, env, a);
    return 0;
}

// cotangents of the three outputs (NULL == 0) -> gq [n*Q], gqd [n*D] (NULL: skip)
int emu_link_state_backward(const EmuPack* p, int n, const float* q, const float* qd, const float* g_X_sc, const float* g_X_sm,
                            const float* g_v_s, float* gq, float* gqd) {
    LinkStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.g_X_sc = g_X_sc; a.g_X_sm = g_X_sm; a.g_v_s = g_v_s; a.gq = gq; a.gqd = gqd;
    std::vector<float> scratch((size_t)(p->host.layout_bwd.bwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) link_state_backward(p->pack, p->host.layout_bwd, SP{scratch.data()}, g, env, a);
    return 0;
}

}  // extern "C"
