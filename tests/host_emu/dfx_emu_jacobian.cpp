// dfx_emu_jacobian.cpp -- HOST EMULATION of the Jacobian-state kernels (include/dfx.h dfx_jacobian_state_forward / _backward), for
// CPU-side unit tests only.  The link-state emulation (dfx_emu_link.cpp, unchanged, with the whole host emulation) plus two entries,
// built into a library of its own (tests/jacobian_util.py).  The step entries of this same library give the derived dumps the
// Jacobian state is compared with bit for bit.
#include "dfx_emu_link.cpp"

extern "C" {

// q [n*Q], qd [n*D] -> J [n*L*6*D], body_a_s [n*L*6] (any NULL: skip)
int emu_jacobian_state_forward(const EmuPack* p, int n, const float* q, const float* qd, float* J, float* a_s) {
    JacobianStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.J = J; a.a_s = a_s;
    // (filled with NaN, as emu_step_forward: a field read before it is written shows up)
    std::vector<float> scratch((size_t)(p->host.layout.fwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) jacobian_state_forward(p->pack, p->host.layout, SP{scratch.data()}, g, env, a);
    return 0;
}

// cotangents g_J, g_a_s (NULL == 0) -> gq [n*Q], gqd [n*D] (NULL: skip)
int emu_jacobian_state_backward(const EmuPack* p, int n, const float* q, const float* qd, const float* g_J, const float* g_a_s,
                                float* gq, float* gqd) {
    JacobianStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.g_J = g_J; a.g_a_s = g_a_s; a.gq = gq; a.gqd = gqd;
    std::vector<float> scratch((size_t)(p->host.layout_bwd.bwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) jacobian_state_backward(p->pack, p->host.layout_bwd, SP{scratch.data()}, g, env, a);
    return 0;
}

}  // extern "C"
