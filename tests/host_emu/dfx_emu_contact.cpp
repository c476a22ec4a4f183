// dfx_emu_contact.cpp -- HOST EMULATION of the contact-state kernels (include/dfx.h dfx_contact_state_forward / _backward), for
// CPU-side unit tests only.  The host emulation with the external-wrench entries (dfx_emu_ext.cpp, unchanged) plus two entries,
// built into a library of its own (tests/contact_util.py), so the libraries the other tests load keep their code.  The _ext step
// entries of this same library run the convention check: an env-step with the ground off under f_ext = body_f_contact against
// the same env-step with the ground on.
#include "dfx_emu_ext.cpp"

extern "C" {

// q [n*Q], qd [n*D] -> contact_f [n*C*3], contact_height [n*C], body_f_contact [n*L*6] (any NULL: skip)
int emu_contact_state_forward(const EmuPack* p, int n, const float* q, const float* qd, float* contact_f, float* contact_height,
                              float* body_f_contact) {
    ContactStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.corder = p->host.corder.data();
    a.contact_f = contact_f; a.contact_height = contact_height; a.body_f = body_f_contact;
    // (filled with NaN, as emu_step_forward: a field read before it is written shows up)
    std::vector<float> scratch((size_t)(p->host.layout.fwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) contact_state_forward(p->pack, p->host.layout, SP{scratch.data()}, g, env, a);
    return 0;
}

// cotangents of the three outputs (NULL == 0) -> gq [n*Q], gqd [n*D] (NULL: skip)
int emu_contact_state_backward(const EmuPack* p, int n, const float* q, const float* qd, const float* g_contact_f,
                               const float* g_contact_height, const float* g_body_f_contact, float* gq, float* gqd) {
    ContactStateArgs a;
    memset(&a, 0, sizeof a);
    a.q = q; a.qd = qd; a.corder = p->host.corder.data();
    a.g_contact_f = g_contact_f; a.g_contact_height = g_contact_height; a.g_body_f = g_body_f_contact; a.gq = gq; a.gqd = gqd;
    std::vector<float> scratch((size_t)(p->host.layout_bwd.bwd_size + 16) * DFX_ES, nanf(""));
    GroupSerial g{0};
    for (int env = 0; env < n; ++env) contact_state_backward(p->pack, p->host.layout_bwd, SP{scratch.data()}, g, env, a);
    return 0;
}

}  // extern "C"
