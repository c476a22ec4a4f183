// dfx_step.h -- one environment's whole env-step (all substeps) forward and backward, for a
// group policy owning the environment's scratch.  Shared verbatim by the tile kernels (dfx_tile.cu), the
// lane-group kernels (dfx_kernels.cu) and the host emulation used by CPU-side unit tests.
//
// Tape (written by forward when taping, read by backward), all fp32, one block per substep / per update:
//   rows   per substep: the (q, qd) ENTERING it and the forward intermediates the adjoint
//          needs -- X_sc, X_sm, S, v, a, total link wrenches, q'' (32 L + 8 D + Q floats, padded to 4)
//   H^-1   D * D floats per mass-matrix update
// laid out [block][env][n] (lane-group kernels, host) or [block][tile of 32 envs][n][32] (tile kernels): the
// group policy's block_in / row_in / block_out hide the difference.
// The path is issue / latency bound with HBM idle, so the adjoint trades bandwidth for instructions: it reads these
// rows back (coalesced, tile-contiguous per substep) instead of re-running the forward dynamics.  Ant: 1.7 KB
// per env-substep vs the reference's ~3.7 KB (it keeps every State tensor alive, SURVEY.md section 5).
#pragma once

#include "../../include/dfx.h"
#include "dfx_pack_build.h"
#include "dfx_phases.h"

namespace dfx {

struct StepArgs {
    int N, substeps, mm_freq;
    float dt_sub;
    const float* q; const float* qd; const float* act; const float* musc;
    float* q_out; float* qd_out;
    float* tape;
    DfxDerived derived; int has_derived;
    // backward
    const float* tape_in;
    const float* gq_out; const float* gqd_out;
    float* gq; float* gqd; float* gact; float* gmusc;
    long long hinv_base;
    int flags;   // bit 1: CTA-wide phase barriers
    int tape_bf16;   // the middle of every tape row (the forward intermediates) is stored as bf16 (tile kernels)
    // action map folded into the step (include/dfx.h dfx_step_*_mapped): raw != nullptr
    const float* raw; const float* strength; float* used; const float* g_used; float* g_raw;
    int map_num_act, map_offset, map_muscle;
    float map_pre_scale, map_pre_bias, map_drive_scale;
    // env transition folded into the step launch (include/dfx.h dfx_env_step_*; tile kernels only): env_kind != 0.  Forward:
    // `env` is read after the step (epilogue); backward: `env_adj` before it (prologue), writing gq_out / gqd_out / g_used.
    int env_kind;
    DfxEnvTransition env;
    DfxEnvTransitionAdj env_adj;
};

// derived State fields of the last substep (reference model.py:375-388); `late` = the ones that exist only after the solve
template <class Grp>
DFX_HD void dump_derived(const Pack& P, const Layout& Y, SP s, const DfxDerived& d, int env, bool late, const Grp& g) {
    const int L = P.L, D = P.D;
    if (late) {
        if (d.joint_qdd) DFX_FOR(i, D) d.joint_qdd[(long long)env * D + i] = s[Y.qdd + i];
        return;
    }
    if (d.body_X_sc) DFX_FOR(i, L * 7) d.body_X_sc[(long long)env * L * 7 + i] = s[Y.Xsc + i];
    if (d.body_X_sm) DFX_FOR(i, L * 7) d.body_X_sm[(long long)env * L * 7 + i] = s[Y.Xsm + i];
    if (d.joint_S_s) DFX_FOR(i, D * 6) d.joint_S_s[(long long)env * D * 6 + i] = s[Y.S + i];
    if (d.body_v_s) DFX_FOR(i, L * 6) d.body_v_s[(long long)env * L * 6 + i] = s[Y.v + i];
    if (d.body_a_s) DFX_FOR(i, L * 6) d.body_a_s[(long long)env * L * 6 + i] = s[Y.a + i];
    if (d.body_f_s) DFX_FOR(i, L * 6) d.body_f_s[(long long)env * L * 6 + i] = s[Y.f + i];
    if (d.body_ft_s) DFX_FOR(i, L * 6) d.body_ft_s[(long long)env * L * 6 + i] = s[Y.ft + i] - s[Y.f + i];
    if (d.joint_tau) DFX_FOR(i, D) d.joint_tau[(long long)env * D + i] = s[Y.tau + i];
}

// actuation of one environment: from the caller's arrays, or formed from the raw policy output (same arithmetic as
// dfx_action_map_forward: used = clip(raw, -1, 1) * pre_scale + pre_bias ; drive = (used * drive_scale) * strength)
template <class Grp>
DFX_HD void load_actuation(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const StepArgs& a, bool write_used) {
    const int D = P.D, M = P.M;
    if (!a.raw) {
        DFX_FOR(i, D) s[Y.act + i] = a.act[(long long)env * D + i];
        DFX_FOR(i, M) s[Y.musc + i] = a.musc[(long long)env * M + i];
        return;
    }
    const int A = a.map_num_act, off = a.map_offset;
    const float* re = a.raw + (long long)env * A;
    const int width = a.map_muscle ? M : D;
    const int dst = a.map_muscle ? Y.musc : Y.act;
    DFX_FOR(i, width) {
        const int j = i - off;
        float out = 0.0f;
        if (j >= 0 && j < A) {
            const float u = fminf(fmaxf(re[j], -1.0f), 1.0f) * a.map_pre_scale + a.map_pre_bias;
            out = (u * a.map_drive_scale) * a.strength[j];
        }
        s[dst + i] = out;
    }
    if (a.map_muscle) { DFX_FOR(i, D) s[Y.act + i] = a.act ? a.act[(long long)env * D + i] : 0.0f; }
    else { DFX_FOR(i, M) s[Y.musc + i] = a.musc ? a.musc[(long long)env * M + i] : 0.0f; }
    if (write_used && a.used) DFX_FOR(j, A) a.used[(long long)env * A + j] = fminf(fmaxf(re[j], -1.0f), 1.0f) * a.map_pre_scale + a.map_pre_bias;
}

// External wrench (include/dfx.h DfxExternalWrench, the _ex entries): kWrench instantiations read w.f_ext [N, L, 6] once per
// env-step into the scratch past the layout's end (dfx_pack.h wrench_offset) and hold it over the substeps, as the actuation; the
// adjoint writes its cotangent to w.g_f_ext (when not NULL) at the end, as gact.  The pointers travel next to StepArgs, at the
// end of the kernel argument block, so the parameter offsets of the kernels without a wrench stay as they are.
template <class Grp>
DFX_HD void load_wrench(const Pack& P, SP s, const Grp& g, int env, const DfxExternalWrench& w, int xw) {
    DFX_FOR(i, P.L * 6) s[xw + i] = w.f_ext[(long long)env * P.L * 6 + i];
}

// kNullWrench (the dynamics state's one-substep forward, dfx_tile_dynamics_backward_kernel): a NULL w.f_ext reads as zero, so one
// instantiation serves with and without a wrench; off for the step kernels, which keep their code.
template <bool kWrench = false, bool kNullWrench = false, class Grp>
DFX_HD void env_step_forward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const StepArgs& a,
                             const DfxExternalWrench& w = DfxExternalWrench{nullptr, nullptr}) {
    const int Q = P.Q, D = P.D, DD = D * D;
    const RowFmt rf = row_fmt(P, Y, a.tape_bf16 != 0);
    const int xw = kWrench ? wrench_offset(Y, false) : -1;
    DFX_FOR(i, Q) s[Y.q + i] = a.q[(long long)env * Q + i];
    DFX_FOR(i, D) s[Y.qd + i] = a.qd[(long long)env * D + i];
    load_actuation(P, Y, s, g, env, a, true);
    if constexpr (kWrench && kNullWrench) {
        DFX_FOR(i, P.L * 6) s[xw + i] = w.f_ext ? w.f_ext[(long long)env * P.L * 6 + i] : 0.0f;
    } else if constexpr (kWrench) {
        load_wrench(P, s, g, env, w, xw);
    }
    for (int i = Y.qdd + D + g.lane; i < Y.q + Y.tape_row; i += Grp::G) s[i] = 0.0f;   // row padding
    if (g.lane == 0) s[Y.cmask] = 0.0f;
    DFX_FOR(i, P.L * 12) s[Y.fx + i] = 0.0f;   // fixed-point wrench accumulators (L x 6 low + high words)
    g.pre_store();
    g.sync();
    if constexpr (Grp::kFusedPhases) {      // K1 of the first substep (later ones: inside integrate_fwd)
        DFX_FOR(i, P.L) kin_local_fwd(P, Y, s, i);
        g.sync();
    }
    for (int sub = 0; sub < a.substeps; ++sub) {
        const bool upd = (sub % a.mm_freq) == 0;
        // (q, qd) ENTERING this substep: every thread fenced its writes before the barrier that closed the previous
        // integrate_fwd (or the loads above), so the store is issued without a barrier of its own
        if (a.tape) g.block_out_part(a.tape, sub, a.N, env, s + Y.q, rf, s + Y.stage, true, true);
        kin_fwd(P, Y, s, g);
        g.phase_sync();
        body_and_contact_fwd<kWrench>(P, Y, s, g, xw);
        muscle_fwd(P, Y, s, g);
        wrench_collect(P, Y, s, g);
        g.phase_sync();
        tau_fwd(P, Y, s, g);
        g.phase_sync();
        if (a.has_derived && sub == a.substeps - 1) dump_derived(P, Y, s, a.derived, env, false, g);
        if (upd) {
            if (Y.overlay) g.sync();               // (Lm, Icmp) overlay (Xl, vj, f, fx): every reader of those is done
            crba_fwd(P, Y, s, g);
            if (a.has_derived && a.derived.H) DFX_FOR(e, DD) a.derived.H[(long long)env * DD + e] = s[Y.A + e];
            g.sync();
            chol_inverse(P, Y, s, g);
            if (a.has_derived && a.derived.L) DFX_FOR(e, DD) a.derived.L[(long long)env * DD + e] = s[Y.Lm + e];
            if (a.tape) g.block_out(a.tape + a.hinv_base, sub / a.mm_freq, a.N, env, s + Y.A, DD, false);
            if (Y.overlay) {                       // the fixed-point accumulators must read zero again
                g.sync();
                DFX_FOR(i, P.L * 12) s[Y.fx + i] = 0.0f;
            }
        }
        solve_fwd(P, Y, s, g);
        // the forward intermediates and q'': fenced before solve_fwd's closing barrier (a bf16 tape converts first and
        // fences again)
        if (a.tape) g.block_out_part(a.tape, sub, a.N, env, s + Y.q, rf, s + Y.stage, false, !rf.bf16);
        if (a.has_derived && sub == a.substeps - 1) dump_derived(P, Y, s, a.derived, env, true, g);
        g.phase_sync();
        g.store_sync();   // (synchronous tape stores / dumps above must finish before integrate_fwd overwrites q, qd)
        integrate_fwd(P, Y, s, a.dt_sub, g);
    }
    DFX_FOR(i, Q) a.q_out[(long long)env * Q + i] = s[Y.q + i];
    DFX_FOR(i, D) a.qd_out[(long long)env * D + i] = s[Y.qd + i];
}

template <bool kWrench = false, class Grp>
DFX_HD void env_step_backward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const StepArgs& a,
                              const DfxExternalWrench& w = DfxExternalWrench{nullptr, nullptr}) {
    const int Q = P.Q, D = P.D, M = P.M, DD = D * D;
    const RowFmt rf = row_fmt(P, Y, a.tape_bf16 != 0);
    const int xw = kWrench ? wrench_offset(Y, true) : -1;
    load_actuation(P, Y, s, g, env, a, false);
    if constexpr (kWrench) {
        load_wrench(P, s, g, env, w, xw);
        DFX_FOR(i, P.L * 6) s[xw + P.L * 6 + i] = 0.0f;
    }
    DFX_FOR(i, D) s[Y.aact + i] = 0.0f;
    DFX_FOR(i, M) s[Y.amusc + i] = 0.0f;
    if (g.lane == 0) s[Y.cmask] = 0.0f;
    if (P.M > 0) DFX_FOR(i, P.L * 13) s[Y.fxH + i] = 0.0f;  // high words of the fixed-point cotangent accumulators
    DFX_FOR(i, Q) s[Y.aq + i] = a.gq_out ? a.gq_out[(long long)env * Q + i] : 0.0f;
    DFX_FOR(i, D) s[Y.aqd + i] = a.gqd_out ? a.gqd_out[(long long)env * D + i] : 0.0f;
    for (int sub = a.substeps - 1; sub >= 0; --sub) {
        const int seg = sub / a.mm_freq;
        const int s0 = seg * a.mm_freq;
        const bool seg_last = (sub == a.substeps - 1) || ((sub + 1) % a.mm_freq == 0);   // first visited of its segment
        // the row arrives in two asynchronous parts: (q, qd, q'') -- all that the first two adjoint phases read -- then
        // the rest, which substep_adj() waits for only before the phases that need it
        if constexpr (Grp::kBulkRows) {
            const bool want_hinv = seg_last && Y.A >= 0;
            g.rows_in(s + Y.q, a.tape_in, sub, rf, s + Y.stage, s + (want_hinv ? Y.A : 0),
                      want_hinv ? g.block_ptr(a.tape_in + a.hinv_base, seg, DD) : nullptr, DD);
            if (sub > 0 && !(a.flags & 128)) g.prefetch_row(a.tape_in, sub - 1, rf);
        } else {
            g.row_in(s + Y.q, a.tape_in, sub, a.N, env, rf.n, rf.early, rf.tail, true);
            if (seg_last && Y.A >= 0) g.block_in(s + Y.A, a.tape_in + a.hinv_base, seg, a.N, env, DD, false);
        }
        if (seg_last) DFX_FOR(e, dfx_sym_count(D)) s[Y.Lm + e] = 0.0f;      // symmetrised cotangent of H (packed)
        // layouts that do not stage H^-1 read its rows from the tape block in place (L2)
        const HinvView hv = (Y.A >= 0) ? HinvView{nullptr, 0} : g.hinv_view(a.tape_in + a.hinv_base, seg, a.N, env, DD);
        if constexpr (!Grp::kBulkRows) g.row_in(s + Y.q, a.tape_in, sub, a.N, env, rf.n, rf.early, rf.tail, false);
        g.copy_wait_first();
        g.sync();
        substep_adj<kWrench>(P, Y, s, a.dt_sub, sub == s0, hv, rf, g, xw);
    }
    if constexpr (kWrench) {
        if (w.g_f_ext) DFX_FOR(i, P.L * 6) w.g_f_ext[(long long)env * P.L * 6 + i] = s[xw + P.L * 6 + i];
    }
    if (a.gq) DFX_FOR(i, Q) a.gq[(long long)env * Q + i] = s[Y.aq + i];
    if (a.gqd) DFX_FOR(i, D) a.gqd[(long long)env * D + i] = s[Y.aqd + i];
    if (a.gact) DFX_FOR(i, D) a.gact[(long long)env * D + i] = s[Y.aact + i];
    if (a.gmusc) DFX_FOR(i, M) a.gmusc[(long long)env * M + i] = s[Y.amusc + i];
    if (a.g_raw) {      // cotangent of the raw policy output (dfx_action_map_backward's arithmetic; clip passes the gradient on [-1, 1])
        const int A = a.map_num_act, src = (a.map_muscle ? Y.amusc : Y.aact) + a.map_offset;
        DFX_FOR(j, A) {
            const float r = a.raw[(long long)env * A + j];
            float gg = a.g_used ? a.g_used[(long long)env * A + j] : 0.0f;
            gg += (s[src + j] * a.strength[j]) * a.map_drive_scale;
            a.g_raw[(long long)env * A + j] = (r >= -1.0f && r <= 1.0f) ? gg * a.map_pre_scale : 0.0f;
        }
    }
}

// ---- link state of (q, qd) (include/dfx.h dfx_link_state_forward / _backward): the kinematics of one substep on its own --
// X_sc, X_sm (reference eval_rigid_fk) and v (the velocity half of eval_rigid_id) -- in the step's forward and backward
// layouts, which hold every field these touch.  The kernels get these pointers as a kernel parameter of their own, next to
// KernelArgs (whose `step.N` and `step.flags` they read), so KernelArgs / StepArgs stay as the step kernels have them.
struct LinkStateArgs {
    const float* q; const float* qd;
    float* X_sc; float* X_sm; float* v_s;                       // forward outputs [N, L, 7 / 7 / 6] (NULL: skip)
    const float* g_X_sc; const float* g_X_sm; const float* g_v_s;   // backward: their cotangents (NULL == 0)
    float* gq; float* gqd;                                      // backward outputs [N, Q], [N, D] (NULL: skip)
};

// (q, qd) -> X_sc, X_sm, S, v, a in the scratch, as a substep's kinematics (K1 first when the fused phases leave it to
// integrate_fwd, as env_step_forward does before its first substep)
template <class Grp>
DFX_HD void link_state_kinematics(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const LinkStateArgs& a) {
    DFX_FOR(i, P.Q) s[Y.q + i] = a.q[(long long)env * P.Q + i];
    DFX_FOR(i, P.D) s[Y.qd + i] = a.qd[(long long)env * P.D + i];
    g.sync();
    if constexpr (Grp::kFusedPhases) {
        DFX_FOR(i, P.L) kin_local_fwd(P, Y, s, i);
        g.sync();
    }
    kin_fwd(P, Y, s, g);
    g.sync();
}

template <class Grp>
DFX_HD void link_state_forward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const LinkStateArgs& a) {
    const int L = P.L;
    link_state_kinematics(P, Y, s, g, env, a);
    if (a.X_sc) DFX_FOR(i, L * 7) a.X_sc[(long long)env * L * 7 + i] = s[Y.Xsc + i];
    if (a.X_sm) DFX_FOR(i, L * 7) a.X_sm[(long long)env * L * 7 + i] = s[Y.Xsm + i];
    if (a.v_s) DFX_FOR(i, L * 6) a.v_s[(long long)env * L * 6 + i] = s[Y.v + i];
}

// adjoint: the kinematics recomputed from (q, qd), the cotangents of X_sc, X_sm, v seeded, nothing downstream (aa, aS zero),
// then A1 for every link and the rest of the kinematics adjoint, as at the end of substep_adj
template <class Grp>
DFX_HD void link_state_backward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const LinkStateArgs& a) {
    const int L = P.L, Q = P.Q, D = P.D;
    link_state_kinematics(P, Y, s, g, env, a);
    DFX_FOR(i, L * 7) s[Y.aXsc + i] = a.g_X_sc ? a.g_X_sc[(long long)env * L * 7 + i] : 0.0f;
    DFX_FOR(i, L * 7) s[Y.aXsm + i] = a.g_X_sm ? a.g_X_sm[(long long)env * L * 7 + i] : 0.0f;
    DFX_FOR(i, L * 6) s[Y.av + i] = a.g_v_s ? a.g_v_s[(long long)env * L * 6 + i] : 0.0f;
    DFX_FOR(i, L * 6) s[Y.aa + i] = 0.0f;
    DFX_FOR(i, D * 6) s[Y.aS + i] = 0.0f;
    DFX_FOR(i, Q) s[Y.aq + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aqd + i] = 0.0f;
    g.sync();
    DFX_FOR(i, L) kin_adj_local(P, Y, s, i);
    g.sync();
    kin_adj(P, Y, s, g);
    g.sync();
    if (a.gq) DFX_FOR(i, Q) a.gq[(long long)env * Q + i] = s[Y.aq + i];
    if (a.gqd) DFX_FOR(i, D) a.gqd[(long long)env * D + i] = s[Y.aqd + i];
}

// ---- contact state of (q, qd) (include/dfx.h dfx_contact_state_forward / _backward): the step's ground-contact model
// (contact_point_fwd) at the state, as the first substep of an env-step from it applies it.  Per point k, in the Model's contact
// order: the force the ground exerts on the link, -ftot (ftot is what the step adds to body_f_s, where it acts like gravity:
// f = f_b - (...)), and the height c of the point above the plane; per link, the sum (tau, F) of its points' forces, tau about
// the link's centre of mass (the DfxExternalWrench convention).  One item per link walks its points in pack order (cbody_start),
// so every sum is in a fixed order, with no atomics.
struct ContactStateArgs {
    const float* q; const float* qd;
    const int* corder;                                          // [C]: Model index of the pack's contact n (dfx_pack_create)
    float* contact_f; float* contact_height; float* body_f;     // forward outputs [N, C, 3], [N, C], [N, L, 6] (NULL: skip)
    const float* g_contact_f; const float* g_contact_height; const float* g_body_f;   // backward: their cotangents (NULL == 0)
    float* gq; float* gqd;                                      // backward outputs [N, Q], [N, D] (NULL: skip)
};

template <class Grp>
DFX_HD void contact_state_kinematics(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const ContactStateArgs& a) {
    LinkStateArgs la{};
    la.q = a.q; la.qd = a.qd;
    link_state_kinematics(P, Y, s, g, env, la);
}

// contact point k (pack order) on link b: the point p after the contact_dist shift, where the step applies the force
DFX_HD V3 contact_point_world(const Pack& P, const Layout& Y, SP s, int b, int k) {
    V3 p = xf_point(ld7(s + Y.Xsc + b * 7), ld3(P.cpoint + k * 3));
    p.y -= P.cdist[k];
    return p;
}

template <class Grp>
DFX_HD void contact_state_forward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const ContactStateArgs& a) {
    const int L = P.L, C = P.C;
    contact_state_kinematics(P, Y, s, g, env, a);
    DFX_FOR(i, L) {
        const V3 cm = ld3(s + Y.Xsm + i * 7);
        V3 F = v3zero(), tau = v3zero();
        for (int k = P.cbody_start[i]; k < P.cbody_start[i + 1]; ++k) {
            const long long o = (long long)env * C + a.corder[k];
            const V3 p = contact_point_world(P, Y, s, i, k);
            const V3 f = P.ground ? v3zero() - contact_point_fwd(P, Y, s, k).v : v3zero();
            if (a.contact_f) st3(a.contact_f + o * 3, f);
            if (a.contact_height) a.contact_height[o] = p.y;
            F += f;
            tau += cross(p - cm, f);
        }
        if (a.body_f) {
            float* w = a.body_f + ((long long)env * L + i) * 6;
            st3(w, tau);
            st3(w + 3, F);
        }
    }
}

// Adjoint of the force model of one penetrating point: the cotangent aftot of ftot -> those of p (ap) and dp/dt (adpdt).  This
// restates the part of contact_point_adj (dfx_phases.h) after its torque term, which it must mirror line for line: that
// function stays as it is so that the step kernels keep their code.
DFX_HD void contact_force_adj(V3 p, V3 dpdt, float ke, float kd, float kf, float mu, V3 aftot, V3& ap, V3& adpdt) {
    const float c = p.y;
    const float vn = dpdt.y;
    const V3 vt = V3{dpdt.x, 0.0f, dpdt.z};
    const float mn = fminf(vn, 0.0f);
    const float len = sqrtf(dot(vt, vt));
    const V3 nvt = len > 0.0f ? V3{vt.x / len, vt.y / len, vt.z / len} : v3zero();
    const float A = kf * len, Bc = 0.0f - mu * c * ke;
    const float cap = fminf(A, Bc);
    const float a_nf = aftot.y;  // d/d(fn+fd)
    const V3 aft = aftot;
    // ft = nvt * cap
    const V3 anvt = aft * cap;
    const float acap = dot(nvt, aft);
    float ac = 0.0f, alen = 0.0f;
    if (A < Bc) alen += kf * acap; else ac += -mu * ke * acap;
    V3 avt = nvt * alen;
    if (len > 0.0f) {
        const float inv = 1.0f / len;
        avt += (anvt - nvt * dot(nvt, anvt)) * inv;
    }
    // fd = min(vn,0) * kd * (-c)
    float avn = 0.0f;
    if (vn < 0.0f) avn += kd * (0.0f - c) * a_nf;
    ac += -(mn * kd) * a_nf;
    // fn = c ke
    ac += ke * a_nf;
    // vt = dpdt - n vn ; vn = dpdt.y
    adpdt = avt;
    avn -= avt.y;
    adpdt.y += avn;
    ap.y += ac;
}

// adjoint: the kinematics recomputed from (q, qd); per link item, its points' cotangents (height: every point; force: penetrating
// points with the ground on) added into aXsc, av and aXsm (the centre of mass of the torque) of that link, in pack order, then A1
// and the rest of the kinematics adjoint, as link_state_backward
template <class Grp>
DFX_HD void contact_state_backward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const ContactStateArgs& a) {
    const int L = P.L, C = P.C, Q = P.Q, D = P.D;
    contact_state_kinematics(P, Y, s, g, env, a);
    DFX_FOR(i, L * 7) s[Y.aXsc + i] = 0.0f;
    DFX_FOR(i, L * 7) s[Y.aXsm + i] = 0.0f;
    DFX_FOR(i, L * 6) s[Y.av + i] = 0.0f;
    DFX_FOR(i, L * 6) s[Y.aa + i] = 0.0f;
    DFX_FOR(i, D * 6) s[Y.aS + i] = 0.0f;
    DFX_FOR(i, Q) s[Y.aq + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aqd + i] = 0.0f;
    g.sync();
    DFX_FOR(i, L) {
        const Xf X = ld7(s + Y.Xsc + i * 7);
        const SV vs = ld6(s + Y.v + i * 6);
        const V3 cm = ld3(s + Y.Xsm + i * 7);
        const V3 gtau = a.g_body_f ? ld3(a.g_body_f + ((long long)env * L + i) * 6) : v3zero();
        const V3 gF = a.g_body_f ? ld3(a.g_body_f + ((long long)env * L + i) * 6 + 3) : v3zero();
        V3 acm = v3zero();
        for (int k = P.cbody_start[i]; k < P.cbody_start[i + 1]; ++k) {
            const long long o = (long long)env * C + a.corder[k];
            const V3 pt = ld3(P.cpoint + k * 3);
            const V3 p = contact_point_world(P, Y, s, i, k);
            V3 ap = v3zero(), aw = v3zero(), adpdt = v3zero();
            if (a.g_contact_height) ap.y += a.g_contact_height[o];
            if (P.ground && !(p.y >= 0.0f)) {       // (a NaN height takes this branch, as in contact_point_adj)
                const V3 f = v3zero() - contact_point_fwd(P, Y, s, k).v;
                // loss terms g_f . f + gF . f + gtau . ((p - cm) x f)
                V3 af = gF, ar = v3zero();
                if (a.g_contact_f) af += ld3(a.g_contact_f + o * 3);
                cross_adj(p - cm, f, gtau, ar, af);
                ap += ar;
                acm -= ar;
                const float ke = P.cmat[k * 4 + 0], kd = P.cmat[k * 4 + 1], kf = P.cmat[k * 4 + 2], mu = P.cmat[k * 4 + 3];
                contact_force_adj(p, vs.v + cross(vs.w, p), ke, kd, kf, mu, v3zero() - af, ap, adpdt);
                // dpdt = v + w x p
                cross_adj(vs.w, p, adpdt, aw, ap);
            }
            // p = X.p + R(X.q) pt - n d
            const Q4 aq = qrot_adj_q(X.q, pt, ap);
            const SP ax = s + Y.aXsc + i * 7;
            const SP avp = s + Y.av + i * 6;
            const float c7[7] = {ap.x, ap.y, ap.z, aq.x, aq.y, aq.z, aq.w};
            const float c6[6] = {aw.x, aw.y, aw.z, adpdt.x, adpdt.y, adpdt.z};
#pragma unroll
            for (int c = 0; c < 7; ++c) ax[c] += c7[c];
#pragma unroll
            for (int c = 0; c < 6; ++c) avp[c] += c6[c];
        }
        add3(s + Y.aXsm + i * 7, acm);
        kin_adj_local(P, Y, s, i);
    }
    g.sync();
    kin_adj(P, Y, s, g);
    g.sync();
    if (a.gq) DFX_FOR(i, Q) a.gq[(long long)env * Q + i] = s[Y.aq + i];
    if (a.gqd) DFX_FOR(i, D) a.gqd[(long long)env * D + i] = s[Y.aqd + i];
}

// ---- dynamics state of (q, qd, act, musc, f_ext) (include/dfx.h dfx_dynamics_state_forward / _backward): what the first substep
// of an env-step from the state computes before it integrates -- the joint forces tau (the right-hand side of the solve), the
// joint-space inertia H = J^T M J (without armature) and q'' = (H + diag(armature))^-1 tau.  The wrench is always built in
// (f_ext NULL reads as zero), so the scratch ends past the layout's (dfx_pack.h wrench_scratch_end).
struct DynamicsStateArgs {
    const float* q; const float* qd; const float* act; const float* musc; const float* f_ext;   // inputs (f_ext NULL == 0)
    float* joint_qdd; float* joint_tau; float* H;               // forward outputs [N, D], [N, D], [N, D, D] (NULL: skip)
    const float* g_qdd; const float* g_tau; const float* g_H;   // backward: their cotangents (NULL == 0; g_H need not be symmetric)
    float* gq; float* gqd; float* gact; float* gmusc; float* g_f_ext;   // backward outputs [N, Q / D / D / M / L*6] (NULL: skip)
};

// The first substep of env_step_forward<true> up to and including solve_fwd, phase for phase and barrier for barrier, with the
// stores of the derived dumps (tau after tau_fwd, H after crba_fwd, q'' after solve_fwd) and no tape.  It restates that function,
// which it must stay in step with: env_step_forward stays as it is so that the step kernels keep their code, and the readouts are
// checked bit for bit against the derived dumps of a one-substep env-step.
template <class Grp>
DFX_HD void dynamics_state_forward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const DynamicsStateArgs& a) {
    const int Q = P.Q, D = P.D, M = P.M, L = P.L, DD = D * D;
    const int xw = wrench_offset(Y, false);
    DFX_FOR(i, Q) s[Y.q + i] = a.q[(long long)env * Q + i];
    DFX_FOR(i, D) s[Y.qd + i] = a.qd[(long long)env * D + i];
    DFX_FOR(i, D) s[Y.act + i] = a.act[(long long)env * D + i];
    DFX_FOR(i, M) s[Y.musc + i] = a.musc[(long long)env * M + i];
    DFX_FOR(i, L * 6) s[xw + i] = a.f_ext ? a.f_ext[(long long)env * L * 6 + i] : 0.0f;
    if (g.lane == 0) s[Y.cmask] = 0.0f;
    DFX_FOR(i, L * 12) s[Y.fx + i] = 0.0f;   // fixed-point wrench accumulators
    g.sync();
    if constexpr (Grp::kFusedPhases) {
        DFX_FOR(i, L) kin_local_fwd(P, Y, s, i);
        g.sync();
    }
    kin_fwd(P, Y, s, g);
    g.phase_sync();
    body_and_contact_fwd<true>(P, Y, s, g, xw);
    muscle_fwd(P, Y, s, g);
    wrench_collect(P, Y, s, g);
    g.phase_sync();
    tau_fwd(P, Y, s, g);
    g.phase_sync();
    if (a.joint_tau) DFX_FOR(i, D) a.joint_tau[(long long)env * D + i] = s[Y.tau + i];
    if (Y.overlay) g.sync();               // (Lm, Icmp) overlay (Xl, vj, f, fx): every reader of those is done
    crba_fwd(P, Y, s, g);
    if (a.H) DFX_FOR(e, DD) a.H[(long long)env * DD + e] = s[Y.A + e];
    g.sync();
    chol_inverse(P, Y, s, g);
    solve_fwd(P, Y, s, g);
    if (a.joint_qdd) DFX_FOR(i, D) a.joint_qdd[(long long)env * D + i] = s[Y.qdd + i];
}

// Adjoint, on the tape row and H^-1 block of a one-substep env-step from the same inputs (ta.tape_in: substeps = mm_freq = 1, fp32
// rows, the external-wrench path; env_step_backward's loads): aq = aqd = 0, aqdd = g_qdd, the packed symmetrised cotangent of H
// (Lm slot) = sym(g_H) -- g_H + g_H^T off the diagonal, as solve_adj keeps it -- instead of zero, then substep_adj<true, true>:
// no integrator adjoint, g_tau joining the cotangent of tau after solve_adj.  Outputs as env_step_backward<true> writes them.
template <class Grp>
DFX_HD void dynamics_state_backward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const StepArgs& ta,
                                    const DynamicsStateArgs& a) {
    const int Q = P.Q, D = P.D, M = P.M, L = P.L, DD = D * D;
    const RowFmt rf = row_fmt(P, Y, false);
    const int xw = wrench_offset(Y, true);
    DFX_FOR(i, D) s[Y.act + i] = a.act[(long long)env * D + i];
    DFX_FOR(i, M) s[Y.musc + i] = a.musc[(long long)env * M + i];
    DFX_FOR(i, L * 6) s[xw + i] = a.f_ext ? a.f_ext[(long long)env * L * 6 + i] : 0.0f;
    DFX_FOR(i, L * 6) s[xw + L * 6 + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aact + i] = 0.0f;
    DFX_FOR(i, M) s[Y.amusc + i] = 0.0f;
    if (g.lane == 0) s[Y.cmask] = 0.0f;
    if (M > 0) DFX_FOR(i, L * 13) s[Y.fxH + i] = 0.0f;
    DFX_FOR(i, Q) s[Y.aq + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aqd + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aqdd + i] = a.g_qdd ? a.g_qdd[(long long)env * D + i] : 0.0f;
    if constexpr (Grp::kBulkRows) {
        g.rows_in(s + Y.q, ta.tape_in, 0, rf, s + Y.stage, s + (Y.A >= 0 ? Y.A : 0),
                  Y.A >= 0 ? g.block_ptr(ta.tape_in + ta.hinv_base, 0, DD) : nullptr, DD);
    } else {
        g.row_in(s + Y.q, ta.tape_in, 0, ta.N, env, rf.n, rf.early, rf.tail, true);
        if (Y.A >= 0) g.block_in(s + Y.A, ta.tape_in + ta.hinv_base, 0, ta.N, env, DD, false);
    }
    DFX_FOR(i, D) {                 // row i of the packed triangle: entries (i, i..D-1)
        const SP row = s + Y.Lm + symD_idx(D, i, i);
        if (a.g_H) {
            const float* gH = a.g_H + (long long)env * DD;
            row[0] = gH[i * D + i];
            for (int j = i + 1; j < D; ++j) row[j - i] = gH[i * D + j] + gH[j * D + i];
        } else {
            for (int j = i; j < D; ++j) row[j - i] = 0.0f;
        }
    }
    const HinvView hv = (Y.A >= 0) ? HinvView{nullptr, 0} : g.hinv_view(ta.tape_in + ta.hinv_base, 0, ta.N, env, DD);
    if constexpr (!Grp::kBulkRows) g.row_in(s + Y.q, ta.tape_in, 0, ta.N, env, rf.n, rf.early, rf.tail, false);
    g.copy_wait_first();
    g.sync();
    substep_adj<true, true>(P, Y, s, 0.0f, true, hv, rf, g, xw, a.g_tau ? a.g_tau + (long long)env * D : nullptr);
    if (a.g_f_ext) DFX_FOR(i, L * 6) a.g_f_ext[(long long)env * L * 6 + i] = s[xw + L * 6 + i];
    if (a.gq) DFX_FOR(i, Q) a.gq[(long long)env * Q + i] = s[Y.aq + i];
    if (a.gqd) DFX_FOR(i, D) a.gqd[(long long)env * D + i] = s[Y.aqd + i];
    if (a.gact) DFX_FOR(i, D) a.gact[(long long)env * D + i] = s[Y.aact + i];
    if (a.gmusc) DFX_FOR(i, M) a.gmusc[(long long)env * M + i] = s[Y.amusc + i];
}

// ---- Jacobian state of (q, qd) (include/dfx.h dfx_jacobian_state_forward / _backward): the link Jacobians J [L, 6, D] -- column d
// of link i's block is S[d] when dof d moves link i (a dof of i or of an ancestor: the pack's anc_dofs list of i), 0 otherwise -- and
// the bias accelerations a (reference State body_a_s, J-dot qd), both from the kinematics link_state_kinematics leaves in the scratch.
struct JacobianStateArgs {
    const float* q; const float* qd;
    float* J; float* a_s;                           // forward outputs [N, L, 6, D], [N, L, 6] (NULL: skip)
    const float* g_J; const float* g_a_s;           // backward: their cotangents (NULL == 0)
    float* gq; float* gqd;                          // backward outputs [N, Q], [N, D] (NULL: skip)
};

// element k = (i * 6 + r) * D + d of one environment's J: S[d][r] when d is in link i's ancestor-or-self dof list (ascending), else 0
DFX_HD float jacobian_entry(const Pack& P, const Layout& Y, SP s, int k) {
    const int D = P.D, d = k % D, ir = k / D, i = ir / 6, r = ir - i * 6;
    for (int j = P.anc_start[i]; j < P.anc_start[i + 1]; ++j) {
        const int a = P.anc_dofs[j];
        if (a >= d) return a == d ? s[Y.S + d * 6 + r] : 0.0f;
    }
    return 0.0f;
}

// every element of J is written (zeros included), one environment per item group
template <class Grp>
DFX_HD void jacobian_state_forward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const JacobianStateArgs& a) {
    const int L = P.L, LD6 = L * 6 * P.D;
    LinkStateArgs la{};
    la.q = a.q; la.qd = a.qd;
    link_state_kinematics(P, Y, s, g, env, la);
    if (a.J) DFX_FOR(k, LD6) a.J[(long long)env * LD6 + k] = jacobian_entry(P, Y, s, k);
    if (a.a_s) DFX_FOR(i, L * 6) a.a_s[(long long)env * L * 6 + i] = s[Y.a + i];
}

// adjoint: the kinematics recomputed from (q, qd); aS[d][r] = the sum of g_J[l][r][d] over the links l that dof d moves (the subtree
// of its link, sub_links in list order; one item per link over its dofs and rows -- no atomics, so the sums are bit-reproducible),
// aa = g_a_s, the other cotangents zero; then A1 for every link and the rest of the kinematics adjoint, as link_state_backward
template <class Grp>
DFX_HD void jacobian_state_backward(const Pack& P, const Layout& Y, SP s, const Grp& g, int env, const JacobianStateArgs& a) {
    const int L = P.L, Q = P.Q, D = P.D, LD6 = L * 6 * D;
    LinkStateArgs la{};
    la.q = a.q; la.qd = a.qd;
    link_state_kinematics(P, Y, s, g, env, la);
    DFX_FOR(i, L * 7) s[Y.aXsc + i] = 0.0f;
    DFX_FOR(i, L * 7) s[Y.aXsm + i] = 0.0f;
    DFX_FOR(i, L * 6) s[Y.av + i] = 0.0f;
    DFX_FOR(i, L * 6) s[Y.aa + i] = a.g_a_s ? a.g_a_s[(long long)env * L * 6 + i] : 0.0f;
    DFX_FOR(i, L) {          // (one item per link, over its dofs and rows)
        for (int d = P.qd_start[i]; d < P.qd_start[i + 1]; ++d) {
            for (int r = 0; r < 6; ++r) {
                float acc = 0.0f;
                if (a.g_J)
                    for (int k = P.sub_start[i]; k < P.sub_start[i + 1]; ++k)
                        acc += a.g_J[(long long)env * LD6 + (P.sub_links[k] * 6 + r) * D + d];
                s[Y.aS + d * 6 + r] = acc;
            }
        }
    }
    DFX_FOR(i, Q) s[Y.aq + i] = 0.0f;
    DFX_FOR(i, D) s[Y.aqd + i] = 0.0f;
    g.sync();
    DFX_FOR(i, L) kin_adj_local(P, Y, s, i);
    g.sync();
    kin_adj(P, Y, s, g);
    g.sync();
    if (a.gq) DFX_FOR(i, Q) a.gq[(long long)env * Q + i] = s[Y.aq + i];
    if (a.gqd) DFX_FOR(i, D) a.gqd[(long long)env * D + i] = s[Y.aqd + i];
}

}  // namespace dfx
