// dfx_phases.h -- the phases of one semi-implicit substep of the articulated rigid-body
// simulator and their hand-derived adjoints, written once against two abstractions: the group policy `Grp`
// (which items of a loop this thread takes, what a barrier is, how tape blocks move) and the scratch pointer `SP`
// (dfx_math.h: an environment's working set, contiguous or strided).  Instantiated by the tile kernels
// (dfx_tile.cu: lane = environment, warp = item), the lane-group kernels (dfx_kernels.cu: lanes = items of one
// environment) and the host emulation (tests/host_emu).
//
// What is computed follows the reference step (NVlabs/DiffRL dflex/dflex/sim.py:2316-2601):
//   kin_*         eval_rigid_fk :1681 + the velocity half of eval_rigid_id :1716-1763
//   body_force_*  the force half of eval_rigid_id :1765-1787 (+ spatial_transform_inertia :1116)
//   contact_*     eval_rigid_contacts_art :1137
//   muscle_*      eval_muscles :1245 / compute_muscle_force :1209
//   tau_*         eval_rigid_tau :1896 / jcalc_tau :1421
//   crba_*        eval_rigid_jacobian/mass + the two batched GEMMs + Cholesky :2475-2561
//   solve_*       eval_dense_solve_batched :2047 (adjoint: matnn.h:310-336)
//   integrate_*   eval_rigid_integrate :2052 / jcalc_integrate :1505
// HOW it is computed is different by design: the joint-space inertia H = J^T M J is accumulated
// with the composite-rigid-body recursion instead of two dense GEMMs, the 6x6 world inertia
// T^T I T is never formed per substep (it is applied in factored form), q'' = H^-1 tau uses an explicitly formed
// H^-1 (one mat-vec per substep instead of two triangular sweeps), scatter-adds are order-independent
// fixed-point integer adds in shared memory, and each substep tapes the block [q .. q''] of its scratch (the
// entering state AND the forward intermediates): the adjoint reads it back instead of re-running the forward.
//
// `Grp` provides: static G, lane, kPathPasses, kConcurrentItems, sync(), cta_tasks(), cta_compact(), cta_compact_with(),
// fx_add(int*, int), atomic_add(float*, float), atomic_or(unsigned*, unsigned), group_max(float, SP slot),
// block_in() / row_in() / block_out() / copy_wait_first() / copy_wait_all() for the tape.
#pragma once

#include <string.h>

#include "dfx_math.h"
#include "dfx_pack.h"

namespace dfx {

// A view of H^-1: in the scratch (stride = the scratch element stride) or, when the layout does not stage it
// (Y.A < 0), in the tape block in global memory (element stride hs)
struct HinvView {
    const float* g;   // global rows, or nullptr
    int hs;
};

// Geometry of a tape row of n scratch floats: [0, early) = (q, qd), known when the substep starts and all that the first two
// adjoint phases need (with q''); [early, tail) = the forward intermediates; [tail, n) = q'' + padding.  With a bf16 tape the
// sub-range [head, tail) = (v, a, f_tot) is stored as bf16 ([early, head) = the link transforms and S stay fp32); otherwise
// head == early.  `units` = 4-byte units the row occupies in the tape: n, or n - (tail - head) / 2.
struct RowFmt {
    int n, early, head, tail, units;
    bool bf16;
};
DFX_HD RowFmt row_fmt(const Pack& P, const Layout& Y, bool bf16) {
    const int early = P.Q + P.D;
    return RowFmt{Y.tape_row, early, bf16 ? Y.v - Y.q : early, Y.qdd - Y.q, dfx_row_units(Y.tape_row, P.L, P.D, bf16), bf16};
}
// fp32 -> bf16 -> fp32 (round to nearest even), what a bf16 tape does to a value
DFX_HD float bf16_round(float x) {
    unsigned u;
#if defined(__CUDA_ARCH__)
    u = __float_as_uint(x);
#else
    memcpy(&u, &x, 4);
#endif
    if ((u & 0x7f800000u) != 0x7f800000u) u += 0x7fffu + ((u >> 16) & 1u);     // (NaN / Inf keep their payload)
    u &= 0xffff0000u;
    float r;
#if defined(__CUDA_ARCH__)
    r = __uint_as_float(u);
#else
    memcpy(&r, &u, 4);
#endif
    return r;
}

struct GroupSerial {  // host / single-lane execution
    static constexpr int G = 1;
#ifndef DFX_EMU_PATH_PASSES
#define DFX_EMU_PATH_PASSES 0
#endif
    static constexpr bool kPathPasses = DFX_EMU_PATH_PASSES != 0;   // see kin_fwd / tau_fwd
#ifndef DFX_EMU_FUSED_PHASES
#define DFX_EMU_FUSED_PHASES 0
#endif
    // phases merged to save CTA-wide barriers (tile kernels): the joint-local transforms of the NEXT substep are formed by the
    // thread that integrates the link (integrate_fwd), and the torque adjoint recomputes the ancestors' direct cotangents along
    // each link's root path instead of staging them (tau_adj) -- the same operations in the same order, bit-identical results
    static constexpr bool kFusedPhases = DFX_EMU_FUSED_PHASES != 0;
    int lane;
    DFX_HD void sync() const {}
    DFX_HD void phase_sync() const {}
    DFX_HD void atomic_or(unsigned* p, unsigned v) const { *p |= v; }
    DFX_HD void fx_add(int* p, int v) const { *p += v; }
    DFX_HD void atomic_add(float* p, float v) const { *p += v; }
    DFX_HD float group_max(float v, SP slot) const { (void)slot; return v; }
    // run f(scratch of env, k) for k in [0, n) for every environment the executing CTA holds (here: this one)
    template <class F>
    DFX_HD void cta_tasks(SP s, int n, bool lead, F f) const { (void)lead; for (int k = 0; k < n; ++k) f(s, k); }
    // same, restricted to the (k, env) pairs for which pred() holds (compacted first)
    template <class Pr, class F>
    DFX_HD void cta_compact(SP s, int n, Pr pred, F f) const { for (int k = 0; k < n; ++k) if (pred(s, k)) f(s, k); }
    // cta_compact() plus m independent dense items item(s, k): the two kinds of work may run concurrently
    template <class Pr, class F, class H>
    DFX_HD void cta_compact_with(SP s, int n, Pr pred, F f, int m, H item) const {
        for (int k = 0; k < m; ++k) item(s, k);
        for (int k = 0; k < n; ++k) if (pred(s, k)) f(s, k);
    }
    static constexpr bool kConcurrentItems = false;   // cta_compact_with() really overlaps the two
    // tape blocks: block `b` of environment `env` holds n floats ([b][env][n] here and in the lane-group kernels,
    // [b][tile of 32 envs][n][32] in the tile kernels).  `rows`: n is a multiple of 4 and 16-byte aligned (vector
    // / asynchronous copies allowed); block_in may complete asynchronously until copy_wait_all().
    DFX_HD void block_out(float* base, long long b, int N, int env, SP src, int n, bool rows) const {
        (void)rows;
        float* d = base + (b * N + env) * n;
        for (int i = 0; i < n; ++i) d[i] = src[i];
    }
    // a tape row in two stores: `first`: elements [0, head) -- the state entering the substep, known when it starts;
    // then [head, n) once the substep's intermediates exist.  (Policies without asynchronous stores write the whole row
    // with the second call.)
    // (the host emulation keeps the fp32 tape layout and only ROUNDS the middle through bf16 when f.bf16 is set: the
    //  same values the tile kernels read back from a bf16 tape)
    DFX_HD void block_out_part(float* base, long long b, int N, int env, SP src, const RowFmt& f, SP stage, bool first, bool fenced = false) const {
        (void)stage; (void)fenced;
        float* d = base + (b * N + env) * f.n;
        if (first) { for (int i = 0; i < f.early; ++i) d[i] = src[i]; }
        else { for (int i = f.early; i < f.n; ++i) d[i] = (f.bf16 && i >= f.head && i < f.tail) ? bf16_round(src[i]) : src[i]; }
    }
    DFX_HD void row_unpack(SP dst, SP stage, const RowFmt& f) const { (void)dst; (void)stage; (void)f; }
    DFX_HD void row_reusable() const {}        // every asynchronous store has finished READING the scratch
    // pre_store(): called by every thread before the barrier that precedes a block_out_part(..., fenced = true): policies
    // with asynchronous (bulk) stores publish their scratch writes to the async proxy here, so that the store can be issued
    // right after that barrier without a fence + barrier of its own
    DFX_HD void pre_store() const {}
    DFX_HD void store_sync() const {}          // orders a synchronous tape store before the scratch is overwritten (no-op for bulk stores)
    DFX_HD void finish() const {}
    static constexpr bool kBulkRows = false;   // true: env_step_backward moves rows with rows_in() (TMA bulk copies)
    DFX_HD void block_in(SP dst, const float* base, long long b, int N, int env, int n, bool rows) const {
        (void)rows;
        const float* t = base + (b * N + env) * n;
        for (int i = 0; i < n; ++i) dst[i] = t[i];
    }
    // a tape row in two parts: first == true: elements [0, head) and [tail, n); first == false: [head, tail)
    DFX_HD void row_in(SP dst, const float* base, long long b, int N, int env, int n, int head, int tail, bool first) const {
        const float* t = base + (b * N + env) * n;
        for (int i = 0; i < n; ++i) if (((i < head) || (i >= tail)) == first) dst[i] = t[i];
    }
    // where block b of environment env starts in a [b][env][n] tape, and its element stride
    DFX_HD HinvView hinv_view(const float* base, long long b, int N, int env, int n) const { return HinvView{base + (b * N + env) * n, 1}; }
    DFX_HD void copy_wait_first() const {}     // all asynchronous copies but the most recent one have landed
    DFX_HD void copy_wait_all() const {}
};

// joint-type test that folds away for the types an articulation does not have (P.jmask is a compile-time constant in the
// size-specialised tile kernels, dfx_pack.h)
DFX_HD bool is_joint(const Pack& P, int type, int t) { return ((P.jmask >> t) & 1) != 0 && type == t; }

#define DFX_FOR(i, n) for (int i = g.lane; i < (n); i += Grp::G)

// One level of a HEAVY tree recursion (the two leaf->root passes of the kinematics adjoint).  A level of a DiffRL
// articulation holds 1-4 links, so a lane group of 16 or 32 runs it with most lanes idle; cta_tasks() instead spreads
// the (link, environment) pairs of ALL the environments of the CTA over consecutive threads, link-major: a level
// is then typically ONE warp with full lanes, uniform joint types and broadcast pack reads, at the price of a
// CTA-wide barrier per level.  The adjoint recursions gain from it; the light forward recursions (one
// transform product or two vector adds per level) lose more to the barriers than they gain and stay per group.
template <class Grp, class F>
DFX_HD void level_tasks(const Pack& P, SP s, int lev, bool lead, const Grp& g, F f) {
    const int b = P.level_start[lev], e = P.level_start[lev + 1];
    g.cta_tasks(s, e - b, lead, [&](SP se, int k) { f(se, P.level_links[b + k]); });
}

// Tree recursions by CHAINS (dfx_pack.h): a chain of links without side branches is walked by ONE thread, so consecutive
// links need no barrier; chains that hang below other chains run in an earlier round.  One barrier per round (2-3) instead
// of one per tree level (Humanoid: 10), the same per-link operations in the same order.
// `lead`: what the chains read was last written under group-level barriers only (lane-group kernels spread the tasks of a
// round over the whole CTA: the first round then needs a CTA-wide barrier in front)
template <class Grp, class F>
DFX_HD void chain_rounds_up(const Pack& P, SP s, const Grp& g, F f, bool lead = false) {        // leaves -> root
    for (int r = 0; r < P.nround; ++r) {
        const int b = P.round_start[r], e = P.round_start[r + 1];
        g.cta_tasks(s, e - b, lead && r == 0, [&](SP se, int k) {
            for (int j = P.chain_start[b + k]; j < P.chain_start[b + k + 1]; ++j) f(se, P.chain_links[j]);
        });
    }
}
template <class Grp, class F>
DFX_HD void chain_rounds_down(const Pack& P, SP s, const Grp& g, F f, bool lead = false, bool skip_roots = false) {      // root -> leaves
    // skip_roots: f() does nothing for a root (it only pulls from the parent): a top round of lone roots is skipped
    const int top = P.nround - 1 - ((skip_roots && P.root_round_single && P.nround > 1) ? 1 : 0);
    for (int r = top; r >= 0; --r) {
        const int b = P.round_start[r], e = P.round_start[r + 1];
        g.cta_tasks(s, e - b, lead && r == top, [&](SP se, int k) {
            for (int j = P.chain_start[b + k + 1] - 1; j >= P.chain_start[b + k]; --j) f(se, P.chain_links[j]);
        });
    }
}

template <class Grp>
DFX_HD void zero_range(SP p, int n, const Grp& g) {
    DFX_FOR(i, n) p[i] = 0.0f;
}

// =====================================================================================
// kinematics: transforms, motion subspace, velocity and bias acceleration.
// Organised as PARALLEL per-link passes:
//   K1 (parallel)   X_l = X_pj X_jc(q)                                  joint-local transform
//   K2   (root->leaf, or per link along its path) X_sc = X_sc[parent] X_l
//   K3 (parallel)   X_sm = X_sc X_cm ;
//                   X_sj = X_sc[parent] X_pj ; S ; v_j = S qd
//   K4   (root->leaf, or per link along its path) v = v[parent] + v_j ; a = a[parent] + v x v_j
// With Grp::kPathPasses (tile kernels: every barrier is CTA-wide) each link walks its own path from the root
// instead of waiting for its parent -- three barriers per substep, same operations in the same order; the
// lane-group kernels (cheap barriers, deeper trees) keep the level-by-level recursions K2 / K4.
// Scratch: Y.Xl (L,7) and Y.vj (L,6).
// =====================================================================================
DFX_HD Xf joint_transform(const Pack& P, SP q, int i) {
    const int type = P.type[i], qs = P.q_start[i];
    Xf Xjc = xf_ident();
    if (is_joint(P, type, JOINT_PRISMATIC)) Xjc.p = ld3(P.axis + i * 3) * q[qs];
    else if (is_joint(P, type, JOINT_REVOLUTE)) Xjc.q = q_from_axis_angle(ld3(P.axis + i * 3), q[qs]);
    else if (is_joint(P, type, JOINT_BALL)) Xjc.q = ld4(q + qs);
    else if (is_joint(P, type, JOINT_FREE)) { Xjc.p = ld3(q + qs); Xjc.q = ld4(q + qs + 3); }
    return Xjc;
}

DFX_HD void kin_local_fwd(const Pack& P, const Layout& Y, SP s, int i) {   // K1
    st7(s + Y.Xl + i * 7, xf_mul_rn(ld7(P.X_pj + i * 7), joint_transform(P, s + Y.q, i)));   // (see xf_mul_rn)
}

// call f(p) for the links on the path root -> ... -> parent(i) [-> i], in that order (the pack lists every link's path:
// independent look-ups instead of a chain of dependent parent[] loads per depth)
template <class F>
DFX_HD void for_path_root_first(const Pack& P, int i, bool include_self, F f) {
    const int b = P.path_start[i], e = P.path_start[i + 1] - (include_self ? 0 : 1);
    for (int k = b; k < e; ++k) f(P.path_links[k]);
}

// K2: X_sc[parent] as the product of the joint-local transforms along the path from the root, multiplied in the
// same order (and so to the same bits) as a level-by-level recursion X_sc = X_sc[parent] X_l would
DFX_HD Xf kin_parent_transform(const Pack& P, const Layout& Y, SP s, int i) {
    Xf Xp = xf_ident();
    // X_sc = X_sp (X_pj X_jc): same association as the reference (sim.py:1668) so that even the
    // derivative along |q| (q is not assumed unit) agrees
    for_path_root_first(P, i, false, [&](int p) { Xp = xf_mul(Xp, ld7(s + Y.Xl + p * 7)); });
    return Xp;
}

// K3, and with PATH also K2 (X_sc of this link from the path product instead of a preceding level recursion)
template <bool PATH>
DFX_HD void kin_motion_fwd(const Pack& P, const Layout& Y, SP s, int i) {
    const int par = P.parent[i], type = P.type[i], ds = P.qd_start[i];
    Xf Xp, Xsc;
    if (PATH) {
        Xp = kin_parent_transform(P, Y, s, i);
        Xsc = xf_mul(Xp, ld7(s + Y.Xl + i * 7));
        st7(s + Y.Xsc + i * 7, Xsc);
    } else {
        Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
        Xsc = ld7(s + Y.Xsc + i * 7);
    }
    const Xf Xsj = xf_mul(Xp, ld7(P.X_pj + i * 7));
    const V3 axis = ld3(P.axis + i * 3);
    const SP qd = s + Y.qd;
    const SP S = s + Y.S;
    SV vj = sv_zero();
    if (is_joint(P, type, JOINT_PRISMATIC)) {
        SV Sk = SV{v3zero(), qrot(Xsj.q, axis)};
        st6(S + ds * 6, Sk);
        vj = Sk * qd[ds];
    } else if (is_joint(P, type, JOINT_REVOLUTE)) {
        V3 w = qrot(Xsj.q, axis);
        SV Sk = SV{w, cross(Xsj.p, w)};
        st6(S + ds * 6, Sk);
        vj = Sk * qd[ds];
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k) {
            V3 e = V3{k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f};
            V3 w = qrot(Xsj.q, e);
            SV Sk = SV{w, cross(Xsj.p, w)};
            st6(S + (ds + k) * 6, Sk);
            vj = (k == 0) ? Sk * qd[ds] : vj + Sk * qd[ds + k];
        }
    } else if (is_joint(P, type, JOINT_FREE)) {
        for (int k = 0; k < 6; ++k)
            for (int c = 0; c < 6; ++c) S[(ds + k) * 6 + c] = (k == c) ? 1.0f : 0.0f;
        vj = ld6(qd + ds);
    }
    st6(s + Y.vj + i * 6, vj);
    st7(s + Y.Xsm + i * 7, xf_mul(Xsc, ld7(P.X_cm + i * 7)));
}

DFX_HD void kin_velocity_path_fwd(const Pack& P, const Layout& Y, SP s, int i) {  // K4
    // v = v[parent] + v_j ; a = a[parent] + v x v_j, accumulated along the path from the root (same order, same bits)
    SV v = sv_zero(), a = sv_zero();
    for_path_root_first(P, i, true, [&](int p) {
        const SV vj = ld6(s + Y.vj + p * 6);
        v = v + vj;
        a = a + sv_cross(v, vj);
    });
    st6(s + Y.v + i * 6, v);
    st6(s + Y.a + i * 6, a);
}

DFX_HD void kin_chain_fwd(const Pack& P, const Layout& Y, SP s, int i) {   // K2
    const int par = P.parent[i];
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    // X_sc = X_sp (X_pj X_jc): same association as the reference (sim.py:1668) so that even the
    // derivative along |q| (q is not assumed unit) agrees
    st7(s + Y.Xsc + i * 7, xf_mul(Xp, ld7(s + Y.Xl + i * 7)));
}

DFX_HD void kin_velocity_fwd(const Pack& P, const Layout& Y, SP s, int i) {  // K4
    const int par = P.parent[i];
    SV vp = sv_zero(), ap = sv_zero();
    if (par >= 0) { vp = ld6(s + Y.v + par * 6); ap = ld6(s + Y.a + par * 6); }
    const SV vj = ld6(s + Y.vj + i * 6);
    const SV v = vp + vj;
    st6(s + Y.v + i * 6, v);
    st6(s + Y.a + i * 6, ap + sv_cross(v, vj));
}

template <class Grp>
DFX_HD void kin_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if constexpr (!Grp::kFusedPhases) {
        DFX_FOR(i, P.L) kin_local_fwd(P, Y, s, i);
        g.row_reusable();      // (K1 wrote temporaries only; from the next pass on the tape row of the previous substep is overwritten)
        g.sync();
    }   // (kFusedPhases: K1 ran at the end of the previous substep, inside integrate_fwd -- or before the first substep)
    if constexpr (Grp::kPathPasses) {
        // every barrier is CTA-wide here: each link walks its own path from the root, three barriers in all
        DFX_FOR(i, P.L) kin_motion_fwd<true>(P, Y, s, i);
        g.sync();
        DFX_FOR(i, P.L) kin_velocity_path_fwd(P, Y, s, i);
        g.sync();
    } else {
        // root -> leaf recursions by chains: one barrier per round, each link multiplies ONE transform (O(L) work; the path
        // passes above do O(L * depth) to save the rounds' barriers)
        chain_rounds_down(P, s, g, [&](SP se, int i) { kin_chain_fwd(P, Y, se, i); }, true);
        DFX_FOR(i, P.L) kin_motion_fwd<false>(P, Y, s, i);
        g.sync();
        chain_rounds_down(P, s, g, [&](SP se, int i) { kin_velocity_fwd(P, Y, se, i); }, true);
    }
}

// ---- adjoint.  On entry aXsc[i], aXsm[i], aS[dofs of i], av[i], aa[i] hold the cotangents from everything
// downstream of the kinematics.  Passes (leaves -> root recursions are thin):
//   A1 (parallel)   aXsc += adj(X_sm = X_sc X_cm) ; recompute X_l, v_j
//   A2 (leaf->root) av, aa totals (children gathered), adjoint of a = a_p + v x v_j  -> avj (in the vj slot)
//   A3 (parallel)   adjoint of v_j = S qd and of S(X_sj): aS, aqd, aX_sj and its push to the parent (pX slot)
//   A4 (leaf->root) aXsc totals (children's pushes gathered); push of this link to its parent -> pX
//   A5 (parallel)   adjoint of X_l = X_pj X_jc(q) -> aq
// A1 runs as the tail of the rigid-body force adjoint of the SAME link (body_force_link_adj: aXsm[i] is final there and
// everything A1 touches is private to the link): it leaves the link's contribution to aXsc in the aXsm slot -- A4 adds it --
// so it never races with the contact / muscle cotangents that other threads scatter into aXsc at the same time.
DFX_HD void kin_adj_local(const Pack& P, const Layout& Y, SP s, int i) {    // A1
    Xf acc = xf_zero();
    xf_mul_adj_a(ld7(s + Y.Xsc + i * 7), ld7(P.X_cm + i * 7), ld7(s + Y.aXsm + i * 7), acc);
    st7(s + Y.aXsm + i * 7, acc);                       // from here on: d/dX_sc[i] through X_sm = X_sc X_cm
    st7(s + Y.Xl + i * 7, xf_mul_rn(ld7(P.X_pj + i * 7), joint_transform(P, s + Y.q, i)));   // (see xf_mul_rn)
    const int type = P.type[i], ds = P.qd_start[i];
    const SP qd = s + Y.qd;
    const SP S = s + Y.S;
    SV vj = sv_zero();
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) vj = ld6(S + ds * 6) * qd[ds];
    else if (is_joint(P, type, JOINT_BALL)) { for (int k = 0; k < 3; ++k) vj += ld6(S + (ds + k) * 6) * qd[ds + k]; }
    else if (is_joint(P, type, JOINT_FREE)) vj = ld6(qd + ds);
    st6(s + Y.vj + i * 6, vj);
}

#ifndef DFX_KIN_ADJ_CHAINS
#define DFX_KIN_ADJ_CHAINS 0     // 1: the leaf -> root recursions A2 / A4 as chain rounds (A/B builds); 0: as subtree sums
#endif

#if DFX_KIN_ADJ_CHAINS
DFX_HD void kin_adj_velocity(const Pack& P, const Layout& Y, SP s, int i) {  // A2
    SV av = ld6(s + Y.av + i * 6), aa = ld6(s + Y.aa + i * 6);
    for (int k = P.child_start[i]; k < P.child_start[i + 1]; ++k) {
        const int c = P.child_idx[k];
        av += ld6(s + Y.av + c * 6);
        aa += ld6(s + Y.aa + c * 6);
    }
    SV avj = sv_zero();
    sv_cross_adj(ld6(s + Y.v + i * 6), ld6(s + Y.vj + i * 6), aa, av, avj);   // a = a_p + v x v_j
    avj += av;                                                                // v = v_p + v_j
    st6(s + Y.av + i * 6, av);   // == cotangent pushed to v[parent]
    st6(s + Y.aa + i * 6, aa);
    st6(s + Y.vj + i * 6, avj);
}

DFX_HD void kin_adj_motion(const Pack& P, const Layout& Y, SP s, int i) {    // A3
    const int par = P.parent[i], type = P.type[i], ds = P.qd_start[i];
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    const Xf Xsj = xf_mul(Xp, ld7(P.X_pj + i * 7));
    const V3 axis = ld3(P.axis + i * 3);
    const SV avj = ld6(s + Y.vj + i * 6);
    const SP qd = s + Y.qd;
    const SP S = s + Y.S;
    const SP aS = s + Y.aS;
    const SP aqd = s + Y.aqd;
    Xf aXsj = xf_zero();
    if (is_joint(P, type, JOINT_PRISMATIC)) {
        const SV aSk = ld6(aS + ds * 6) + avj * qd[ds];
        aqd[ds] += sv_dot(ld6(S + ds * 6), avj);
        aXsj.q += qrot_adj_q(Xsj.q, axis, aSk.v);   // S.v = R axis
    } else if (is_joint(P, type, JOINT_REVOLUTE)) {
        const SV aSk = ld6(aS + ds * 6) + avj * qd[ds];
        aqd[ds] += sv_dot(ld6(S + ds * 6), avj);
        xf_twist_adj_t(Xsj, SV{axis, v3zero()}, aSk, aXsj);
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k) {
            const SV aSk = ld6(aS + (ds + k) * 6) + avj * qd[ds + k];
            aqd[ds + k] += sv_dot(ld6(S + (ds + k) * 6), avj);
            V3 e = V3{k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f};
            xf_twist_adj_t(Xsj, SV{e, v3zero()}, aSk, aXsj);
        }
    } else if (is_joint(P, type, JOINT_FREE)) {
        add6(aqd + ds, avj);
    }
    // X_sj = X_p X_pj: this link's push to its parent through the joint frame does not depend on the recursion
    // below, so it is formed here (parallel over the links) and A4 only adds the X_sc = X_p X_l part per level
    Xf aXp = xf_zero();
    xf_mul_adj_a(Xp, ld7(P.X_pj + i * 7), aXsj, aXp);
    st7(s + Y.pX + i * 7, aXp);
}

DFX_HD void kin_adj_chain(const Pack& P, const Layout& Y, SP s, int i) {     // A4
    const int par = P.parent[i];
    Xf aXsc = ld7(s + Y.aXsc + i * 7);
    aXsc += ld7(s + Y.aXsm + i * 7);                                      // A1's share (through X_sm)
    for (int k = P.child_start[i]; k < P.child_start[i + 1]; ++k) aXsc += ld7(s + Y.pX + P.child_idx[k] * 7);
    st7(s + Y.aXsc + i * 7, aXsc);                       // total, consumed by A5
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    Xf aXp = xf_zero();
    xf_mul_adj_a(Xp, ld7(s + Y.Xl + i * 7), aXsc, aXp);                   // X_sc = X_p X_l
    aXp += ld7(s + Y.pX + i * 7);                                         // + the X_sj = X_p X_pj part from A3
    st7(s + Y.pX + i * 7, aXp);
}

DFX_HD void kin_adj_joint(const Pack& P, const Layout& Y, SP s, int i) {     // A5
    const int par = P.parent[i], type = P.type[i], qs = P.q_start[i];
    if (is_joint(P, type, JOINT_FIXED)) return;
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    const Xf Xpj = ld7(P.X_pj + i * 7);
    const SP q = s + Y.q;
    const SP aq = s + Y.aq;
    const Xf aXl = xf_mul_adj_b(Xp, ld7(s + Y.aXsc + i * 7));   // X_sc = X_p X_l
    const Xf aXjc = xf_mul_adj_b(Xpj, aXl);                      // X_l = X_pj X_jc
    const V3 axis = ld3(P.axis + i * 3);
    if (is_joint(P, type, JOINT_PRISMATIC)) aq[qs] += dot(axis, aXjc.p);
    else if (is_joint(P, type, JOINT_REVOLUTE)) aq[qs] += q_from_axis_angle_adj_angle(axis, q[qs], aXjc.q);
    else if (is_joint(P, type, JOINT_BALL)) add4(aq + qs, aXjc.q);
    else if (is_joint(P, type, JOINT_FREE)) { add3(aq + qs, aXjc.p); add4(aq + qs + 3, aXjc.q); }
}

template <class Grp>
DFX_HD void kin_adj(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    // all five passes run as CTA-wide (link, environment) tasks, link-major: uniform joint types per warp
    // (A1 already ran inside the rigid-body force adjoint)
    chain_rounds_up(P, s, g, [&](SP se, int i) { kin_adj_velocity(P, Y, se, i); }, true);
    g.cta_tasks(s, P.L, false, [&](SP se, int i) { kin_adj_motion(P, Y, se, i); });
    chain_rounds_up(P, s, g, [&](SP se, int i) { kin_adj_chain(P, Y, se, i); });
    g.cta_tasks(s, P.L, false, [&](SP se, int i) { kin_adj_joint(P, Y, se, i); });
}

#else
// The two leaf -> root recursions without a recursion.  Both are LINEAR accumulations towards the root:
//   * av, aa: a child's cotangent reaches the parent unchanged (v = v_p + v_j, a = a_p + v x v_j), so a link's total is the
//     sum over its subtree of the links' own terms;
//   * aX_sc: through X_sc[c] = X_sc[p] X_l[c] the translation part reaches the parent unchanged and the quaternion part as
//     r (x) conj(X_l[c].q), plus a term at p that depends on the child's translation total.  Writing every quaternion
//     cotangent w that lives at link j in the WORLD form u = w (x) conj(X_sc[j].q) turns the chain of right-multiplications
//     into the identity (X_sc[j].q = X_sc[i].q (x) q_(i->j) for i above j): the total at link i is
//     (sum of u over the subtree) (x) X_sc[i].q / |X_sc[i].q|^2  -- exact for non-unit quaternions too.
// Every pass is then parallel over ALL links with the subtree lists of the pack (O(L * depth) cheap additions instead of a
// dependent walk of heavy per-link steps by a handful of threads): four barriers, no idle warps.
//   B1  aa total (subtree sum) ; adjoint of a = a_p + v x v_j : av[i] += d/dv, vj slot <- d/dv_j
//   B2  av total (subtree sum) -> av_j ; A3 (S, qd, X_sj) ; pX[i] <- what this link sends to its ancestors through
//       X_sj = X_p X_pj: translation part and the world form (at the parent) of the quaternion part
//   B3  translation total of aX_sc (subtree sum) -> vj slot ; world forms: aXsc.q slot <- own quaternion part, aXsm.q slot <-
//       own + what the link sends to its ancestors (from B2, plus the term of X_sc[i] = X_p X_l through the translation total)
//       (own and sent-upwards parts are pre-added per link so that every subtree sum runs over ONE array)
//   B4  quaternion total (subtree sums), back to the link's frame ; A5
DFX_HD void kin_adj_acc(const Pack& P, const Layout& Y, SP s, int i) {        // B1
    SV aa = sv_zero();
    for (int k = P.sub_start[i]; k < P.sub_start[i + 1]; ++k) aa += ld6(s + Y.aa + P.sub_links[k] * 6);
    SV dv = sv_zero(), dvj = sv_zero();
    sv_cross_adj(ld6(s + Y.v + i * 6), ld6(s + Y.vj + i * 6), aa, dv, dvj);   // a = a_p + v x v_j
    add6(s + Y.av + i * 6, dv);      // (own slot: the other links read aa only in this pass)
    st6(s + Y.vj + i * 6, dvj);
}

DFX_HD Q4 q_conj(Q4 q) { return Q4{-q.x, -q.y, -q.z, q.w}; }

DFX_HD void kin_adj_motion(const Pack& P, const Layout& Y, SP s, int i) {    // B2
    const int par = P.parent[i], type = P.type[i], ds = P.qd_start[i];
    SV avj = ld6(s + Y.vj + i * 6);
    for (int k = P.sub_start[i]; k < P.sub_start[i + 1]; ++k) avj += ld6(s + Y.av + P.sub_links[k] * 6);   // v = v_p + v_j
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    const Xf Xpj = ld7(P.X_pj + i * 7);
    const Xf Xsj = xf_mul(Xp, Xpj);
    const V3 axis = ld3(P.axis + i * 3);
    const SP qd = s + Y.qd;
    const SP S = s + Y.S;
    const SP aS = s + Y.aS;
    const SP aqd = s + Y.aqd;
    Xf aXsj = xf_zero();
    if (is_joint(P, type, JOINT_PRISMATIC)) {
        const SV aSk = ld6(aS + ds * 6) + avj * qd[ds];
        aqd[ds] += sv_dot(ld6(S + ds * 6), avj);
        aXsj.q += qrot_adj_q(Xsj.q, axis, aSk.v);   // S.v = R axis
    } else if (is_joint(P, type, JOINT_REVOLUTE)) {
        const SV aSk = ld6(aS + ds * 6) + avj * qd[ds];
        aqd[ds] += sv_dot(ld6(S + ds * 6), avj);
        xf_twist_adj_t(Xsj, SV{axis, v3zero()}, aSk, aXsj);
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k) {
            const SV aSk = ld6(aS + (ds + k) * 6) + avj * qd[ds + k];
            aqd[ds + k] += sv_dot(ld6(S + (ds + k) * 6), avj);
            V3 e = V3{k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f};
            xf_twist_adj_t(Xsj, SV{e, v3zero()}, aSk, aXsj);
        }
    } else if (is_joint(P, type, JOINT_FREE)) {
        add6(aqd + ds, avj);
    }
    // X_sj = X_p X_pj: the cotangent of X_p, quaternion part in the world form at the parent
    Xf aXp = xf_zero();
    xf_mul_adj_a(Xp, Xpj, aXsj, aXp);
    // translation parts, pre-added so that B3 sums ONE array over the subtree: the link's own (aXsc slot, with A1's share from
    // the aXsm slot) and, for its ancestors, own + what it sends upwards (pX slot)
    const V3 own = ld3(s + Y.aXsc + i * 7) + ld3(s + Y.aXsm + i * 7);
    st3(s + Y.aXsc + i * 7, own);
    st3(s + Y.pX + i * 7, own + aXp.p);
    st4(s + Y.pX + i * 7 + 3, qmul(aXp.q, q_conj(Xp.q)));
}

DFX_HD void kin_adj_world(const Pack& P, const Layout& Y, SP s, int i) {     // B3
    const int par = P.parent[i];
    V3 ap = ld3(s + Y.aXsc + i * 7);                                      // own part (B2 added A1's share)
    for (int k = P.sub_start[i] + 1; k < P.sub_start[i + 1]; ++k)         // (the list starts with i itself)
        ap += ld3(s + Y.pX + P.sub_links[k] * 7);                         // descendants: own + what they sent upwards through X_sj
    const Q4 own = ld4(s + Y.aXsc + i * 7 + 3) + ld4(s + Y.aXsm + i * 7 + 3);
    const Q4 qi = ld4(s + Y.Xsc + i * 7 + 3);
    Q4 up = ld4(s + Y.pX + i * 7 + 3);
    if (par >= 0) {      // X_sc = X_p X_l: the translation total turns X_p.q
        const Q4 qp = ld4(s + Y.Xsc + par * 7 + 3);
        up += qmul(qrot_adj_q(qp, ld3(s + Y.Xl + i * 7), ap), q_conj(qp));
    }
    st3(s + Y.vj + i * 6, ap);                                  // (vj slot: B2 consumed av_j)
    const Q4 uo = qmul(own, q_conj(qi));
    st4(s + Y.aXsc + i * 7 + 3, uo);                            // (quaternion slots of this link: read by nobody else in this pass)
    st4(s + Y.aXsm + i * 7 + 3, uo + up);                       // for the ancestors: own + sent upwards, pre-added (one array in B4)
}

DFX_HD void kin_adj_joint(const Pack& P, const Layout& Y, SP s, int i) {     // B4 + A5
    const int par = P.parent[i], type = P.type[i], qs = P.q_start[i];
    if (is_joint(P, type, JOINT_FIXED)) return;
    Q4 u = ld4(s + Y.aXsc + i * 7 + 3);
    for (int k = P.sub_start[i] + 1; k < P.sub_start[i + 1]; ++k) u += ld4(s + Y.aXsm + P.sub_links[k] * 7 + 3);
    const Q4 qi = ld4(s + Y.Xsc + i * 7 + 3);
    const float n2 = qi.x * qi.x + qi.y * qi.y + qi.z * qi.z + qi.w * qi.w;
    const Xf aXsc = Xf{ld3(s + Y.vj + i * 6), qmul(u, qi) * (1.0f / n2)};     // total cotangent of X_sc[i]
    const Xf Xp = par >= 0 ? ld7(s + Y.Xsc + par * 7) : xf_ident();
    const Xf Xpj = ld7(P.X_pj + i * 7);
    const SP q = s + Y.q;
    const SP aq = s + Y.aq;
    const Xf aXl = xf_mul_adj_b(Xp, aXsc);                       // X_sc = X_p X_l
    const Xf aXjc = xf_mul_adj_b(Xpj, aXl);                      // X_l = X_pj X_jc
    const V3 axis = ld3(P.axis + i * 3);
    if (is_joint(P, type, JOINT_PRISMATIC)) aq[qs] += dot(axis, aXjc.p);
    else if (is_joint(P, type, JOINT_REVOLUTE)) aq[qs] += q_from_axis_angle_adj_angle(axis, q[qs], aXjc.q);
    else if (is_joint(P, type, JOINT_BALL)) add4(aq + qs, aXjc.q);
    else if (is_joint(P, type, JOINT_FREE)) { add3(aq + qs, aXjc.p); add4(aq + qs + 3, aXjc.q); }
}

template <class Grp>
DFX_HD void kin_adj(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    // four passes of CTA-wide (link, environment) tasks, link-major: uniform joint types per warp
    // (A1 already ran inside the rigid-body force adjoint)
    g.cta_tasks(s, P.L, true, [&](SP se, int i) { kin_adj_acc(P, Y, se, i); });
    g.cta_tasks(s, P.L, false, [&](SP se, int i) { kin_adj_motion(P, Y, se, i); });
    g.cta_tasks(s, P.L, false, [&](SP se, int i) { kin_adj_world(P, Y, se, i); });
    g.cta_tasks(s, P.L, false, [&](SP se, int i) { kin_adj_joint(P, Y, se, i); });
}
#endif

// =====================================================================================
// rigid-body forces per link:  f = I a + v x* I v - f_gravity, with I in closed form
// =====================================================================================
// World-frame spatial inertia of a link, kept factored exactly as the reference builds it
// (sim.py:1116-1134:  T^T I_m T  with  T = [[R^T, 0], [skew(-R^T c) R^T, R^T]]):
//     I_s = Rb I_body Rb^T ,  Rb = blockdiag(R, R),  I_body = [[I_c + m(u.u 1 - u u^T), m[u]x], [m[u]x^T, m 1]],  u = R^T c
// with R = R(q) the polynomial rotation of X_sm.q and c = X_sm.p.  R is NOT assumed orthogonal,
// so the derivative along |q| matches the reference's as well.
struct BodyInertia {
    M3 R;     // R(X_sm.q)
    M3 Ic;    // body-frame rotational inertia about the COM
    V3 u;     // R^T c
    float m;
};
DFX_HD BodyInertia body_inertia(const Pack& P, SP Xsm7, int i) {
    BodyInertia B;
    B.R = q_to_m3(ld4(Xsm7 + 3));
    B.Ic = ld9(P.I_c + i * 9);
    B.u = m3_tmul(B.R, ld3(Xsm7));
    B.m = P.mass[i];
    return B;
}
// y = I_s x
DFX_HD SV inertia_apply(const BodyInertia& B, SV x) {
    const V3 wb = m3_tmul(B.R, x.w), vb = m3_tmul(B.R, x.v);
    const V3 mu = (vb + cross(wb, B.u)) * B.m;
    const V3 top = m3_mul(B.Ic, wb) + cross(B.u, mu);
    return SV{m3_mul(B.R, top), m3_mul(B.R, mu)};
}
DFX_HD void outer_acc(M3& a, V3 x, V3 y) {  // a += x y^T
    a.m[0][0] += x.x * y.x; a.m[0][1] += x.x * y.y; a.m[0][2] += x.x * y.z;
    a.m[1][0] += x.y * y.x; a.m[1][1] += x.y * y.y; a.m[1][2] += x.y * y.z;
    a.m[2][0] += x.z * y.x; a.m[2][1] += x.z * y.y; a.m[2][2] += x.z * y.z;
}
// adjoint of y = I_s x given dL/dy = r: accumulates dL/dR, dL/du, dL/dx
DFX_HD void inertia_apply_adj(const BodyInertia& B, SV x, SV r, M3& aR, V3& au, SV& ax) {
    const V3 wb = m3_tmul(B.R, x.w), vb = m3_tmul(B.R, x.v);
    const V3 mu = (vb + cross(wb, B.u)) * B.m;
    const V3 top = m3_mul(B.Ic, wb) + cross(B.u, mu);
    // y.w = R top ; y.v = R mu
    const V3 atop = m3_tmul(B.R, r.w);
    V3 amu = m3_tmul(B.R, r.v);
    outer_acc(aR, r.w, top);
    outer_acc(aR, r.v, mu);
    // top = Ic wb + u x mu
    V3 awb = m3_tmul(B.Ic, atop);
    cross_adj(B.u, mu, atop, au, amu);
    // mu = m (vb + wb x u)
    const V3 a2 = amu * B.m;
    V3 avb = a2;
    cross_adj(wb, B.u, a2, awb, au);
    // wb = R^T x.w ; vb = R^T x.v
    ax.w += m3_mul(B.R, awb);
    ax.v += m3_mul(B.R, avb);
    outer_acc(aR, x.w, awb);
    outer_acc(aR, x.v, avb);
}

// kWrench: the link also feels the caller's external wrench (tau, F) at scratch offset xw (dfx_pack.h wrench_offset): a force F
// in world axes at its centre of mass and a pure torque tau -- F enters like extra gravity, f = fb - (c x (m g + F) + tau, m g + F)
template <bool kWrench = false>
DFX_HD void body_force_link_fwd(const Pack& P, const Layout& Y, SP s, int i, int xw = -1) {
    const BodyInertia B = body_inertia(P, s + Y.Xsm + i * 7, i);
    const V3 c = ld3(s + Y.Xsm + i * 7);
    const SV v = ld6(s + Y.v + i * 6), a = ld6(s + Y.a + i * 6);
    const SV Ia = inertia_apply(B, a);
    const SV h = inertia_apply(B, v);
    const SV fb = Ia + sv_cross_dual(v, h);
    if constexpr (kWrench) {
        const SV w = ld6(s + xw + i * 6);
        const V3 mgF = V3{P.gx, P.gy, P.gz} * B.m + w.v;
        st6(s + Y.f + i * 6, fb - SV{cross(c, mgF) + w.w, mgF});
    } else {
        (void)xw;
        const V3 mg = V3{P.gx, P.gy, P.gz} * B.m;
        const SV fg = SV{cross(c, mg), mg};
        st6(s + Y.f + i * 6, fb - fg);
    }
}

template <bool kWrench = false, class Grp>
DFX_HD void body_force_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g, int xw = -1) {
    DFX_FOR(i, P.L) body_force_link_fwd<kWrench>(P, Y, s, i, xw);
    g.sync();
}

// adjoint: af[i] (adjoint of body_f_s[i]) plus what crba_adj left in aR[i] / au[i] -> aXsm, av, aa.  kWrench: the wrench at
// scratch offset xw enters the c cotangent as m g + F does, and its own cotangent (-af.w, -af.v + c x af.w) is added to the
// accumulator at xw + 6 L -- one owner per link, the substeps in order: a deterministic sum
template <bool kWrench = false>
DFX_HD void body_force_link_adj(const Pack& P, const Layout& Y, SP s, int i, int xw = -1) {
    const SP Xsm7 = s + Y.Xsm + i * 7;
    const BodyInertia B = body_inertia(P, Xsm7, i);
    const V3 c = ld3(Xsm7);
    const SV v = ld6(s + Y.v + i * 6), a = ld6(s + Y.a + i * 6);
    const SV h = inertia_apply(B, v);
    const SV af = ld6(s + Y.af + i * 6);
    M3 aR = ld9(s + Y.aIbar + i * 12);
    V3 au = ld3(s + Y.aIbar + i * 12 + 9);
    V3 ac = v3zero();
    SV av = sv_zero(), aa = sv_zero(), ah = sv_zero();
    // f = fb - fg ; fg = (c x mg, mg)
    if constexpr (kWrench) {     // fg = (c x (mg + F) + tau, mg + F)
        const SV w = ld6(s + xw + i * 6);
        const V3 mgF = V3{P.gx, P.gy, P.gz} * B.m + w.v;
        ac += cross(mgF, -af.w);
        add6(s + xw + P.L * 6 + i * 6, SV{-af.w, cross(c, af.w) - af.v});
    } else {
        (void)xw;
        const V3 mg = V3{P.gx, P.gy, P.gz} * B.m;
        ac += cross(mg, -af.w);
    }
    // fb = Ia + v x* h
    sv_cross_dual_adj(v, h, af, av, ah);
    inertia_apply_adj(B, v, ah, aR, au, av);
    inertia_apply_adj(B, a, af, aR, au, aa);
    // u = R^T c
    ac += m3_mul(B.R, au);
    outer_acc(aR, c, au);
    add3(s + Y.aXsm + i * 7, ac);
    add4(s + Y.aXsm + i * 7 + 3, q_to_m3_adj(ld4(Xsm7 + 3), aR));
    add6(s + Y.av + i * 6, av);
    add6(s + Y.aa + i * 6, aa);
    kin_adj_local(P, Y, s, i);      // A1 of the kinematics adjoint, same link
}

template <bool kWrench = false, class Grp>
DFX_HD void body_force_adj(const Pack& P, const Layout& Y, SP s, const Grp& g, int xw = -1) {
    DFX_FOR(i, P.L) body_force_link_adj<kWrench>(P, Y, s, i, xw);
    g.sync();
}

// =====================================================================================
// Deterministic scatter-adds.  Shared memory on sm_90 has native atomics for 32-bit integers only: atomicAdd(float*)
// and the 64-bit integer atomicAdd both compile to ATOMS.CAST.SPIN compare-and-swap loops, which serialise badly when
// many lanes hit one body (152 muscles on 11 bodies: 69 % of all stall samples).  Integer adds are also associative,
// so a fixed-point sum is bit-reproducible whatever the order.  A contribution x is scaled by a power of two, rounded
// to an integer v and split sign-symmetrically into two words, v = hi * 2^21 + lo with |lo| < 2^21: both are added
// with fire-and-forget ATOMS.ADD (no carry between the words, so no returned value to wait for), and a contribution
// with |v| < 2^21 costs one atomic.  Capacity: up to 1024 contributions per accumulator, |sum| < 2^52, each
// contribution < 2^47 in magnitude.  Forward wrenches use the fixed scale 2^24 (resolution 6e-8 N, limit 8.4e6 N per
// contribution); cotangents use 2^27 / 2^floor(log2 max|af|) per environment and substep.  A contribution that is
// not representable (NaN, Inf, beyond the limit) raises the body's poison bit instead and the sum reads back NaN.
// =====================================================================================
constexpr int kFxLowBits = 21;
constexpr float kFxLimit = 140737488355328.0f;      // 2^47
constexpr float kFxForward = 16777216.0f;           // 2^24
constexpr float kFxForwardInv = 1.0f / 16777216.0f;
constexpr int kFxAdjointLog2 = 27;

// the low words can live in the (still all-zero) fp32 destination array itself; the high words have their own array.
// Split in fp32: x = w * scale (exact, power-of-two scale), h = rint(x / 2^21), l = x - h * 2^21 (exact: fma),
// so that hi * 2^21 + rint(l) == rint(x) with |rint(l)| <= 2^20, using 32-bit conversions only.
template <int N, class Grp>
DFX_HD void fx_scatter(SPi lo, SPi hi, SPu poison, int body, const float (&w)[N], float scale, const Grp& g) {
    bool ok = true;
#pragma unroll
    for (int c = 0; c < N; ++c) ok = ok && (fabsf(w[c] * scale) < kFxLimit);     // false for NaN / Inf / out of range
    if (!ok) { g.atomic_or(&poison[0], 1u << (body & 31)); return; }
    constexpr float kUnit = (float)(1 << kFxLowBits), kUnitInv = 1.0f / (float)(1 << kFxLowBits);
#pragma unroll
    for (int c = 0; c < N; ++c) {
        const float x = w[c] * scale;
        const float h = rintf(x * kUnitInv);
        const int l = (int)rintf(fmaf(h, -kUnit, x));
        const int hw = (int)h;
        if (l != 0) g.fx_add(&lo[c], l);
        if (hw != 0) g.fx_add(&hi[c], hw);
    }
}
// the fp32 value of an accumulator (two roundings at most; exact whenever |hi| < 2^24 and |lo| < 2^24)
DFX_HD float fx_value(int lo, int hi, float inv_scale) {
    return fmaf((float)hi, (float)(1 << kFxLowBits) * inv_scale, (float)lo * inv_scale);
}
// 2^(kFxAdjointLog2 - floor(log2 m)): the largest incoming cotangent maps to [2^27, 2^28); contact / muscle
// cotangents may be up to 2^20 times larger than that before they poison
DFX_HD float fx_pow2_scale(float m) {
    if (!(m > 0.0f)) return 1.0f;
    unsigned bits;
#if defined(__CUDA_ARCH__)
    bits = __float_as_uint(m);
#else
    memcpy(&bits, &m, 4);
#endif
    int field = (254 + kFxAdjointLog2) - (int)((bits >> 23) & 0xffu);
    field = field > 254 ? 254 : (field < 1 ? 1 : field);
    bits = (unsigned)field << 23;
    float r;
#if defined(__CUDA_ARCH__)
    r = __uint_as_float(bits);
#else
    memcpy(&r, &bits, 4);
#endif
    return r;
}

// =====================================================================================
// penalty ground contact (y-up plane), smooth Coulomb friction
// =====================================================================================
DFX_HD SV contact_point_fwd(const Pack& P, const Layout& Y, SP s, int k) {
    const int b = P.cbody[k];
    const Xf X = ld7(s + Y.Xsc + b * 7);
    const SV vs = ld6(s + Y.v + b * 6);
    const float ke = P.cmat[k * 4 + 0], kd = P.cmat[k * 4 + 1], kf = P.cmat[k * 4 + 2], mu = P.cmat[k * 4 + 3];
    V3 p = xf_point(X, ld3(P.cpoint + k * 3));
    p.y -= P.cdist[k];
    const V3 dpdt = vs.v + cross(vs.w, p);
    const float c = p.y;
    if (c >= 0.0f) return sv_zero();     // (callers compact with contact_penetrates() first)
    const float vn = dpdt.y;
    const V3 vt = V3{dpdt.x, 0.0f, dpdt.z};
    const float fn = c * ke;
    const float fd = fminf(vn, 0.0f) * kd * (0.0f - c);
    const float len = sqrtf(dot(vt, vt));
    const V3 nvt = len > 0.0f ? V3{vt.x / len, vt.y / len, vt.z / len} : v3zero();
    const float cap = fminf(kf * len, 0.0f - mu * c * ke);
    const V3 ft = nvt * cap;
    const V3 ftot = V3{ft.x, (fn + fd) + ft.y, ft.z};
    return SV{cross(p, ftot), ftot};
}

// signed height of contact point k above the ground plane (negative: penetrating); NaN counts as penetrating
// so that a non-finite state still reaches the poison bit
DFX_HD bool contact_penetrates(const Pack& P, const Layout& Y, SP s, int k) {
    const V3 p = xf_point(ld7(s + Y.Xsc + P.cbody[k] * 7), ld3(P.cpoint + k * 3));
    return !(p.y - P.cdist[k] >= 0.0f);
}

// contact + muscle wrenches are scattered into the fixed-point accumulators; wrench_collect() adds them to body_f_s.
// Typically a fifth of the points penetrate: the (point, environment) pairs that do are compacted over the whole
// CTA first, so the force model runs with full warps instead of a few lanes per group.
template <class Grp>
DFX_HD void contact_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if (!P.ground) return;
    g.cta_compact(s, P.C, [&](SP se, int k) { return contact_penetrates(P, Y, se, k); },
                  [&](SP se, int k) {
        const SV w = contact_point_fwd(P, Y, se, k);
        const SPi lo = sp_int(se + Y.fx);
        const float c6[6] = {w.w.x, w.w.y, w.w.z, w.v.x, w.v.y, w.v.z};
        fx_scatter(lo + P.cbody[k] * 6, lo + P.L * 6 + P.cbody[k] * 6, sp_uint(se + Y.cmask), P.cbody[k], c6, kFxForward, g);
    });
}

// rigid-body forces (dense: one item per link) and contact forces (sparse: compacted tasks) are independent: policies
// whose barriers are CTA-wide run them as ONE phase, the link items on some warps and the contact tasks on the rest
template <bool kWrench = false, class Grp>
DFX_HD void body_and_contact_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g, int xw = -1) {
    if (!Grp::kConcurrentItems || !P.ground) {
        body_force_fwd<kWrench>(P, Y, s, g, xw);
        contact_fwd(P, Y, s, g);
        return;
    }
    g.cta_compact_with(s, P.C, [&](SP se, int k) { return contact_penetrates(P, Y, se, k); },
                       [&](SP se, int k) {
        const SV w = contact_point_fwd(P, Y, se, k);
        const SPi lo = sp_int(se + Y.fx);
        const float c6[6] = {w.w.x, w.w.y, w.w.z, w.v.x, w.v.y, w.v.z};
        fx_scatter(lo + P.cbody[k] * 6, lo + P.L * 6 + P.cbody[k] * 6, sp_uint(se + Y.cmask), P.cbody[k], c6, kFxForward, g);
    }, P.L, [&](SP se, int i) { body_force_link_fwd<kWrench>(P, Y, se, i, xw); });
}

template <class Grp>
DFX_HD void wrench_collect(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if (!P.ground && P.M == 0) return;
    if (!Grp::kPathPasses || P.M > 0) g.sync();   // (tile kernels: the contact tasks ended with a CTA-wide barrier)
    const SPi lo = sp_int(s + Y.fx);
    const SPi hi = lo + P.L * 6;
    const SPu poison = sp_uint(s + Y.cmask);
    const unsigned bad = *poison;
    DFX_FOR(i, P.L) {          // one item per link: its six components are independent loads (ILP), one pass
        int l[6], h[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) { l[c] = lo[i * 6 + c]; h[c] = hi[i * 6 + c]; }
#pragma unroll
        for (int c = 0; c < 6; ++c)
            if ((l[c] | h[c]) != 0) { s[Y.f + i * 6 + c] += fx_value(l[c], h[c], kFxForwardInv); lo[i * 6 + c] = 0; hi[i * 6 + c] = 0; }
        if ((bad >> (i & 31)) & 1u) {
#pragma unroll
            for (int c = 0; c < 6; ++c) s[Y.f + i * 6 + c] = nanf("");
        }
    }
    g.sync();                  // (barriers stay unconditional: `bad` differs between the environments of a tile)
    if (g.lane == 0) *poison = 0u;
}

// adjoint for one contact: cotangent r = af[body]; accumulates into aXsc[body], av[body] (only penetrating contacts do
// any work): muscle models through the fixed-point scatter, contact-only models with plain adds by the body's owner.
// Either way the sums do not depend on thread timing, so the gradient is as bit-reproducible as the forward pass.
template <class Grp>
DFX_HD void contact_point_adj(const Pack& P, const Layout& Y, SP s, int k, float scale, const Grp& g) {
    const int b = P.cbody[k];
    const Xf X = ld7(s + Y.Xsc + b * 7);
    const SV vs = ld6(s + Y.v + b * 6);
    const V3 pt = ld3(P.cpoint + k * 3);
    V3 p = xf_point(X, pt);
    p.y -= P.cdist[k];
    const float c = p.y;
    if (c >= 0.0f) return;
    const float ke = P.cmat[k * 4 + 0], kd = P.cmat[k * 4 + 1], kf = P.cmat[k * 4 + 2], mu = P.cmat[k * 4 + 3];
    const V3 dpdt = vs.v + cross(vs.w, p);
    const SV r = ld6(s + Y.af + b * 6);
    const float vn = dpdt.y;
    const V3 vt = V3{dpdt.x, 0.0f, dpdt.z};
    const float fn = c * ke;
    const float mn = fminf(vn, 0.0f);
    const float fd = mn * kd * (0.0f - c);
    const float len = sqrtf(dot(vt, vt));
    const V3 nvt = len > 0.0f ? V3{vt.x / len, vt.y / len, vt.z / len} : v3zero();
    const float A = kf * len, Bc = 0.0f - mu * c * ke;
    const float cap = fminf(A, Bc);
    const V3 ft = nvt * cap;
    const V3 ftot = V3{ft.x, (fn + fd) + ft.y, ft.z};
    // t = p x ftot
    V3 ap = v3zero(), aftot = r.v;
    cross_adj(p, ftot, r.w, ap, aftot);
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
    V3 adpdt = avt;
    avn -= avt.y;
    adpdt.y += avn;
    ap.y += ac;
    // dpdt = v + w x p
    V3 aw = v3zero();
    cross_adj(vs.w, p, adpdt, aw, ap);
    // p = X.p + R(X.q) pt - n d
    const Q4 aq = qrot_adj_q(X.q, pt, ap);
    const SPu poison = sp_uint(s + Y.cmask);
    const float c7[7] = {ap.x, ap.y, ap.z, aq.x, aq.y, aq.z, aq.w};
    const float c6[6] = {aw.x, aw.y, aw.z, adpdt.x, adpdt.y, adpdt.z};
    if (P.M > 0) {
        // muscle models scatter everything in fixed point: low words accumulate in aXsc / av themselves (both are
        // still all-zero in this phase), high words in fxH; adj_collect() converts back
        const SPi hi = sp_int(s + Y.fxH);
        fx_scatter(sp_int(s + Y.aXsc) + b * 7, hi + b * 7, poison, b, c7, scale, g);
        fx_scatter(sp_int(s + Y.av) + b * 6, hi + P.L * 7 + b * 6, poison, b, c6, scale, g);
    } else {
        // contact-only models: called by the item that owns body b (substep_adj), in the pack's contact order --
        // one writer, a fixed order: plain adds, and the gradient is bit-reproducible
        const SP ax = s + Y.aXsc + b * 7;
        const SP avp = s + Y.av + b * 6;
#pragma unroll
        for (int c = 0; c < 7; ++c) ax[c] += c7[c];
#pragma unroll
        for (int c = 0; c < 6; ++c) avp[c] += c6[c];
    }
}

// power-of-two fixed-point scale of the cotangent scatter of this environment and substep, from max|af|
template <class Grp>
DFX_HD float adj_scatter_scale(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    float m = 0.0f;
    DFX_FOR(i, P.L * 6) { const float v = fabsf(s[Y.af + i]); m = (v > m) ? v : m; }   // NaN never wins: the poison bit handles it
    const float scale = fx_pow2_scale(g.group_max(m, s + Y.fxs));
    if (g.lane == 0) s[Y.fxs] = scale;       // CTA-wide contact tasks of this environment read it from here
    return scale;
}

template <class Grp>
DFX_HD void adj_collect(const Pack& P, const Layout& Y, SP s, float scale, const Grp& g) {
    g.sync();
    const SPu poison = sp_uint(s + Y.cmask);
    const SPi hi = sp_int(s + Y.fxH);
    const unsigned bad = *poison;
    const float inv = 1.0f / scale;
    const SP dst = s + Y.aXsc;                       // aXsc (L,7) and av (L,6) are adjacent
    DFX_FOR(it, P.L * 13) {
        const int l = sp_int(dst)[it];
        const int h = hi[it];
        if ((l | h) != 0) { dst[it] = fx_value(l, h, inv); hi[it] = 0; }
        const int body = (it < P.L * 7) ? it / 7 : (it - P.L * 7) / 6;
        if ((bad >> (body & 31)) & 1u) dst[it] = nanf("");
    }
    g.sync();
    if (g.lane == 0) *poison = 0u;
}

template <class Grp>
DFX_HD void contact_adj(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if (!P.ground) return;
    g.cta_compact(s, P.C, [&](SP se, int k) { return contact_penetrates(P, Y, se, k); },
                  [&](SP se, int k) { contact_point_adj(P, Y, se, k, se[Y.fxs], g); });
}

// =====================================================================================
// muscles: straight-line way-point segments pulling two links together
// =====================================================================================
template <class Grp>
DFX_HD void muscle_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if (P.M == 0) return;
    const SPi lo = sp_int(s + Y.fx);
    const SPi hi = lo + P.L * 6;
    const SPu poison = sp_uint(s + Y.cmask);
    DFX_FOR(gi, P.MG) {        // one item = a group of muscles whose active segments connect the same links
        const int mb = P.mgrp_start[gi], me = P.mgrp_start[gi + 1];
        const int m0 = P.morder[mb];
        const int nseg = P.aseg_start[m0 + 1] - P.aseg_start[m0];
        for (int j = 0; j < nseg; ++j) {
            const int i0 = P.aseg_way[P.aseg_start[m0] + j];
            const int l0 = P.mlinks[i0], l1 = P.mlinks[i0 + 1];
            const Xf X0 = ld7(s + Y.Xsc + l0 * 7), X1 = ld7(s + Y.Xsc + l1 * 7);
            V3 fs = v3zero(), t0s = v3zero(), t1s = v3zero();
            for (int k = mb; k < me; ++k) {
                const int m = P.morder[k];
                const int i = P.aseg_way[P.aseg_start[m] + j];
                const V3 p0 = xf_point(X0, ld3(P.mpoints + i * 3));
                const V3 p1 = xf_point(X1, ld3(P.mpoints + (i + 1) * 3));
                const V3 d = p1 - p0;
                const float len = sqrtf(dot(d, d));
                const V3 n = len > 0.0f ? V3{d.x / len, d.y / len, d.z / len} : v3zero();
                const V3 f = n * s[Y.musc + m];
                fs += f;
                t0s += cross(p0, f);
                t1s += cross(p1, f);
            }
            const float w0[6] = {-t0s.x, -t0s.y, -t0s.z, -fs.x, -fs.y, -fs.z};
            const float w1[6] = {t1s.x, t1s.y, t1s.z, fs.x, fs.y, fs.z};
            fx_scatter(lo + l0 * 6, hi + l0 * 6, poison, l0, w0, kFxForward, g);
            fx_scatter(lo + l1 * 6, hi + l1 * 6, poison, l1, w1, kFxForward, g);
        }
    }
}

template <class Grp>
DFX_HD void muscle_adj(const Pack& P, const Layout& Y, SP s, float scale, const Grp& g) {
    if (P.M == 0) return;
    const SPi lo = sp_int(s + Y.aXsc);   // still all-zero in this phase: doubles as the low words
    const SPi hi = sp_int(s + Y.fxH);
    const SPu poison = sp_uint(s + Y.cmask);
    DFX_FOR(gi, P.MG) {
        const int mb = P.mgrp_start[gi], me = P.mgrp_start[gi + 1];
        const int m0 = P.morder[mb];
        const int nseg = P.aseg_start[m0 + 1] - P.aseg_start[m0];
        for (int j = 0; j < nseg; ++j) {
            const int i0 = P.aseg_way[P.aseg_start[m0] + j];
            const int l0 = P.mlinks[i0], l1 = P.mlinks[i0 + 1];
            const Xf X0 = ld7(s + Y.Xsc + l0 * 7), X1 = ld7(s + Y.Xsc + l1 * 7);
            const SV c0 = ld6(s + Y.af + l0 * 6), c1 = ld6(s + Y.af + l1 * 6);
            V3 ap0s = v3zero(), ap1s = v3zero();
            Q4 aq0s = qzero(), aq1s = qzero();
            for (int k = mb; k < me; ++k) {
                const int m = P.morder[k];
                const int i = P.aseg_way[P.aseg_start[m] + j];
                const float act = s[Y.musc + m];
                const V3 r0 = ld3(P.mpoints + i * 3), r1 = ld3(P.mpoints + (i + 1) * 3);
                const V3 p0 = xf_point(X0, r0), p1 = xf_point(X1, r1);
                const V3 d = p1 - p0;
                const float len = sqrtf(dot(d, d));
                const V3 n = len > 0.0f ? V3{d.x / len, d.y / len, d.z / len} : v3zero();
                const V3 f = n * act;
                // L = -c0.(p0 x f, f) + c1.(p1 x f, f)
                const V3 af = c1.v - c0.v + cross(c1.w, p1) - cross(c0.w, p0);
                V3 ap0 = -cross(f, c0.w);
                V3 ap1 = cross(f, c1.w);
                s[Y.amusc + m] += dot(n, af);
                const V3 an = af * act;
                if (len > 0.0f) {
                    const V3 ad = (an - n * dot(n, an)) * (1.0f / len);
                    ap1 += ad;
                    ap0 -= ad;
                }
                ap0s += ap0; ap1s += ap1;
                aq0s += qrot_adj_q(X0.q, r0, ap0);
                aq1s += qrot_adj_q(X1.q, r1, ap1);
            }
            const float g0[7] = {ap0s.x, ap0s.y, ap0s.z, aq0s.x, aq0s.y, aq0s.z, aq0s.w};
            const float g1[7] = {ap1s.x, ap1s.y, ap1s.z, aq1s.x, aq1s.y, aq1s.z, aq1s.w};
            fx_scatter(lo + l0 * 7, hi + l0 * 7, poison, l0, g0, scale, g);
            fx_scatter(lo + l1 * 7, hi + l1 * 7, poison, l1, g1, scale, g);
        }
    }
}

// =====================================================================================
// joint torques: leaf -> root wrench accumulation and projection on the motion subspace
// =====================================================================================
// per link, in one pass: f_tot[i] = sum of f over the subtree of i (the pack lists it, i first), then the projection
// on the joint axes plus PD targets and limits.  (A leaf->root recursion f_tot[i] = f[i] + sum f_tot[children]
// would need a barrier per tree level; the flat sum associates differently, within rounding.)
DFX_HD SV tau_subtree_force(const Pack& P, const Layout& Y, SP s, int i) {
    SV ft = sv_zero();
    for (int k = P.sub_start[i + 1] - 1; k >= P.sub_start[i]; --k) ft += ld6(s + Y.f + P.sub_links[k] * 6);
    st6(s + Y.ft + i * 6, ft);
    return ft;
}

DFX_HD void tau_accum_fwd(const Pack& P, const Layout& Y, SP s, int i) {
    SV ft = sv_zero();
    for (int k = P.child_start[i + 1] - 1; k >= P.child_start[i]; --k) ft += ld6(s + Y.ft + P.child_idx[k] * 6);
    st6(s + Y.ft + i * 6, ld6(s + Y.f + i * 6) + ft);
}

template <bool SUBTREE>
DFX_HD void tau_project_fwd(const Pack& P, const Layout& Y, SP s, int i) {
    const int type = P.type[i], qs = P.q_start[i], ds = P.qd_start[i];
    const SV f = SUBTREE ? tau_subtree_force(P, Y, s, i) : ld6(s + Y.ft + i * 6);
    const SP q = s + Y.q;
    const SP qd = s + Y.qd;
    const SP S = s + Y.S;
    const SP tau = s + Y.tau;
    const float tke = P.target_ke[i], tkd = P.target_kd[i];
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) {
        const float qq = q[qs], qdv = qd[ds];
        const float lower = P.limit_lower[qs], upper = P.limit_upper[qs];
        float limit_f = 0.0f;
        if (qq < lower) limit_f = P.limit_ke[i] * (lower - qq);
        if (qq > upper) limit_f = P.limit_ke[i] * (upper - qq);
        const float damping_f = (0.0f - P.limit_kd[i]) * qdv;
        tau[ds] = 0.0f - sv_dot(ld6(S + ds * 6), f) - tke * (qq - P.target[qs]) - tkd * qdv + s[Y.act + ds] + limit_f + damping_f;
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k)
            tau[ds + k] = 0.0f - sv_dot(ld6(S + (ds + k) * 6), f) - qd[ds + k] * tkd - q[qs + k] * tke;
    } else if (is_joint(P, type, JOINT_FREE)) {
        tau[ds + 0] = 0.0f - f.w.x; tau[ds + 1] = 0.0f - f.w.y; tau[ds + 2] = 0.0f - f.w.z;
        tau[ds + 3] = 0.0f - f.v.x; tau[ds + 4] = 0.0f - f.v.y; tau[ds + 5] = 0.0f - f.v.z;
    }
}

template <class Grp>
DFX_HD void tau_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    if constexpr (Grp::kPathPasses) {
        DFX_FOR(i, P.L) tau_project_fwd<true>(P, Y, s, i);
        g.sync();
    } else {
        chain_rounds_up(P, s, g, [&](SP se, int i) { tau_accum_fwd(P, Y, se, i); }, true);
        DFX_FOR(i, P.L) tau_project_fwd<false>(P, Y, s, i);
        g.sync();
    }
}

// adjoint: `atau` (D) in; af[] becomes the adjoint of body_f_s; aS, aq, aqd, aact accumulate.
// T2' (parallel): per-link contribution to a(f_tot) + aS, aq, aqd, aact ;  T1' (root->leaf, thin): af[i] += af[parent]
DFX_HD void tau_project_adj(const Pack& P, const Layout& Y, SP s, SP atau, int i) {
    const int type = P.type[i], qs = P.q_start[i], ds = P.qd_start[i];
    SV af = sv_zero();
    const SV f = ld6(s + Y.ft + i * 6);
    const SP q = s + Y.q;
    const SP S = s + Y.S;
    const SP aS = s + Y.aS;
    const SP aq = s + Y.aq;
    const SP aqd = s + Y.aqd;
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) {
        const float at = atau[ds];
        add6(aS + ds * 6, f * (-at));
        af += ld6(S + ds * 6) * (-at);
        const float qq = q[qs];
        float dlim = 0.0f;
        if (qq < P.limit_lower[qs]) dlim = -P.limit_ke[i];
        if (qq > P.limit_upper[qs]) dlim = -P.limit_ke[i];
        aq[qs] += (dlim - P.target_ke[i]) * at;
        aqd[ds] += (0.0f - P.target_kd[i] - P.limit_kd[i]) * at;
        s[Y.aact + ds] += at;
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k) {
            const float at = atau[ds + k];
            add6(aS + (ds + k) * 6, f * (-at));
            af += ld6(S + (ds + k) * 6) * (-at);
            aqd[ds + k] += -P.target_kd[i] * at;
            aq[qs + k] += -P.target_ke[i] * at;
        }
    } else if (is_joint(P, type, JOINT_FREE)) {
        for (int k = 0; k < 6; ++k) add6(aS + (ds + k) * 6, f * (-atau[ds + k]));
        af += SV{V3{-atau[ds], -atau[ds + 1], -atau[ds + 2]}, V3{-atau[ds + 3], -atau[ds + 4], -atau[ds + 5]}};
    }
    st6(s + Y.pX + i * 7, af);      // (direct part, in the idle pX slot: tau_adj sums it along the root paths into af)
}

// the direct part of a(f_tot[j]) alone: what tau_project_adj() stages in pX, recomputed by every link below j (kFusedPhases)
DFX_HD SV tau_direct_af(const Pack& P, const Layout& Y, SP s, SP atau, int j) {
    const int type = P.type[j], ds = P.qd_start[j];
    const SP S = s + Y.S;
    SV af = sv_zero();
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) {
        af += ld6(S + ds * 6) * (-atau[ds]);
    } else if (is_joint(P, type, JOINT_BALL)) {
        for (int k = 0; k < 3; ++k) af += ld6(S + (ds + k) * 6) * (-atau[ds + k]);
    } else if (is_joint(P, type, JOINT_FREE)) {
        af += SV{V3{-atau[ds], -atau[ds + 1], -atau[ds + 2]}, V3{-atau[ds + 3], -atau[ds + 4], -atau[ds + 5]}};
    }
    return af;
}

template <class Grp>
DFX_HD void tau_adj(const Pack& P, const Layout& Y, SP s, SP atau, const Grp& g) {
    const int atau_off = (int)(atau - s);   // (element offset inside the scratch)
    if constexpr (Grp::kFusedPhases) {
        // ONE pass: a link's own projection adjoint (aS, aq, aqd, aact) and af[i] = the direct cotangents summed along its root
        // path, each ancestor's recomputed on the fly (one scaled load of S per dof) -- same values, same root-first order
        g.cta_tasks(s, P.L, true, [&](SP se, int i) {
            SV acc = sv_zero();
            bool first = true;
            for_path_root_first(P, i, false, [&](int j) {
                const SV x = tau_direct_af(P, Y, se, se + atau_off, j);
                acc = first ? x : acc + x;
                first = false;
            });
            tau_project_adj(P, Y, se, se + atau_off, i);              // (leaves the link's own direct part in pX[i])
            const SV own = ld6(se + Y.pX + i * 7);
            st6(se + Y.af + i * 6, first ? own : acc + own);
        });
        return;
    }
    g.cta_tasks(s, P.L, true, [&](SP se, int i) { tau_project_adj(P, Y, se, se + atau_off, i); });
    // T1': af[i] = af_direct[i] + af[parent], root -> leaves, as PATH SUMS: tau_project_adj left the direct cotangents in the
    // (idle) pX slot; every link adds them along its own root path in root-first order (the same association as the
    // recursion, so the same bits) -- two barriers with all links busy instead of a serial walk down the chains
    g.cta_tasks(s, P.L, false, [&](SP se, int i) {
        SV acc = sv_zero();
        bool first = true;
        for_path_root_first(P, i, true, [&](int j) {
            const SV x = ld6(se + Y.pX + j * 7);
            acc = first ? x : acc + x;
            first = false;
        });
        st6(se + Y.af + i * 6, acc);
    });
}

// =====================================================================================
// joint-space inertia by composite rigid bodies, Cholesky, explicit inverse
// =====================================================================================
DFX_HD int sym_idx(int i, int j) {  // packed upper triangle of a symmetric 6x6, i <= j
    return i * 6 - (i * (i - 1)) / 2 + (j - i);
}
// the 21 unique entries (packed upper triangle) of  I_s = Rb I_body Rb^T
DFX_HD void inertia_sym21(const BodyInertia& B, SP o) {
    const float uu = dot(B.u, B.u);
    const float uv[3] = {B.u.x, B.u.y, B.u.z};
    M3 TLb, K;  // body-frame top-left block and [u]x
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) TLb.m[i][j] = B.Ic.m[i][j] + B.m * ((i == j ? uu : 0.0f) - uv[i] * uv[j]);
    K.m[0][0] = 0.f;    K.m[0][1] = -B.u.z; K.m[0][2] = B.u.y;
    K.m[1][0] = B.u.z;  K.m[1][1] = 0.f;    K.m[1][2] = -B.u.x;
    K.m[2][0] = -B.u.y; K.m[2][1] = B.u.x;  K.m[2][2] = 0.f;
    const M3 TL = m3_mmt(m3_mm(B.R, TLb), B.R);
    const M3 TR = m3_mmt(m3_mm(B.R, K), B.R);
    const M3 BR = m3_mmt(B.R, B.R);
    for (int i = 0; i < 3; ++i)
        for (int j = i; j < 3; ++j) {
            o[sym_idx(i, j)] = 0.5f * (TL.m[i][j] + TL.m[j][i]);
            o[sym_idx(3 + i, 3 + j)] = B.m * 0.5f * (BR.m[i][j] + BR.m[j][i]);
        }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) o[sym_idx(i, 3 + j)] = B.m * TR.m[i][j];
}
DFX_HD SV sym21_apply(SP o, SV x) {
    const float xv[6] = {x.w.x, x.w.y, x.w.z, x.v.x, x.v.y, x.v.z};
    float y[6];
    for (int i = 0; i < 6; ++i) {
        float acc = 0.0f;
        for (int j = 0; j < 6; ++j) acc += o[i <= j ? sym_idx(i, j) : sym_idx(j, i)] * xv[j];
        y[i] = acc;
    }
    return SV{V3{y[0], y[1], y[2]}, V3{y[3], y[4], y[5]}};
}

template <class Grp>
DFX_HD void crba_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    const int D = P.D, L = P.L;
    const SP Ic = s + Y.Icmp;
    const SP F = s + Y.Icmp + L * 21;
    const SP H = s + Y.A;
    const SP Lm = s + Y.Lm;
    DFX_FOR(i, L) inertia_sym21(body_inertia(P, s + Y.Xsm + i * 7, i), Ic + i * 21);
    DFX_FOR(e, D * D) { H[e] = 0.0f; Lm[e] = 0.0f; }
    g.sync();
    // composite inertias, leaves -> root
    for (int lev = P.nlev - 1; lev >= 0; --lev) {
        const int b = P.level_start[lev], e = P.level_start[lev + 1];
        for (int it = g.lane; it < (e - b) * 21; it += Grp::G) {
            const int i = P.level_links[b + it / 21], c = it % 21;
            float acc = Ic[i * 21 + c];
            for (int k = P.child_start[i]; k < P.child_start[i + 1]; ++k) acc += Ic[P.child_idx[k] * 21 + c];
            Ic[i * 21 + c] = acc;
        }
        g.sync();
    }
    DFX_FOR(d, D) st6(F + d * 6, sym21_apply(Ic + P.dof_link[d] * 21, ld6(s + Y.S + d * 6)));
    g.sync();
    DFX_FOR(d, D) {
        const int l = P.dof_link[d];
        const SV Fd = ld6(F + d * 6);
        for (int k = P.anc_start[l]; k < P.anc_start[l + 1]; ++k) {
            const int j = P.anc_dofs[k];
            if (j > d) break;
            const float h = sv_dot(Fd, ld6(s + Y.S + j * 6));
            H[d * D + j] = h;
            H[j * D + d] = h;
        }
    }
    g.sync();
}

// Cholesky  L L^T = H + diag(armature), then A <- (L L^T)^-1 column-wise.
// The factorisation runs TWO columns per barrier: every thread forms the 2 x 2 diagonal block (L[j][j], L[j+1][j], L[j+1][j+1])
// itself -- three short dot products, independent of each other -- and its rows' entries of both columns from ONE pass over the
// row (the column-(j+1) entry needs the thread's own column-j entry, still in a register).  Every entry is the same expression,
// accumulated in the same order, as in the column-by-column form (kept below for the host-emulation A/B,
// tests/test_emu_golden.py): bit-identical factors with half the barriers and two independent FMA chains per thread.
#ifndef DFX_CHOL_UNBLOCKED
#define DFX_CHOL_UNBLOCKED 0
#endif
template <class Grp>
DFX_HD void chol_inverse(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    const int D = P.D;
    const SP A = s + Y.A;
    const SP Lm = s + Y.Lm;
#if DFX_CHOL_UNBLOCKED
    for (int j = 0; j < D; ++j) {
        float sj = A[j * D + j] + P.armature[j];
#pragma unroll 4
        for (int k = 0; k < j; ++k) { const float r = Lm[j * D + k]; sj -= r * r; }   // (unrolled: the loads pipeline)
        const float ljj = sqrtf(sj);
        const float inv = 1.0f / ljj;
        for (int i = j + 1 + g.lane; i < D; i += Grp::G) {
            float si = A[i * D + j];
#pragma unroll 4
            for (int k = 0; k < j; ++k) si -= Lm[i * D + k] * Lm[j * D + k];
            Lm[i * D + j] = si * inv;
        }
        if (g.lane == j % Grp::G) Lm[j * D + j] = ljj;
        g.sync();
    }
#else
    for (int j = 0; j < D; j += 2) {
        const bool two = j + 1 < D;
        const int j1 = two ? j + 1 : j;          // (a lone last column reads its own row twice; the second set of results is dropped)
        float s00 = A[j * D + j] + P.armature[j];
        float s10 = A[j1 * D + j];
        float s11 = A[j1 * D + j1] + P.armature[j1];
#pragma unroll 4
        for (int k = 0; k < j; ++k) {
            const float r0 = Lm[j * D + k], r1 = Lm[j1 * D + k];
            s00 -= r0 * r0;
            s10 -= r1 * r0;
            s11 -= r1 * r1;
        }
        const float l00 = sqrtf(s00);
        const float inv0 = 1.0f / l00;
        const float l10 = s10 * inv0;
        s11 -= l10 * l10;
        const float l11 = sqrtf(s11);
        const float inv1 = 1.0f / l11;
        for (int i = j + 2 + g.lane; i < D; i += Grp::G) {
            float si0 = A[i * D + j], si1 = A[i * D + j1];
#pragma unroll 4
            for (int k = 0; k < j; ++k) {
                const float lik = Lm[i * D + k];
                si0 -= lik * Lm[j * D + k];
                si1 -= lik * Lm[j1 * D + k];
            }
            const float li0 = si0 * inv0;
            Lm[i * D + j] = li0;
            if (two) { si1 -= li0 * l10; Lm[i * D + j1] = si1 * inv1; }
        }
        if (g.lane == j % Grp::G) {
            Lm[j * D + j] = l00;
            if (two) { Lm[j1 * D + j] = l10; Lm[j1 * D + j1] = l11; }
        }
        g.sync();
    }
#endif
    DFX_FOR(c, D) {
        // L y = e_c  (y_i = 0 for i < c)
        for (int i = 0; i < D; ++i) {
            float acc = (i == c) ? 1.0f : 0.0f;
#pragma unroll 4
            for (int k = c; k < i; ++k) acc -= Lm[i * D + k] * A[k * D + c];
            A[i * D + c] = (i < c) ? 0.0f : acc / Lm[i * D + i];
        }
        // L^T x = y
        for (int i = D - 1; i >= 0; --i) {
            float acc = A[i * D + c];
#pragma unroll 4
            for (int k = i + 1; k < D; ++k) acc -= Lm[k * D + i] * A[k * D + c];
            A[i * D + c] = acc / Lm[i * D + i];
        }
    }
    g.sync();
}

// q'' = H^-1 tau
template <class Grp>
DFX_HD void solve_fwd(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    const int D = P.D;
#if defined(DFX_EMU_SWEEPS) && !defined(__CUDACC__)
    // Host-emulation A/B only (tests/test_emu_golden.py::test_explicit_inverse_is_not_the_parity_floor): the reference's two
    // triangular sweeps with the Cholesky factor (matnn.h:188-230) instead of the H^-1 mat-vec.  Needs a layout that keeps Lm.
    if (g.lane == 0) {
        float y[64];
        for (int i = 0; i < D; ++i) {
            float acc = s[Y.tau + i];
            for (int k = 0; k < i; ++k) acc -= s[Y.Lm + i * D + k] * y[k];
            y[i] = acc / s[Y.Lm + i * D + i];
        }
        for (int i = D - 1; i >= 0; --i) {
            float acc = y[i];
            for (int k = i + 1; k < D; ++k) acc -= s[Y.Lm + k * D + i] * s[Y.qdd + k];
            s[Y.qdd + i] = acc / s[Y.Lm + i * D + i];
        }
    }
    g.sync();
    return;
#endif
    DFX_FOR(i, D) {
        float acc = 0.0f;
        for (int j = 0; j < D; ++j) acc += s[Y.A + i * D + j] * s[Y.tau + j];
        s[Y.qdd + i] = acc;
    }
    g.pre_store();         // the row's intermediates and q'' leave for the tape right after this barrier
    g.sync();
}
// the cotangent of H is kept SYMMETRISED and packed (upper triangle, row-major): only aH + aH^T enters crba_adj, because
// every use of H there is through a symmetric bilinear form.  Hs[i][i] = aH[i][i], Hs[i][j] = aH[i][j] + aH[j][i] (i < j).
DFX_HD int symD_idx(int D, int i, int j) { return i * D - (i * (i - 1)) / 2 + (j - i); }   // i <= j

// atau = H^-1 aqdd (written over tau);  Hs -= sym(atau (x) qdd)   (Hs lives in the Lm slot during backward)
template <class Grp>
DFX_HD void solve_adj(const Pack& P, const Layout& Y, SP s, HinvView hv, const Grp& g) {
    const int D = P.D;
    if (hv.g) {
        DFX_FOR(i, D) {
            // (rows come from L2: keep many loads in flight -- with 4 at a time the 27 loads of a Humanoid row cost 7 round trips)
            const float* row = hv.g + (long long)i * D * hv.hs;
            float acc = 0.0f;
#pragma unroll 1
            for (int j0 = 0; j0 < D; j0 += 14) {
                float h[14];
#pragma unroll
                for (int k = 0; k < 14; ++k) h[k] = (j0 + k < D) ? row[(long long)(j0 + k) * hv.hs] : 0.0f;
#pragma unroll
                for (int k = 0; k < 14; ++k) if (j0 + k < D) acc += h[k] * s[Y.aqdd + j0 + k];
            }
            s[Y.tau + i] = acc;
        }
    } else {
        DFX_FOR(i, D) {
            float acc = 0.0f;
            for (int j = 0; j < D; ++j) acc += s[Y.A + i * D + j] * s[Y.aqdd + j];
            s[Y.tau + i] = acc;
        }
    }
    g.sync();
    DFX_FOR(i, D) {                 // row i of the packed triangle: entries (i, i..D-1)
        const float ti = s[Y.tau + i], qi = s[Y.qdd + i];
        const SP row = s + Y.Lm + symD_idx(D, i, i);
        row[0] -= ti * qi;
        for (int j = i + 1; j < D; ++j) row[j - i] -= ti * s[Y.qdd + j] + s[Y.tau + j] * qi;
    }
    // (no barrier here: the caller's next one -- substep_adj waits for the bulk of the tape row -- comes before any reader of Hs, tau)
}

#ifndef DFX_CRBA_ADJ_DIRECT
#define DFX_CRBA_ADJ_DIRECT 0     // 1: the direct double sums (A/B builds); 0: composite inertias + per-link moment matrices
#endif
#if DFX_CRBA_ADJ_DIRECT
// adjoint of H(S, I) w.r.t. S (-> aS) and the body inertias (-> aIbar, aXsm.p), from the symmetrised cotangent Hs
template <class Grp>
DFX_HD void crba_adj(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    const int D = P.D, L = P.L;
    const SP Hs = s + Y.Lm;
    // body inertia parameters: for each link l and each ancestor dof a:  z = sum_b c_ab S_b with c_aa = Hs_aa,
    // c_ab = Hs_ab / 2 ; cotangent S_a on  I_l z   (sum_ab aH_ab Phi(S_a, S_b) with Phi symmetric)
    DFX_FOR(l, L) {
        const BodyInertia B = body_inertia(P, s + Y.Xsm + l * 7, l);
        M3 aR = m3_zero();
        V3 au = v3zero();
        SV dummy = sv_zero();
        for (int ka = P.anc_start[l]; ka < P.anc_start[l + 1]; ++ka) {
            const int a = P.anc_dofs[ka];
            SV z = sv_zero();
            for (int kb = P.anc_start[l]; kb < P.anc_start[l + 1]; ++kb) {
                const int b = P.anc_dofs[kb];
                const float c = (a == b) ? Hs[symD_idx(D, a, a)] : 0.5f * Hs[a < b ? symD_idx(D, a, b) : symD_idx(D, b, a)];
                z += ld6(s + Y.S + b * 6) * c;
            }
            inertia_apply_adj(B, z, ld6(s + Y.S + a * 6), aR, au, dummy);
        }
        const SP o = s + Y.aIbar + l * 12;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) o[r * 3 + c] += aR.m[r][c];
        add3(o + 9, au);
    }
    // motion subspace: aS_a += sum_{l in subtree(link(a))} I_l sum_{b in anc(l)} (aH[a][b] + aH[b][a]) S_b
    DFX_FOR(a, D) {
        const int la = P.dof_link[a];
        SV acc = sv_zero();
        for (int kl = P.sub_start[la]; kl < P.sub_start[la + 1]; ++kl) {
            const int l = P.sub_links[kl];
            const BodyInertia B = body_inertia(P, s + Y.Xsm + l * 7, l);
            SV y = sv_zero();
            for (int kb = P.anc_start[l]; kb < P.anc_start[l + 1]; ++kb) {
                const int b = P.anc_dofs[kb];
                const float c = (a == b) ? 2.0f * Hs[symD_idx(D, a, a)] : Hs[a < b ? symD_idx(D, a, b) : symD_idx(D, b, a)];
                y += ld6(s + Y.S + b * 6) * c;
            }
            acc += inertia_apply(B, y);
        }
        add6(s + Y.aS + a * 6, acc);
    }
    g.sync();
}

#else
// adjoint of H(S, I) w.r.t. S (-> aS) and the body inertias (-> aIbar, aXsm.p), from the symmetrised cotangent Hs.
// With c_aa = Hs_aa, c_ab = Hs_ab / 2 the cotangent is that of  sum_l sum_{a,b in anc(l)} c_ab S_a^T I_l S_b :
//   * body inertias: the bilinear form of link l is tr(I_l K_l) with the symmetric moment matrix
//         K_l = sum_{a,b in anc(l)} c_ab S_b S_a^T = sum_{a in anc(l)} (S_a g_a^T + g_a S_a^T),   g_a = c_aa/2 S_a + sum_{b < a} c_ab S_b
//     (g_a depends on the dof only: formed once per dof), and d tr(I K)/d(R, u) is the vector-pair adjoint of y = I x
//     summed over the six pairs (x = column k of K, r = e_k) -- 6 instead of |anc(l)| (8-15) evaluations per link and
//     |anc(l)| rank-2 updates instead of |anc(l)|^2 axpys;
//   * motion subspace:  aS_a = sum_{l in subtree(link(a))} I_l (2 sum_{b in anc(l)} c_ab S_b)
//                            = Ic_link(a) p_a + sum_{m strictly below link(a)} Ic_m (sum_{b in dofs(m)} Hs_ab S_b),
//     p_a = 2 Hs_aa S_a + sum_{b in anc(link(a)), b != a} Hs_ab S_b, with the COMPOSITE inertias Ic_m = sum_{l in subtree(m)} I_l
//     (packed symmetric 6x6, accumulated leaves -> root in place in the reference's reversed link order, sim.py eval_crba):
//     one 6x6 product per (dof, link below it) instead of a factored-inertia evaluation plus |anc(l)| axpys.
// Scratch: the composites (L,21) live in the idle (Xl, vj, pX, af) region; g (D,6) in the aS slot itself, which is still all-zero
// here (crba_adj is its first writer of the substep) and receives aS in the last pass.
DFX_HD float hs_at(SP Hs, int D, int a, int b) { return Hs[a < b ? symD_idx(D, a, b) : symD_idx(D, b, a)]; }

template <class Grp>
DFX_HD void crba_adj(const Pack& P, const Layout& Y, SP s, const Grp& g) {
    const int D = P.D, L = P.L;
    const SP Hs = s + Y.Lm;
    const SP Ic = s + Y.Xl;          // (L,21) <= (L,26)
    const SP G = s + Y.aS;           // (D,6)
    DFX_FOR(l, L) inertia_sym21(body_inertia(P, s + Y.Xsm + l * 7, l), Ic + l * 21);
    DFX_FOR(a, D) {
        const int la = P.dof_link[a];
        SV ga = ld6(s + Y.S + a * 6) * (0.5f * Hs[symD_idx(D, a, a)]);
        for (int kb = P.anc_start[la]; kb < P.anc_start[la + 1]; ++kb) {
            const int b = P.anc_dofs[kb];
            if (b >= a) break;                   // (ascending dof index)
            ga += ld6(s + Y.S + b * 6) * (0.5f * Hs[symD_idx(D, b, a)]);
        }
        st6(G + a * 6, ga);
    }
    g.sync();
    // composite inertias in place, leaves -> root (children have larger indices than their parents): one thread per packed entry
    DFX_FOR(c, 21) {
        for (int l = L - 1; l > 0; --l) {
            const int par = P.parent[l];
            if (par >= 0) Ic[par * 21 + c] += Ic[l * 21 + c];
        }
    }
    // body inertia parameters from the moment matrix of the link
    DFX_FOR(l, L) {
        float K[21];
#pragma unroll
        for (int e = 0; e < 21; ++e) K[e] = 0.0f;
        for (int ka = P.anc_start[l]; ka < P.anc_start[l + 1]; ++ka) {
            const int a = P.anc_dofs[ka];
            const SV Sa = ld6(s + Y.S + a * 6), ga = ld6(G + a * 6);
            const float sv[6] = {Sa.w.x, Sa.w.y, Sa.w.z, Sa.v.x, Sa.v.y, Sa.v.z};
            const float gv[6] = {ga.w.x, ga.w.y, ga.w.z, ga.v.x, ga.v.y, ga.v.z};
#pragma unroll
            for (int i = 0; i < 6; ++i)
#pragma unroll
                for (int j = i; j < 6; ++j) K[sym_idx(i, j)] += sv[i] * gv[j] + gv[i] * sv[j];
        }
        const BodyInertia B = body_inertia(P, s + Y.Xsm + l * 7, l);
        M3 aR = m3_zero();
        V3 au = v3zero();
        SV dummy = sv_zero();
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            float col[6], ek[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) { col[i] = K[i <= k ? sym_idx(i, k) : sym_idx(k, i)]; ek[i] = (i == k) ? 1.0f : 0.0f; }
            inertia_apply_adj(B, SV{V3{col[0], col[1], col[2]}, V3{col[3], col[4], col[5]}},
                              SV{V3{ek[0], ek[1], ek[2]}, V3{ek[3], ek[4], ek[5]}}, aR, au, dummy);
        }
        const SP o = s + Y.aIbar + l * 12;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) o[r * 3 + c] += aR.m[r][c];
        add3(o + 9, au);
    }
    g.sync();
    // motion subspace
    DFX_FOR(a, D) {
        const int la = P.dof_link[a];
        SV pa = ld6(s + Y.S + a * 6) * (2.0f * Hs[symD_idx(D, a, a)]);
        for (int kb = P.anc_start[la]; kb < P.anc_start[la + 1]; ++kb) {
            const int b = P.anc_dofs[kb];
            if (b != a) pa += ld6(s + Y.S + b * 6) * hs_at(Hs, D, a, b);
        }
        SV acc = sym21_apply(Ic + la * 21, pa);
        for (int km = P.sub_start[la] + 1; km < P.sub_start[la + 1]; ++km) {      // (the list starts with la itself)
            const int m = P.sub_links[km];
            SV x = sv_zero();
            for (int b = P.qd_start[m]; b < P.qd_start[m + 1]; ++b) x += ld6(s + Y.S + b * 6) * Hs[symD_idx(D, a, b)];    // (a < b)
            acc += sym21_apply(Ic + m * 21, x);
        }
        st6(s + Y.aS + a * 6, acc);      // (over g_a: nobody reads g in this pass, and aS was zero on entry)
    }
    g.sync();
}
#endif

// =====================================================================================
// semi-implicit Euler
// =====================================================================================
DFX_HD void integrate_link_fwd(const Pack& P, const Layout& Y, SP s, float dt, int i) {
    const int type = P.type[i], qs = P.q_start[i], ds = P.qd_start[i];
    const SP q = s + Y.q;
    const SP qd = s + Y.qd;
    const SP qdd = s + Y.qdd;
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) {
        const float qd_new = qd[ds] + qdd[ds] * dt;
        q[qs] = q[qs] + qd_new * dt;
        qd[ds] = qd_new;
    } else if (is_joint(P, type, JOINT_BALL)) {
        const V3 w = ld3(qd + ds) + ld3(qdd + ds) * dt;
        const Q4 r = ld4(q + qs);
        const Q4 drdt = qmul(Q4{w.x, w.y, w.z, 0.0f}, r) * 0.5f;
        st4(q + qs, qnormalize(r + drdt * dt));
        st3(qd + ds, w);
    } else if (is_joint(P, type, JOINT_FREE)) {
        const V3 w = ld3(qd + ds) + ld3(qdd + ds) * dt;
        const V3 v = ld3(qd + ds + 3) + ld3(qdd + ds + 3) * dt;
        const V3 p = ld3(q + qs);
        const V3 dpdt = v + cross(w, p);
        const Q4 r = ld4(q + qs + 3);
        const Q4 drdt = qmul(Q4{w.x, w.y, w.z, 0.0f}, r) * 0.5f;
        st3(q + qs, p + dpdt * dt);
        st4(q + qs + 3, qnormalize(r + drdt * dt));
        st3(qd + ds, w);
        st3(qd + ds + 3, v);
    }
}

template <class Grp>
DFX_HD void integrate_fwd(const Pack& P, const Layout& Y, SP s, float dt, const Grp& g) {
    DFX_FOR(i, P.L) {
        integrate_link_fwd(P, Y, s, dt, i);
        // K1 of the next substep: the joint-local transform depends on the link's own coordinates only, which this thread just
        // wrote -- no phase and no barrier of its own
        if constexpr (Grp::kFusedPhases) kin_local_fwd(P, Y, s, i);
    }
    g.pre_store();         // (q, qd) of the next substep leave for the tape right after this barrier
    // the next phase (K2 / K3 of the next substep) overwrites the row fields this substep's tape store may still be reading
    if constexpr (Grp::kFusedPhases) g.row_reusable();
    g.sync();
}

// adjoint: aq/aqd hold d/d(q', qd') on entry and d/d(q, qd) (direct part) on exit; aqdd is written.
// q, qd, qdd in scratch are the substep INPUT values.
DFX_HD void integrate_link_adj(const Pack& P, const Layout& Y, SP s, float dt, int i) {
    const int type = P.type[i], qs = P.q_start[i], ds = P.qd_start[i];
    const SP q = s + Y.q;
    const SP qd = s + Y.qd;
    const SP qdd = s + Y.qdd;
    const SP aq = s + Y.aq;
    const SP aqd = s + Y.aqd;
    const SP aqdd = s + Y.aqdd;
    if (is_joint(P, type, JOINT_PRISMATIC) || is_joint(P, type, JOINT_REVOLUTE)) {
        const float aqdn = aqd[ds] + aq[qs] * dt;
        aqd[ds] = aqdn;
        aqdd[ds] = aqdn * dt;
    } else if (is_joint(P, type, JOINT_BALL)) {
        const V3 w = ld3(qd + ds) + ld3(qdd + ds) * dt;
        const Q4 r = ld4(q + qs);
        const Q4 W = Q4{w.x, w.y, w.z, 0.0f};
        const Q4 rr = r + qmul(W, r) * (0.5f * dt);
        const Q4 arr = qnormalize_adj(rr, ld4(aq + qs));
        Q4 ar = arr, aW = qzero();
        qmul_adj(W, r, arr * (0.5f * dt), aW, ar);
        const V3 aw = ld3(aqd + ds) + qv(aW);
        st4(aq + qs, ar);
        st3(aqd + ds, aw);
        st3(aqdd + ds, aw * dt);
    } else if (is_joint(P, type, JOINT_FREE)) {
        const V3 w = ld3(qd + ds) + ld3(qdd + ds) * dt;
        const V3 p = ld3(q + qs);
        const Q4 r = ld4(q + qs + 3);
        const Q4 W = Q4{w.x, w.y, w.z, 0.0f};
        const Q4 rr = r + qmul(W, r) * (0.5f * dt);
        const Q4 arr = qnormalize_adj(rr, ld4(aq + qs + 3));
        Q4 ar = arr, aW = qzero();
        qmul_adj(W, r, arr * (0.5f * dt), aW, ar);
        V3 aw = ld3(aqd + ds) + qv(aW);
        V3 av = ld3(aqd + ds + 3);
        V3 ap = ld3(aq + qs);
        const V3 adpdt = ap * dt;
        av += adpdt;
        cross_adj(w, p, adpdt, aw, ap);
        st3(aq + qs, ap);
        st4(aq + qs + 3, ar);
        st3(aqd + ds, aw);
        st3(aqd + ds + 3, av);
        st3(aqdd + ds, aw * dt);
        st3(aqdd + ds + 3, av * dt);
    }
}

template <class Grp>
DFX_HD void integrate_adj(const Pack& P, const Layout& Y, SP s, float dt, const Grp& g) {
    g.cta_tasks(s, P.L, true, [&](SP se, int i) { integrate_link_adj(P, Y, se, dt, i); });
}

// =====================================================================================
// one substep, forward and adjoint
// =====================================================================================
// adjoint of one substep.  Pre: scratch [q .. qdd] = the substep's taped block (entering q, qd and the
// forward intermediates), act, musc, A = H^-1 of the segment; aq, aqd = cotangents of the substep output.  Post: aq, aqd = cotangents of the substep input;
// aact, amusc, aH (Lm slot) accumulated.  `apply_crba` is set on the substep that built H.
// kSeeded (dfx_step.h dynamics_state_backward): the adjoint of the substep's dynamics without its integrator -- integrate_adj is
// skipped (aqdd, aq, aqd are the caller's seeds), and the cotangent gtau[D] of tau (NULL: none) joins atau after solve_adj's
// Hs update, which reads other threads' atau entries without a barrier of its own; a barrier then precedes crba_adj / tau_adj.
template <bool kWrench = false, bool kSeeded = false, class Grp>
DFX_HD void substep_adj(const Pack& P, const Layout& Y, SP s, float dt, bool apply_crba, HinvView hv, const RowFmt& rf, const Grp& g,
                        int xw = -1, const float* gtau = nullptr) {
    zero_range(s + Y.aXsc, P.L * 32 + P.D * 6, g);      // aXsc, av, aXsm, aS, aa are adjacent (af is overwritten by tau_adj)
    zero_range(s + Y.aIbar, P.L * 12, g);
    // (no barrier: integrate_adj and solve_adj do not touch the zeroed accumulators, and two barriers follow before their first use)
    // phase_sync(): CTA-wide barrier that keeps the warps of a CTA inside the same phase, so that the
    // instruction working set per SM is one or two phases instead of the whole body
    if constexpr (!kSeeded) integrate_adj(P, Y, s, dt, g);
    solve_adj(P, Y, s, hv, g);              // tau slot <- atau
    g.copy_wait_all();                      // the bulk of the tape row (transforms, S, v, a, wrenches) is needed from here on
    g.row_unpack(s + Y.q, s + Y.stage, rf); // (bf16 tape: the staged halves become the fp32 scratch fields)
    g.sync();
    if constexpr (kSeeded) {
        if (gtau) DFX_FOR(i, P.D) s[Y.tau + i] += gtau[i];
        g.sync();
    }
    if (apply_crba) crba_adj(P, Y, s, g);
    tau_adj(P, Y, s, s + Y.tau, g);
    g.phase_sync();
    if (P.M > 0) {
        // muscles (and the contacts of a muscle model) scatter their cotangents in fixed point: deterministic sums
        const float scale = adj_scatter_scale(P, Y, s, g);
        muscle_adj(P, Y, s, scale, g);
        contact_adj(P, Y, s, g);
        adj_collect(P, Y, s, scale, g);
        body_force_adj<kWrench>(P, Y, s, g, xw);
    } else {
        // contact-only model: one item per link -- its rigid-body force adjoint, then the cotangents of its own contact points
        // in the pack's order (contacts are grouped by body, cbody_start).  Every av / aXsc entry has one writer adding in a
        // fixed order, so the sums are bit-reproducible; float atomics from compacted contact tasks would add in an order that
        // varies from run to run.  (A1 inside body_force_link_adj does not read what the contacts add.)
        DFX_FOR(i, P.L) {
            body_force_link_adj<kWrench>(P, Y, s, i, xw);
            if (P.ground)
                for (int k = P.cbody_start[i]; k < P.cbody_start[i + 1]; ++k) contact_point_adj(P, Y, s, k, 1.0f, g);
        }
        g.sync();
    }
    g.phase_sync();
    kin_adj(P, Y, s, g);
    g.phase_sync();
}

}  // namespace dfx
