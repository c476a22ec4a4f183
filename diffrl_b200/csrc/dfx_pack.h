// dfx_pack.h -- "ModelPack": the static description of ONE articulation, shared by every
// environment of a batch (all environments of a DFlexEnv are copies of the same articulation,
// reference envs/ant.py:97-124 with env_dist = 0), plus the per-environment scratch layout.
//
// The pack is built on the host (dfx_capi.cu) from the reference Model's flat tensors
// (dflex/dflex/model.py:1646-1879 field names) and lives in device global memory; kernels read it
// through the read-only path (it is a few KB and stays L1/L2 resident).
#pragma once

namespace dfx {

enum JointType { JOINT_PRISMATIC = 0, JOINT_REVOLUTE = 1, JOINT_BALL = 2, JOINT_FIXED = 3, JOINT_FREE = 4 };
constexpr int kJointMaskAll = 31;

struct Pack {
    // sizes (per environment)
    int L;       // links
    int D;       // dofs            (joint_qd)
    int Q;       // coordinates     (joint_q)
    int C;       // ground-contact points
    int M;       // muscles
    int W;       // muscle way-points
    int nlev;    // tree depth
    int nround;  // rounds of the chain decomposition (below)
    int MG;      // muscle groups (below)
    int root_round_single;   // the last chain round holds nothing but single-link chains of roots (a root -> leaf recursion skips it)
    int ground;  // model.ground && C > 0
    int jmask;   // bit t set: some link has joint type t.  The size-specialised tile kernels overwrite it with a compile-time constant
                 // (like L, D, Q, C, M) so that the branches of absent joint types are not compiled in: the per-substep body of the
                 // adjoint is several times larger than the instruction cache, every dead branch costs fetches
    float gx, gy, gz;

    // ---- per link (L) ----
    const int* type;
    const int* parent;       // local link index, -1 for roots
    const int* q_start;      // (L+1)
    const int* qd_start;     // (L+1)
    const int* level_start;  // (nlev+1) offsets into level_links
    const int* level_links;  // (L) links ordered by depth
    const int* child_start;  // (L+1)
    const int* child_idx;    // children lists
    const int* anc_start;    // (L+1) ancestor-or-self dof lists, ascending dof index
    const int* anc_dofs;
    const int* sub_start;    // (L+1) subtree (descendant-or-self) link lists
    const int* sub_links;
    const int* path_start;   // (L+1) the links on the path root -> ... -> i (i included), root first
    const int* path_links;
    // Chain decomposition for tree recursions: a chain starts at a leaf or at a link with >= 2 children and runs upwards
    // while the parent has no other child; a chain's round is 0 for leaf chains, else 1 + the largest round of the chains
    // hanging below it.  Chains are sorted by round; chain_links lists a chain bottom-up.  A leaves -> root recursion
    // processes round 0, 1, ... with ONE barrier per round (a chain is walked by one thread), a root -> leaves recursion
    // the rounds in reverse and every chain top-down: 2-3 barriers instead of one per tree level (Humanoid: 10 levels).
    const int* round_start;  // (nround+1) offsets into the chain list
    const int* chain_start;  // (nchain+1) offsets into chain_links
    const int* chain_links;  // (L)
    const float* X_pj;       // (L,7)
    const float* X_cm;       // (L,7)
    const float* axis;       // (L,3)
    const float* I_c;        // (L,9) rotational inertia about the COM, body frame (row-major)
    const float* mass;       // (L)
    const float* target_ke;  // (L)
    const float* target_kd;  // (L)
    const float* limit_ke;   // (L)
    const float* limit_kd;   // (L)
    // ---- per coordinate (Q) ----
    const float* target;
    const float* limit_lower;
    const float* limit_upper;
    // ---- per dof (D) ----
    const float* armature;
    const int* dof_link;
    // ---- contacts, grouped by body, original order kept inside a body ----
    const int* cbody_start;  // (L+1)
    const int* cbody;        // (C)
    const float* cpoint;     // (C,3)
    const float* cdist;      // (C)
    const float* cmat;       // (C,4)  ke, kd, kf, mu
    // ---- muscles ----
    const int* mstart;       // (M+1)
    const int* mlinks;       // (W) local link index
    // only the segments whose two way-points sit on DIFFERENT links pull (reference sim.py:1231: l0 == l1 -> skip): the pack
    // lists them per muscle (the SNU model: 198 of 484 segments, 1-2 per muscle).  Muscles whose active segments connect
    // the SAME links (in the same order) form GROUPS of at most 8 segment evaluations: an item slot walks a group, loads the two link
    // transforms (and, in the adjoint, the two wrench cotangents) once, sums the members' wrenches in registers and
    // scatters ONE wrench per link and segment position instead of one per muscle (the fixed-point scatter is half of a
    // muscle's instructions).  Groups are sorted by size, largest first.
    const int* aseg_start;   // (M+1) offsets into aseg_way
    const int* aseg_way;     // way-point index i of an active segment (i, i+1)
    const int* morder;       // (M) muscles sorted by group
    const int* mgrp_start;   // (MG+1) offsets into morder
    const float* mpoints;    // (W,3)
};

// Offsets (in floats) of the per-environment scratch block.  Forward kernels use [0, fwd_size),
// backward kernels [0, bwd_size).  A field that a layout does not hold has offset -1.
struct Layout {
    // primal
    int q, qd, act, musc, tau, qdd, Xl, vj;
    int Xsc, Xsm, S, v, a, f, ft;
    int cmask, fxs, fx, fxH;   // poison bits + int64 fixed-point accumulators of the deterministic scatter-adds
    int A;     // H, then H^-1 (D,D); -1: the adjoint reads H^-1 from the tape in global memory (kLayoutHinvGlobal)
    int Lm;    // forward: Cholesky factor (D,D); backward: the symmetrised cotangent of H, packed upper triangle (D(D+1)/2)
    int Icmp;  // composite inertias (L,21) + F (D,6) during CRBA
    int fwd_size;
    int tape_row;  // floats of the contiguous [q, qd, X_sc, X_sm, S, v, a, f_tot, qdd] block
    // adjoint
    int aq, aqd, aqdd, aact, amusc;
    int aXsc, aXsm, aS, av, aa, af, aIbar /* (L,12): dL/dR (9) + dL/du (3) */, pX;
    int bwd_size;
    int overlay;   // forward: the mass-matrix temporaries (Lm, Icmp) share the region of (Xl, vj, f, fx) -- see make_layout
    int stage;     // staging area of the bf16 tape (tile kernels): (tail - head) / 2 floats that are dead while a row is in flight
};

#if defined(__CUDACC__)
#define DFX_LAYOUT_FN __host__ __device__ constexpr
#else
#define DFX_LAYOUT_FN constexpr
#endif
DFX_LAYOUT_FN int dfx_round_up(int x, int m) { return (x + m - 1) / m * m; }
DFX_LAYOUT_FN int dfx_max(int a, int b) { return a > b ? a : b; }
DFX_LAYOUT_FN int dfx_sym_count(int D) { return D * (D + 1) / 2; }
// a tape row is [q, qd, X_sc, X_sm, S | v, a, f_tot | q'', padding]; with a bf16 tape the middle -- link velocities, bias
// accelerations and total link wrenches: quantities that enter the adjoint as multipliers -- is stored as bf16.  The state,
// q'' and everything that carries POSITIONS stay fp32: the link transforms (contact depths are millimetres of metre-sized
// positions) and the motion subspace S (its linear part is p x w) -- measured on the host emulation, rounding S alone costs
// 1-3 % of the state gradients, rounding (v, a, f_tot) 0.1-0.7 %
DFX_LAYOUT_FN int dfx_row_middle(int L, int D) { (void)D; return L * 18; }      // v, a, f_tot (L,6 each)
// floats (4-byte units) one row occupies in the tape
DFX_LAYOUT_FN int dfx_row_units(int tape_row, int L, int D, bool bf16) { return bf16 ? tape_row - dfx_row_middle(L, D) / 2 : tape_row; }

// layout modes
constexpr int kLayoutLegacy = 0;       // one layout for forward and backward (forward-only and adjoint-only fields share a region)
constexpr int kLayoutCompact = 1;      // separate forward / backward layouts, sized for the large articulations (Humanoid, SNU):
                                       //   forward : the mass-matrix temporaries (Lm, Icmp: live only inside crba_fwd + chol_inverse) OVERLAY
                                       //             the per-substep temporaries (Xl, vj, f, fx: dead by then; fx is re-zeroed afterwards)
                                       //   backward: no forward-only fields at all
constexpr int kLayoutHinvGlobal = 2;   // backward: H^-1 is not staged in shared memory; solve_adj reads its rows from the tape (L2)

DFX_LAYOUT_FN Layout make_layout(int L, int D, int Q, int C, int M, int mode = kLayoutLegacy, bool bwd = false) {
    (void)C;
    Layout y{};
    int o = 0;
#define DFX_TAKE(n) (o += (n), o - (n))
    // [q .. qdd] is one contiguous block: it is what forward writes to the tape per substep and what the
    // adjoint reads back instead of re-running the forward dynamics (tape_row floats)
    y.q = DFX_TAKE(Q); y.qd = DFX_TAKE(D);
    y.Xsc = DFX_TAKE(L * 7); y.Xsm = DFX_TAKE(L * 7); y.S = DFX_TAKE(D * 6); y.v = DFX_TAKE(L * 6); y.a = DFX_TAKE(L * 6);
    y.ft = DFX_TAKE(L * 6); y.qdd = DFX_TAKE(D);
    o = dfx_round_up(o, 4);          // rows are copied with 16-byte transactions
    y.tape_row = o;
    y.act = DFX_TAKE(D); y.musc = DFX_TAKE(M); y.tau = DFX_TAKE(D);
    y.cmask = DFX_TAKE(1);               // poison bits of the fixed-point scatter-adds (bit = body & 31)
    y.fxs = DFX_TAKE(1);                 // fixed-point scale of the cotangent scatter of the current substep
    o = dfx_round_up(o, 4);              // (the H^-1 block is copied with 16-byte transactions in the tile kernels)
    const int adj_floats = Q + 3 * D + M + L * (7 + 6 + 7 + 6 + 6 + 12 + 7) + D * 6 + (M > 0 ? L * 13 : 0);
    if (!(mode & kLayoutCompact)) {
        y.A = DFX_TAKE(D * D); y.Lm = DFX_TAKE(D * D);
        y.Xl = DFX_TAKE(L * 7); y.vj = DFX_TAKE(L * 6);   // kinematics temporaries (joint-local transform, joint velocity)
        // ---- from here on the forward-only and the adjoint-only fields share the same region
        const int shared_end = o;
        y.Icmp = DFX_TAKE(L * 21 + D * 6);
        y.f = DFX_TAKE(L * 6);
        y.fx = DFX_TAKE(L * 12);             // fixed-point accumulators of the contact + muscle wrenches: (L,6) low words, (L,6) high words
        y.fwd_size = o;
        o = shared_end;
        y.overlay = 0;
        // bf16 staging: forward kernels stage in Icmp (live only inside crba_fwd), backward kernels in (Xl, vj, pX, af)
        y.stage = bwd ? y.Xl : y.Icmp;
    } else if (!bwd) {
        y.A = DFX_TAKE(D * D);
        const int u0 = o;
        y.Xl = DFX_TAKE(L * 7); y.vj = DFX_TAKE(L * 6); y.f = DFX_TAKE(L * 6); y.fx = DFX_TAKE(L * 12);
        y.stage = dfx_round_up(o, 4);        // past fx (which must keep reading zero), inside the region of (Lm, Icmp)
        const int u1 = y.stage + dfx_row_middle(L, D) / 2;
        o = u0;
        y.Lm = DFX_TAKE(D * D); y.Icmp = DFX_TAKE(L * 21 + D * 6);
        o = dfx_max(o, u1);
        y.fwd_size = o;
        y.overlay = 1;
        // (adjoint fields: unused by the forward kernels; offsets past the end keep host-side sizing honest)
        y.aq = y.aqd = y.aqdd = y.aact = y.amusc = y.aXsc = y.av = y.aXsm = y.aS = y.aa = y.af = y.aIbar = y.pX = y.fxH = -1;
        y.bwd_size = o;
        return y;
    } else {
        y.A = (mode & kLayoutHinvGlobal) ? -1 : DFX_TAKE(D * D);
        y.Lm = DFX_TAKE(dfx_round_up(dfx_sym_count(D), 4));
        y.Xl = DFX_TAKE(L * 7); y.vj = DFX_TAKE(L * 6);
        y.Icmp = y.f = y.fx = -1;
        y.fwd_size = o + adj_floats;
        y.overlay = 0;
        y.stage = y.Xl;
    }
    // (Xl, vj, pX, af) are contiguous: all four are dead from the moment a substep's adjoint starts until its tape row has
    // landed -- the staging area of the bf16 tape (26 L >= 16 L + 3 D floats for every tree)
    y.pX = DFX_TAKE(L * 7); y.af = DFX_TAKE(L * 6);
    y.aq = DFX_TAKE(Q); y.aqd = DFX_TAKE(D); y.aqdd = DFX_TAKE(D); y.aact = DFX_TAKE(D); y.amusc = DFX_TAKE(M);
    y.aXsc = DFX_TAKE(L * 7); y.av = DFX_TAKE(L * 6); y.aXsm = DFX_TAKE(L * 7); y.aS = DFX_TAKE(D * 6); y.aa = DFX_TAKE(L * 6);
    y.aIbar = DFX_TAKE(L * 12);
    y.fxH = DFX_TAKE(M > 0 ? L * 13 : 0);            // high words of the fixed-point cotangent scatter into aXsc (L,7) and av (L,6); the low words live in aXsc / av
    y.bwd_size = o;
    (void)adj_floats;
#undef DFX_TAKE
    return y;
}

// The external-wrench variants of the step kernels (include/dfx.h DfxExternalWrench) keep two more per-environment fields
// past the end of the layout, so every other offset stays as it is: the wrench of every link (L,6: torque, force), loaded
// once per env-step, and in the adjoint its cotangent (L,6), accumulated over the substeps.
DFX_LAYOUT_FN int wrench_offset(const Layout& Y, bool bwd) { return dfx_round_up(bwd ? Y.bwd_size : Y.fwd_size, 4); }
DFX_LAYOUT_FN int wrench_scratch_end(const Layout& Y, int L, bool bwd) { return wrench_offset(Y, bwd) + dfx_round_up((bwd ? 12 : 6) * L, 4); }

}  // namespace dfx
