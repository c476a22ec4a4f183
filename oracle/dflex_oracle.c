/* dflex_oracle.c -- CPU restatement of the reference's articulated rigid-body step.
 *
 * TEST INFRASTRUCTURE ONLY: the parity checker for the CUDA path.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline leg may build or call this; nothing under diffrl_b200/ does.
 *
 * It follows the reference (NVlabs/DiffRL, dflex/dflex) function by function and keeps its dense
 * formulation and operation order -- 6x6 world inertias T^T I T, dense J (6L x D), block-diagonal M,
 * P = M J, H = J^T P, Cholesky, forward/backward substitution -- i.e. it is deliberately NOT the
 * algorithm of the CUDA kernels (composite-rigid-body H, factored inertias, explicit H^-1, gathers).
 * Each function cites the reference lines it restates.  Parity of THIS file is pinned by
 * tests/test_oracle.py against the golden vectors recorded from the unmodified reference
 * (oracle/make_golden.py) and against the reference's own compiled kernels (oracle/ref_driver.py).
 *
 * Built three times (oracle/Makefile): REAL=float -> liboracle_f32.so (forward parity), REAL=double ->
 * liboracle_f64.so, whose central finite differences of sum(gq.q' + gqd.qd') check the hand-derived
 * adjoint kernels independently of any adjoint code (oracle_fd_gradient below), and REAL=double _Complex ->
 * liboracle_c64.so, whose complex-step derivative of the same loss is exact to rounding on the branches the
 * fp64 forward takes (oracle_exact_gradient).  Every comparison of reals goes through RLT / RGT / RGE, so the
 * three builds take their branches on the same (real) values; the f32 and f64 arithmetic is unchanged by it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/dfx.h"

#ifndef REAL
#define REAL float
#endif
typedef REAL real;
#ifdef ORACLE_COMPLEX
/* Complex-step build (REAL = double _Complex): every input carries an imaginary perturbation i*h, every branch is decided
 * on the real part, so Im(output)/h is the exact derivative of the branch actually taken (oracle_exact_gradient). */
#include <complex.h>
#undef I   /* the inertia parameter below is named I */
#define RE(x) creal(x)
#define R_SQRT(x) csqrt(x)
#define R_SIN(x) csin(x)
#define R_COS(x) ccos(x)
#else
#define RE(x) (x)
#define R_SQRT(x) ((real)sqrt((double)(x)))
#define R_SIN(x) ((sizeof(real) == 4) ? (real)sinf((float)(x)) : (real)sin((double)(x)))
#define R_COS(x) ((sizeof(real) == 4) ? (real)cosf((float)(x)) : (real)cos((double)(x)))
#endif
/* every comparison of reals goes through these: real parts in the complex build, the plain comparison otherwise */
#define RLT(a, b) (RE(a) < RE(b))
#define RGT(a, b) (RE(a) > RE(b))
#define RGE(a, b) (RE(a) >= RE(b))

/* Branch record (oracle_branch_signature): the decisions of the contact and joint-limit model, in the order they are taken */
enum { BR_PENETRATE, BR_VN_NEG, BR_CAP_VISCOUS, BR_CAP_COULOMB, BR_LOWER, BR_UPPER, BR_COUNT };
static struct { int on; uint64_t hash; int64_t counts[BR_COUNT]; } g_branch;
static int branch_record(int kind, int taken) {
    if (g_branch.on) {
        /* FNV-1a over (kind, taken); the friction cap records which of its two branches was taken */
        g_branch.hash = (g_branch.hash ^ (uint64_t)(2 * kind + (taken != 0))) * 1099511628211ull;
        if (kind == BR_CAP_VISCOUS) g_branch.counts[taken ? BR_CAP_VISCOUS : BR_CAP_COULOMB]++;
        else if (taken) g_branch.counts[kind]++;
    }
    return taken;
}
#define BRANCH(kind, cond) branch_record((kind), (cond))

typedef struct { real x, y, z; } v3;
typedef struct { real x, y, z, w; } q4;
typedef struct { v3 p; q4 q; } xf;          /* spatial_transform, spatial.h:166 */
typedef struct { v3 w, v; } sv;             /* spatial_vector, spatial.h:6 */
typedef struct { real d[6][6]; } sm;        /* spatial_matrix, spatial.h:425 */

/* ---- vec3.h:23-62 */
static v3 V(real x, real y, real z) { v3 r = {x, y, z}; return r; }
static v3 vadd(v3 a, v3 b) { return V(a.x + b.x, a.y + b.y, a.z + b.z); }
static v3 vsub(v3 a, v3 b) { return V(a.x - b.x, a.y - b.y, a.z - b.z); }
static v3 vmul(v3 a, real s) { return V(a.x * s, a.y * s, a.z * s); }
static real vdot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static v3 vcross(v3 a, v3 b) { return V(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
static real vlen(v3 a) { return R_SQRT(vdot(a, a)); }
/* vec3.h:96-103: zero vector for zero length (kEps = 0, adjoint.h:73) */
static v3 vnormalize(v3 a) { real l = vlen(a); return RGT(l, 0) ? V(a.x / l, a.y / l, a.z / l) : V(0, 0, 0); }

/* ---- quat.h:44-116 */
static q4 Qn(real x, real y, real z, real w) { q4 r = {x, y, z, w}; return r; }
static q4 quat_from_axis_angle(v3 axis, real angle) {
    real half = angle * (real)0.5, w = R_COS(half), s = R_SIN(half);
    v3 v = vmul(axis, s);
    return Qn(v.x, v.y, v.z, w);
}
static q4 qmul(q4 a, q4 b) {
    return Qn(a.w * b.x + b.w * a.x + a.y * b.z - b.y * a.z, a.w * b.y + b.w * a.y + a.z * b.x - b.z * a.x,
              a.w * b.z + b.w * a.z + a.x * b.y - b.x * a.y, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
static v3 rotate(q4 q, v3 x) { /* quat.h:113-116 */
    v3 u = V(q.x, q.y, q.z);
    return vadd(vadd(vmul(x, (real)2 * q.w * q.w - (real)1), vmul(vmul(vcross(u, x), q.w), (real)2)), vmul(vmul(u, vdot(u, x)), (real)2));
}
static q4 qinverse(q4 q) { return Qn(-q.x, -q.y, -q.z, q.w); }
static q4 qnormalize(q4 q) { /* quat.h:70-83 */
    real l = R_SQRT(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    if (RGT(l, 0)) { real inv = (real)1 / l; return Qn(q.x * inv, q.y * inv, q.z * inv, q.w * inv); }
    return Qn(0, 0, 0, 1);
}

/* ---- spatial.h:190-228, 56-70 */
static xf X(v3 p, q4 q) { xf r; r.p = p; r.q = q; return r; }
static xf xf_identity(void) { return X(V(0, 0, 0), Qn(0, 0, 0, 1)); }
static xf xf_multiply(xf a, xf b) { return X(vadd(rotate(a.q, b.p), a.p), qmul(a.q, b.q)); }
static v3 xf_point(xf t, v3 x) { return vadd(t.p, rotate(t.q, x)); }
static sv SVn(v3 w, v3 v) { sv r; r.w = w; r.v = v; return r; }
static sv sv_add(sv a, sv b) { return SVn(vadd(a.w, b.w), vadd(a.v, b.v)); }
static sv sv_sub(sv a, sv b) { return SVn(vsub(a.w, b.w), vsub(a.v, b.v)); }
static sv sv_mul(sv a, real s) { return SVn(vmul(a.w, s), vmul(a.v, s)); }
static real sv_dot(sv a, sv b) { return vdot(a.w, b.w) + vdot(a.v, b.v); }
static sv sv_cross(sv a, sv b) { return SVn(vcross(a.w, b.w), vadd(vcross(a.v, b.w), vcross(a.w, b.v))); }
static sv sv_cross_dual(sv a, sv b) { return SVn(vadd(vcross(a.w, b.w), vcross(a.v, b.v)), vcross(a.w, b.v)); }
/* sim.py:1076-1103 */
static sv xf_twist(xf t, sv x) { v3 w = rotate(t.q, x.w); return SVn(w, vadd(rotate(t.q, x.v), vcross(t.p, w))); }
static sv xf_wrench(xf t, sv x) { v3 v = rotate(t.q, x.v); return SVn(vadd(rotate(t.q, x.w), vcross(t.p, v)), v); }
static real sv_get(sv a, int i) { return i < 3 ? (i == 0 ? a.w.x : i == 1 ? a.w.y : a.w.z) : (i == 3 ? a.v.x : i == 4 ? a.v.y : a.v.z); }

/* spatial_transform_inertia, sim.py:1116-1134 (+ spatial_adjoint spatial.h:559, mat33.h skew/mul) */
static sm transform_inertia(xf t, const real* I /* 6x6 row-major */) {
    q4 qi = qinverse(t.q);                                          /* spatial_transform_inverse :1105 */
    v3 pi = vmul(rotate(qi, t.p), (real)0 - (real)1);
    v3 r1 = rotate(qi, V(1, 0, 0)), r2 = rotate(qi, V(0, 1, 0)), r3 = rotate(qi, V(0, 0, 1));
    real R[3][3] = {{r1.x, r2.x, r3.x}, {r1.y, r2.y, r3.y}, {r1.z, r2.z, r3.z}};   /* columns r1 r2 r3 */
    real K[3][3] = {{0, -pi.z, pi.y}, {pi.z, 0, -pi.x}, {-pi.y, pi.x, 0}};          /* skew(p) */
    real S[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { real a = 0; for (int k = 0; k < 3; ++k) a += K[i][k] * R[k][j]; S[i][j] = a; }
    real T[6][6]; memset(T, 0, sizeof T);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { T[i][j] = R[i][j]; T[i + 3][j + 3] = R[i][j]; T[i + 3][j] = S[i][j]; }
    real TtI[6][6];
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { real a = 0; for (int k = 0; k < 6; ++k) a += T[k][i] * I[k * 6 + j]; TtI[i][j] = a; }
    sm out;
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { real a = 0; for (int k = 0; k < 6; ++k) a += TtI[i][k] * T[k][j]; out.d[i][j] = a; }
    return out;
}
static sv sm_mul(const sm* a, sv b) { /* spatial.h:506-515 */
    real o[6];
    for (int i = 0; i < 6; ++i) { real acc = 0; for (int j = 0; j < 6; ++j) acc += a->d[i][j] * sv_get(b, j); o[i] = acc; }
    return SVn(V(o[0], o[1], o[2]), V(o[3], o[4], o[5]));
}

/* ------------------------------------------------------------------ per-environment model view */
typedef struct {
    int L, D, Q, C, M;
    const DfxModelDesc* m;
    real g[3];
} Art;
#define F(arr, i) ((real)(a->m->arr[i]))
static v3 ld3(const float* p) { return V((real)p[0], (real)p[1], (real)p[2]); }
static xf ld7(const float* p) { return X(ld3(p), Qn((real)p[3], (real)p[4], (real)p[5], (real)p[6])); }

typedef struct {  /* the reference State fields of one environment (model.py:360-388) */
    xf *X_sc, *X_sm; sv *S_s, *v_s, *a_s, *f_s, *ft_s; sm* I_s; real *tau, *qdd;
    real *J, *Mm, *P, *H, *Lc;
} Work;

/* jcalc_transform sim.py:1269-1319 */
static xf jcalc_transform(int type, v3 axis, const real* q, int s) {
    if (type == 0) return X(vmul(axis, q[s]), Qn(0, 0, 0, 1));
    if (type == 1) return X(V(0, 0, 0), quat_from_axis_angle(axis, q[s]));
    if (type == 2) return X(V(0, 0, 0), Qn(q[s], q[s + 1], q[s + 2], q[s + 3]));
    if (type == 3) return xf_identity();
    if (type == 4) return X(V(q[s], q[s + 1], q[s + 2]), Qn(q[s + 3], q[s + 4], q[s + 5], q[s + 6]));
    return xf_identity();
}
/* eval_rigid_fk / compute_link_transform sim.py:1638-1711 */
static void eval_rigid_fk(const Art* a, const real* q, Work* w) {
    for (int i = 0; i < a->L; ++i) {
        int parent = a->m->joint_parent[i];
        xf X_sp = parent >= 0 ? w->X_sc[parent] : xf_identity();
        xf X_jc = jcalc_transform(a->m->joint_type[i], ld3(a->m->joint_axis + i * 3), q, a->m->joint_q_start[i] - a->m->joint_q_start[0]);
        xf X_sc = xf_multiply(X_sp, xf_multiply(ld7(a->m->joint_X_pj + i * 7), X_jc));
        w->X_sc[i] = X_sc;
        w->X_sm[i] = xf_multiply(X_sc, ld7(a->m->joint_X_cm + i * 7));
    }
}
/* jcalc_motion sim.py:1323-1387 */
static sv jcalc_motion(int type, v3 axis, xf X_sj, sv* S, const real* qd, int s) {
    if (type == 0) { S[s] = xf_twist(X_sj, SVn(V(0, 0, 0), axis)); return sv_mul(S[s], qd[s]); }
    if (type == 1) { S[s] = xf_twist(X_sj, SVn(axis, V(0, 0, 0))); return sv_mul(S[s], qd[s]); }
    if (type == 2) {
        S[s] = xf_twist(X_sj, SVn(V(1, 0, 0), V(0, 0, 0)));
        S[s + 1] = xf_twist(X_sj, SVn(V(0, 1, 0), V(0, 0, 0)));
        S[s + 2] = xf_twist(X_sj, SVn(V(0, 0, 1), V(0, 0, 0)));
        return sv_add(sv_add(sv_mul(S[s], qd[s]), sv_mul(S[s + 1], qd[s + 1])), sv_mul(S[s + 2], qd[s + 2]));
    }
    if (type == 4) {
        for (int k = 0; k < 6; ++k) { real e[6] = {0, 0, 0, 0, 0, 0}; e[k] = 1; S[s + k] = SVn(V(e[0], e[1], e[2]), V(e[3], e[4], e[5])); }
        return SVn(V(qd[s], qd[s + 1], qd[s + 2]), V(qd[s + 3], qd[s + 4], qd[s + 5]));
    }
    return SVn(V(0, 0, 0), V(0, 0, 0));
}
/* eval_rigid_id / compute_link_velocity sim.py:1716-1789 */
static void eval_rigid_id(const Art* a, const real* qd, Work* w) {
    for (int i = 0; i < a->L; ++i) {
        int parent = a->m->joint_parent[i];
        xf X_sp = parent >= 0 ? w->X_sc[parent] : xf_identity();
        xf X_sj = xf_multiply(X_sp, ld7(a->m->joint_X_pj + i * 7));
        sv v_j = jcalc_motion(a->m->joint_type[i], ld3(a->m->joint_axis + i * 3), X_sj, w->S_s, qd, a->m->joint_qd_start[i] - a->m->joint_qd_start[0]);
        sv v_p = SVn(V(0, 0, 0), V(0, 0, 0)), a_p = v_p;
        if (parent >= 0) { v_p = w->v_s[parent]; a_p = w->a_s[parent]; }
        sv v_s = sv_add(v_p, v_j);
        sv a_s = sv_add(a_p, sv_cross(v_s, v_j));
        xf X_sm = w->X_sm[i];
        real I_m[36];
        for (int k = 0; k < 36; ++k) I_m[k] = (real)a->m->body_I_m[i * 36 + k];
        real mass = I_m[3 * 6 + 3];
        sv f_g_m = sv_mul(SVn(V(0, 0, 0), V(a->g[0], a->g[1], a->g[2])), mass);
        sv f_g_s = xf_wrench(X(X_sm.p, Qn(0, 0, 0, 1)), f_g_m);
        sm I_s = transform_inertia(X_sm, I_m);
        sv f_b_s = sv_add(sm_mul(&I_s, a_s), sv_cross_dual(v_s, sm_mul(&I_s, v_s)));
        w->v_s[i] = v_s; w->a_s[i] = a_s; w->f_s[i] = sv_sub(f_b_s, f_g_s); w->I_s[i] = I_s;
    }
}
/* eval_rigid_contacts_art sim.py:1137-1206 (adjoint.h:94-99 min/step) */
static void eval_rigid_contacts(const Art* a, Work* w) {
    for (int k = 0; k < a->C; ++k) {
        int b = a->m->contact_body0[k], mat = a->m->contact_material[k];
        real ke = (real)a->m->shape_materials[mat * 4 + 0], kd = (real)a->m->shape_materials[mat * 4 + 1];
        real kf = (real)a->m->shape_materials[mat * 4 + 2], mu = (real)a->m->shape_materials[mat * 4 + 3];
        v3 n = V(0, 1, 0);
        v3 p = vsub(xf_point(w->X_sc[b], ld3(a->m->contact_point0 + k * 3)), vmul(n, (real)a->m->contact_dist[k]));
        v3 dpdt = vadd(w->v_s[b].v, vcross(w->v_s[b].w, p));
        real c = vdot(n, p);
        if (BRANCH(BR_PENETRATE, RLT(c, 0)) == 0) continue;
        real vn = vdot(n, dpdt);
        v3 vt = vsub(dpdt, vmul(n, vn));
        real fn = c * ke;
        real stepc = RLT(c, 0) ? (real)1 : (real)0;
        real fd = (BRANCH(BR_VN_NEG, RLT(vn, 0)) ? vn : (real)0) * kd * stepc * ((real)0 - c);
        real cap_a = kf * vlen(vt), cap_b = (real)0 - mu * c * ke;
        v3 ft = vmul(vmul(vnormalize(vt), (BRANCH(BR_CAP_VISCOUS, RLT(cap_a, cap_b)) ? cap_a : cap_b)), stepc);
        v3 f_total = vadd(vmul(n, fn + fd), ft);
        v3 t_total = vcross(p, f_total);
        w->f_s[b] = sv_add(w->f_s[b], SVn(t_total, f_total));
    }
}
/* eval_muscles / compute_muscle_force sim.py:1209-1265 */
static void eval_muscles(const Art* a, const real* activation, Work* w) {
    for (int m = 0; m < a->M; ++m)
        for (int i = a->m->muscle_start[m]; i < a->m->muscle_start[m + 1] - 1; ++i) {
            int l0 = a->m->muscle_links[i], l1 = a->m->muscle_links[i + 1];
            if (l0 == l1) continue;
            v3 p0 = xf_point(w->X_sc[l0], ld3(a->m->muscle_points + i * 3));
            v3 p1 = xf_point(w->X_sc[l1], ld3(a->m->muscle_points + (i + 1) * 3));
            v3 f = vmul(vnormalize(vsub(p1, p0)), activation[m]);
            w->f_s[l0] = sv_sub(w->f_s[l0], SVn(vcross(p0, f), f));
            w->f_s[l1] = sv_add(w->f_s[l1], SVn(vcross(p1, f), f));
        }
}
/* eval_rigid_tau / compute_link_tau / jcalc_tau sim.py:1421-1502, 1792-1842, 1896-1948 */
static void eval_rigid_tau(const Art* a, const real* q, const real* qd, const real* act, Work* w) {
    for (int i = 0; i < a->L; ++i) w->ft_s[i] = SVn(V(0, 0, 0), V(0, 0, 0));
    for (int i = a->L - 1; i >= 0; --i) {
        int type = a->m->joint_type[i], parent = a->m->joint_parent[i];
        int cs = a->m->joint_q_start[i] - a->m->joint_q_start[0], ds = a->m->joint_qd_start[i] - a->m->joint_qd_start[0];
        real tke = F(joint_target_ke, i), tkd = F(joint_target_kd, i), lke = F(joint_limit_ke, i), lkd = F(joint_limit_kd, i);
        sv f_s = sv_add(w->f_s[i], w->ft_s[i]);
        if (type == 0 || type == 1) {
            real qq = q[cs], qdv = qd[ds], lower = F(joint_limit_lower, cs), upper = F(joint_limit_upper, cs), limit_f = 0;
            if (BRANCH(BR_LOWER, RLT(qq, lower))) limit_f = lke * (lower - qq);
            if (BRANCH(BR_UPPER, RGT(qq, upper))) limit_f = lke * (upper - qq);
            real damping_f = ((real)0 - lkd) * qdv;
            w->tau[ds] = (real)0 - sv_dot(w->S_s[ds], f_s) - tke * (qq - F(joint_target, cs)) - tkd * qdv + act[ds] + limit_f + damping_f;
        }
        if (type == 2)
            for (int k = 0; k < 3; ++k) w->tau[ds + k] = (real)0 - sv_dot(w->S_s[ds + k], f_s) - qd[ds + k] * tkd - q[cs + k] * tke;
        if (type == 4)
            for (int k = 0; k < 6; ++k) w->tau[ds + k] = (real)0 - sv_dot(w->S_s[ds + k], f_s);
        if (parent >= 0) w->ft_s[parent] = sv_add(w->ft_s[parent], f_s);
    }
}
/* spatial_jacobian spatial.h:691-738, spatial_mass :801-815, dense_gemm matnn.h:23-43, dense_chol :140-169 */
static void eval_mass_matrix(const Art* a, Work* w) {
    int L = a->L, D = a->D, R6 = 6 * L;
    memset(w->J, 0, sizeof(real) * R6 * D);
    memset(w->Mm, 0, sizeof(real) * R6 * R6);
    for (int i = 0; i < L; ++i) {
        int j = i;
        while (j != -1) {
            int d0 = a->m->joint_qd_start[j] - a->m->joint_qd_start[0], d1 = a->m->joint_qd_start[j + 1] - a->m->joint_qd_start[0];
            for (int col = d0; col < d1; ++col)
                for (int r = 0; r < 6; ++r) w->J[(i * 6 + r) * D + col] = sv_get(w->S_s[col], r);
            j = a->m->joint_parent[j];
        }
        for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) w->Mm[(i * 6 + r) * R6 + i * 6 + c] = w->I_s[i].d[r][c];
    }
    for (int i = 0; i < R6; ++i) for (int j = 0; j < D; ++j) { real s = 0; for (int k = 0; k < R6; ++k) s += w->Mm[i * R6 + k] * w->J[k * D + j]; w->P[i * D + j] = s; }
    for (int i = 0; i < D; ++i) for (int j = 0; j < D; ++j) { real s = 0; for (int k = 0; k < R6; ++k) s += w->J[k * D + i] * w->P[k * D + j]; w->H[i * D + j] = s; }
    memset(w->Lc, 0, sizeof(real) * D * D);
    for (int j = 0; j < D; ++j) {
        real s = w->H[j * D + j] + F(joint_armature, j);
        for (int k = 0; k < j; ++k) { real r = w->Lc[j * D + k]; s -= r * r; }
        s = R_SQRT(s);
        real invS = (real)1 / s;
        w->Lc[j * D + j] = s;
        for (int i = j + 1; i < D; ++i) {
            s = w->H[i * D + j];
            for (int k = 0; k < j; ++k) s -= w->Lc[i * D + k] * w->Lc[j * D + k];
            w->Lc[i * D + j] = s * invS;
        }
    }
}
/* dense_subs matnn.h:188-215 */
static void eval_solve(const Art* a, Work* w) {
    int D = a->D;
    real* x = w->qdd;
    for (int i = 0; i < D; ++i) { real s = w->tau[i]; for (int j = 0; j < i; ++j) s -= w->Lc[i * D + j] * x[j]; x[i] = s / w->Lc[i * D + i]; }
    for (int i = D - 1; i >= 0; --i) { real s = x[i]; for (int j = i + 1; j < D; ++j) s -= w->Lc[j * D + i] * x[j]; x[i] = s / w->Lc[i * D + i]; }
}
/* eval_rigid_integrate / jcalc_integrate sim.py:1505-1636 */
static void eval_integrate(const Art* a, const real* q, const real* qd, const real* qdd, real dt, real* qn, real* qdn) {
    for (int i = 0; i < a->L; ++i) {
        int type = a->m->joint_type[i];
        int cs = a->m->joint_q_start[i] - a->m->joint_q_start[0], ds = a->m->joint_qd_start[i] - a->m->joint_qd_start[0];
        if (type == 0 || type == 1) { real qd_new = qd[ds] + qdd[ds] * dt; qdn[ds] = qd_new; qn[cs] = q[cs] + qd_new * dt; }
        if (type == 2) {
            v3 wn = vadd(V(qd[ds], qd[ds + 1], qd[ds + 2]), vmul(V(qdd[ds], qdd[ds + 1], qdd[ds + 2]), dt));
            q4 r = Qn(q[cs], q[cs + 1], q[cs + 2], q[cs + 3]);
            q4 dr = qmul(Qn(wn.x, wn.y, wn.z, 0), r);
            q4 rn = qnormalize(Qn(r.x + dr.x * (real)0.5 * dt, r.y + dr.y * (real)0.5 * dt, r.z + dr.z * (real)0.5 * dt, r.w + dr.w * (real)0.5 * dt));
            qn[cs] = rn.x; qn[cs + 1] = rn.y; qn[cs + 2] = rn.z; qn[cs + 3] = rn.w;
            qdn[ds] = wn.x; qdn[ds + 1] = wn.y; qdn[ds + 2] = wn.z;
        }
        if (type == 4) {
            v3 w_s = vadd(V(qd[ds], qd[ds + 1], qd[ds + 2]), vmul(V(qdd[ds], qdd[ds + 1], qdd[ds + 2]), dt));
            v3 v_s = vadd(V(qd[ds + 3], qd[ds + 4], qd[ds + 5]), vmul(V(qdd[ds + 3], qdd[ds + 4], qdd[ds + 5]), dt));
            v3 p_s = V(q[cs], q[cs + 1], q[cs + 2]);
            v3 dpdt = vadd(v_s, vcross(w_s, p_s));
            q4 r = Qn(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
            q4 dr = qmul(Qn(w_s.x, w_s.y, w_s.z, 0), r);
            v3 pn = vadd(p_s, vmul(dpdt, dt));
            q4 rn = qnormalize(Qn(r.x + dr.x * (real)0.5 * dt, r.y + dr.y * (real)0.5 * dt, r.z + dr.z * (real)0.5 * dt, r.w + dr.w * (real)0.5 * dt));
            qn[cs] = pn.x; qn[cs + 1] = pn.y; qn[cs + 2] = pn.z;
            qn[cs + 3] = rn.x; qn[cs + 4] = rn.y; qn[cs + 5] = rn.z; qn[cs + 6] = rn.w;
            qdn[ds] = w_s.x; qdn[ds + 1] = w_s.y; qdn[ds + 2] = w_s.z; qdn[ds + 3] = v_s.x; qdn[ds + 4] = v_s.y; qdn[ds + 5] = v_s.z;
        }
    }
}

static Work work_alloc(const Art* a) {
    Work w; int L = a->L, D = a->D;
    w.X_sc = malloc(sizeof(xf) * L); w.X_sm = malloc(sizeof(xf) * L); w.S_s = malloc(sizeof(sv) * (D + 1));
    w.v_s = malloc(sizeof(sv) * L); w.a_s = malloc(sizeof(sv) * L); w.f_s = malloc(sizeof(sv) * L); w.ft_s = malloc(sizeof(sv) * L);
    w.I_s = malloc(sizeof(sm) * L); w.tau = calloc(D + 1, sizeof(real)); w.qdd = calloc(D + 1, sizeof(real));
    w.J = malloc(sizeof(real) * 36 * L * (D + 1)); w.Mm = malloc(sizeof(real) * 36 * L * L); w.P = malloc(sizeof(real) * 36 * L * (D + 1));
    w.H = malloc(sizeof(real) * (D * D + 1)); w.Lc = malloc(sizeof(real) * (D * D + 1));
    return w;
}
static void work_free(Work* w) {
    free(w->X_sc); free(w->X_sm); free(w->S_s); free(w->v_s); free(w->a_s); free(w->f_s); free(w->ft_s); free(w->I_s);
    free(w->tau); free(w->qdd); free(w->J); free(w->Mm); free(w->P); free(w->H); free(w->Lc);
}

/* SimulateFunc.forward / SemiImplicitIntegrator._simulate, sim.py:2097-2123, 2225-2601, for ONE environment */
static void env_step_one(const Art* a, Work* w, real* q, real* qd, const real* act, const real* musc,
                         double dt, int substeps, int mm_freq, real* traj /* [substeps, Q+D] or NULL */) {
    real sub_dt = (real)(float)(dt / (double)substeps);   /* python float -> fp32 kernel argument */
    real* qn = malloc(sizeof(real) * (a->Q + 1));
    real* qdn = malloc(sizeof(real) * (a->D + 1));
    for (int s = 0; s < substeps; ++s) {
        eval_rigid_fk(a, q, w);
        eval_rigid_id(a, qd, w);
        if (a->m->ground && a->C > 0) eval_rigid_contacts(a, w);
        if (a->M > 0) eval_muscles(a, musc, w);
        eval_rigid_tau(a, q, qd, act, w);
        if (s % mm_freq == 0) eval_mass_matrix(a, w);
        eval_solve(a, w);
        eval_integrate(a, q, qd, w->qdd, sub_dt, qn, qdn);
        memcpy(q, qn, sizeof(real) * a->Q);
        memcpy(qd, qdn, sizeof(real) * a->D);
        if (traj) { memcpy(traj + (size_t)s * (a->Q + a->D), q, sizeof(real) * a->Q); memcpy(traj + (size_t)s * (a->Q + a->D) + a->Q, qd, sizeof(real) * a->D); }
    }
    free(qn); free(qdn);
}

static Art make_art(const DfxModelDesc* m) {
    Art a; a.L = m->link_count; a.D = m->dof_count; a.Q = m->coord_count; a.C = m->contact_count; a.M = m->muscle_count; a.m = m;
    for (int k = 0; k < 3; ++k) a.g[k] = (real)m->gravity[k];
    return a;
}

/* Public entry points (double in/out regardless of REAL, so one ctypes signature serves both builds). */
int oracle_real_bytes(void) { return (int)sizeof(real); }

/* n environments; q [n*Q], qd [n*D], act [n*D], musc [n*M] -> q_out, qd_out; traj [n, substeps, Q+D] optional */
void oracle_step_forward(const DfxModelDesc* m, int n, int substeps, int mm_freq, double dt,
                         const double* q, const double* qd, const double* act, const double* musc,
                         double* q_out, double* qd_out, double* traj) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ract = malloc(sizeof(real) * (D + 1)); real* rm = malloc(sizeof(real) * (M + 1));
    real* rt = traj ? malloc(sizeof(real) * (size_t)substeps * (Q + D)) : NULL;
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) { rqd[i] = (real)qd[(size_t)e * D + i]; ract[i] = (real)act[(size_t)e * D + i]; }
        for (int i = 0; i < M; ++i) rm[i] = (real)musc[(size_t)e * M + i];
        env_step_one(&a, &w, rq, rqd, ract, rm, dt, substeps, mm_freq, rt);
        for (int i = 0; i < Q; ++i) q_out[(size_t)e * Q + i] = (double)RE(rq[i]);
        for (int i = 0; i < D; ++i) qd_out[(size_t)e * D + i] = (double)RE(rqd[i]);
        if (traj) for (size_t i = 0; i < (size_t)substeps * (Q + D); ++i) traj[(size_t)e * substeps * (Q + D) + i] = (double)RE(rt[i]);
    }
    free(rq); free(rqd); free(ract); free(rm); free(rt);
    work_free(&w);
}

/* Central finite differences of  loss = gq_out . q' + gqd_out . qd'  w.r.t. every input of ONE environment.
 * Meaningful in the REAL=double build.  grads: gq [Q], gqd [D], gact [D], gmusc [M]. */
static double loss_of(const Art* a, Work* w, const double* q, const double* qd, const double* act, const double* musc,
                      const double* gq_out, const double* gqd_out, double dt, int substeps, int mm_freq) {
    int Q = a->Q, D = a->D, M = a->M;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ract = malloc(sizeof(real) * (D + 1)); real* rm = malloc(sizeof(real) * (M + 1));
    for (int i = 0; i < Q; ++i) rq[i] = (real)q[i];
    for (int i = 0; i < D; ++i) { rqd[i] = (real)qd[i]; ract[i] = (real)act[i]; }
    for (int i = 0; i < M; ++i) rm[i] = (real)musc[i];
    env_step_one(a, w, rq, rqd, ract, rm, dt, substeps, mm_freq, NULL);
    double loss = 0;
    for (int i = 0; i < Q; ++i) loss += gq_out[i] * (double)RE(rq[i]);
    for (int i = 0; i < D; ++i) loss += gqd_out[i] * (double)RE(rqd[i]);
    free(rq); free(rqd); free(ract); free(rm);
    return loss;
}
void oracle_fd_gradient(const DfxModelDesc* m, int substeps, int mm_freq, double dt, double eps,
                        const double* q, const double* qd, const double* act, const double* musc,
                        const double* gq_out, const double* gqd_out,
                        double* gq, double* gqd, double* gact, double* gmusc) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int sizes[4] = {a.Q, a.D, a.D, a.M};
    const double* base[4] = {q, qd, act, musc};
    double* outs[4] = {gq, gqd, gact, gmusc};
    for (int g = 0; g < 4; ++g) {
        if (!outs[g]) continue;
        double* tmp = malloc(sizeof(double) * (sizes[g] + 1));
        memcpy(tmp, base[g], sizeof(double) * sizes[g]);
        for (int i = 0; i < sizes[g]; ++i) {
            const double* args[4] = {q, qd, act, musc};
            args[g] = tmp;
            double h = eps * (1.0 + fabs(base[g][i]));
            tmp[i] = base[g][i] + h;
            double lp = loss_of(&a, &w, args[0], args[1], args[2], args[3], gq_out, gqd_out, dt, substeps, mm_freq);
            tmp[i] = base[g][i] - h;
            double lm = loss_of(&a, &w, args[0], args[1], args[2], args[3], gq_out, gqd_out, dt, substeps, mm_freq);
            tmp[i] = base[g][i];
            outs[g][i] = (lp - lm) / (2.0 * h);
        }
        free(tmp);
    }
    work_free(&w);
}

/* Per environment: a 64-bit FNV-1a hash of the sequence of branch decisions of the contact and joint-limit model over all
 * substeps (contact penetrates, vn < 0, friction cap viscous / Coulomb, q < lower, q > upper) and the count of each
 * (counts [n, BR_COUNT] in the order of the BR_ enum).  The f32 and f64 builds decide on their own rounding. */
void oracle_branch_signature(const DfxModelDesc* m, int n, int substeps, int mm_freq, double dt,
                             const double* q, const double* qd, const double* act, const double* musc,
                             uint64_t* hash, int64_t* counts) {
    int Q = m->coord_count, D = m->dof_count, M = m->muscle_count;
    double* q_out = malloc(sizeof(double) * (Q + 1)); double* qd_out = malloc(sizeof(double) * (D + 1));
    for (int e = 0; e < n; ++e) {
        memset(&g_branch, 0, sizeof g_branch);
        g_branch.on = 1; g_branch.hash = 14695981039346656037ull;
        oracle_step_forward(m, 1, substeps, mm_freq, dt, q + (size_t)e * Q, qd + (size_t)e * D, act + (size_t)e * D,
                            musc + (size_t)e * M, q_out, qd_out, NULL);
        hash[e] = g_branch.hash;
        for (int k = 0; k < BR_COUNT; ++k) counts[(size_t)e * BR_COUNT + k] = g_branch.counts[k];
    }
    g_branch.on = 0;
    free(q_out); free(qd_out);
}

#ifdef ORACLE_COMPLEX
/* Complex-step derivative of  loss = gq_out . q' + gqd_out . qd'  w.r.t. every input of ONE environment (same signature
 * as oracle_fd_gradient; h is the imaginary step, 1e-30 when h <= 0).  One complex forward per input component:
 * dloss/dx_i = Im loss(x + i h e_i) / h.  Nothing is subtracted, so the result is exact to rounding for the branch the
 * real part takes -- the quantity a reverse-mode adjoint of the same forward computes. */
void oracle_exact_gradient(const DfxModelDesc* m, int substeps, int mm_freq, double dt, double h,
                           const double* q, const double* qd, const double* act, const double* musc,
                           const double* gq_out, const double* gqd_out,
                           double* gq, double* gqd, double* gact, double* gmusc) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M;
    int sizes[4] = {Q, D, D, M};
    const double* base[4] = {q, qd, act, musc};
    double* outs[4] = {gq, gqd, gact, gmusc};
    real* in[4];
    for (int g = 0; g < 4; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 4; ++g) {
        if (!outs[g]) continue;
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            env_step_one(&a, &w, rq, rqd, in[2], in[3], dt, substeps, mm_freq, NULL);
            double s = 0;
            for (int k = 0; k < Q; ++k) s += gq_out[k] * cimag(rq[k]);
            for (int k = 0; k < D; ++k) s += gqd_out[k] * cimag(rqd[k]);
            outs[g][i] = s / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 4; ++g) free(in[g]);
    free(rq); free(rqd);
    work_free(&w);
}
#endif
