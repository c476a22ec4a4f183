/* contact_oracle.c -- the contact state (include/dfx.h dfx_contact_state_forward) in the C restatement of the step, TEST
 * INFRASTRUCTURE ONLY (tests/test_contact_state_emu.py, tests/test_gpu_contact_state.py).
 *
 * Takes the link oracle as it is (tests/link_oracle/link_oracle.c, which includes the wrench oracle and oracle/dflex_oracle.c;
 * every function unchanged) and adds:
 *   oracle_contact_state             per contact point, in the Model's order, the force the ground exerts on the link and the
 *                                    point's height above the plane; per link, (tau, F) of its points about its centre of mass;
 *   oracle_contact_state_gradient    the complex-step gradient of sum(g . outputs) with respect to (q, qd), one environment;
 *   oracle_contact_rollout           T env-steps (the oracle's own step), then the contact state of the end state;
 *   oracle_contact_rollout_gradient  its complex-step gradient with respect to (q, qd, act [T*D]).
 * Built (tests/contact_util.py) as the oracle is: REAL = double, or REAL = double _Complex for the complex step. */
#include "../link_oracle/link_oracle.c"

/* The contact state of one environment whose kinematics are in w: f [C*3], height [C], body [L*6] (tau, F).  Per point, the
 * restatement of eval_rigid_contacts_art sim.py:1137-1206 (as eval_rigid_contacts above): the reference ADDS f_total to body_f_s
 * (sim.py:1206), which eval_rigid_tau then subtracts from the joint forces, so the force the ground exerts is -f_total. */
static void contact_state_one(const Art* a, Work* w, real* f, real* height, real* body) {
    for (int i = 0; i < a->L * 6; ++i) body[i] = 0;
    for (int k = 0; k < a->C; ++k) {
        int b = a->m->contact_body0[k], mat = a->m->contact_material[k];
        real ke = (real)a->m->shape_materials[mat * 4 + 0], kd = (real)a->m->shape_materials[mat * 4 + 1];
        real kf = (real)a->m->shape_materials[mat * 4 + 2], mu = (real)a->m->shape_materials[mat * 4 + 3];
        v3 n = V(0, 1, 0);
        /* sim.py:1165-1177: the point in world, shifted by contact_dist along the normal; its velocity; c = dot(n, p) */
        v3 p = vsub(xf_point(w->X_sc[b], ld3(a->m->contact_point0 + k * 3)), vmul(n, (real)a->m->contact_dist[k]));
        v3 dpdt = vadd(w->v_s[b].v, vcross(w->v_s[b].w, p));
        real c = vdot(n, p);
        v3 force = V(0, 0, 0);
        if (a->m->ground && RLT(c, 0)) {
            /* sim.py:1179-1203: normal, damping and friction forces (min / step of adjoint.h:94-99) */
            real vn = vdot(n, dpdt);
            v3 vt = vsub(dpdt, vmul(n, vn));
            real fn = c * ke;
            real fd = (RLT(vn, 0) ? vn : (real)0) * kd * ((real)0 - c);
            real cap_a = kf * vlen(vt), cap_b = (real)0 - mu * c * ke;
            v3 ft = vmul(vnormalize(vt), RLT(cap_a, cap_b) ? cap_a : cap_b);
            v3 f_total = vadd(vmul(n, fn + fd), ft);
            force = vmul(f_total, (real)-1);
        }
        f[k * 3] = force.x; f[k * 3 + 1] = force.y; f[k * 3 + 2] = force.z;
        height[k] = c;
        v3 tau = vcross(vsub(p, w->X_sm[b].p), force);
        body[b * 6] += tau.x; body[b * 6 + 1] += tau.y; body[b * 6 + 2] += tau.z;
        body[b * 6 + 3] += force.x; body[b * 6 + 4] += force.y; body[b * 6 + 5] += force.z;
    }
}

/* the contact state of (q, qd) as one array o = [f (C*3) | height (C) | body (L*6)] */
static void contact_state_of(const Art* a, Work* w, const real* q, const real* qd, real* o) {
    link_kinematics(a, q, qd, w);
    contact_state_one(a, w, o, o + a->C * 3, o + a->C * 4);
}

/* q [n*Q], qd [n*D] -> contact_f [n*C*3], contact_height [n*C], body_f_contact [n*L*6] */
void oracle_contact_state(const DfxModelDesc* m, int n, const double* q, const double* qd, double* contact_f, double* contact_height,
                          double* body_f) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L, C = a.C;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* o = malloc(sizeof(real) * (C * 4 + L * 6 + 1));
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) rqd[i] = (real)qd[(size_t)e * D + i];
        contact_state_of(&a, &w, rq, rqd, o);
        for (int i = 0; i < C * 3; ++i) contact_f[(size_t)e * C * 3 + i] = (double)RE(o[i]);
        for (int i = 0; i < C; ++i) contact_height[(size_t)e * C + i] = (double)RE(o[C * 3 + i]);
        for (int i = 0; i < L * 6; ++i) body_f[(size_t)e * L * 6 + i] = (double)RE(o[C * 4 + i]);
    }
    free(rq); free(rqd); free(o);
    work_free(&w);
}

/* T env-steps from (q, qd) with act [T*D], musc [T*M] (M > 0), then the contact state of the end state into o.  q, qd are
 * overwritten. */
static void contact_rollout_one(const Art* a, Work* w, real* q, real* qd, const real* act, const real* musc, int T, double dt,
                                int substeps, int mm_freq, real* o) {
    for (int t = 0; t < T; ++t)
        env_step_one(a, w, q, qd, act + (size_t)t * a->D, a->M > 0 ? musc + (size_t)t * a->M : musc, dt, substeps, mm_freq, NULL);
    contact_state_of(a, w, q, qd, o);
}

/* one environment: the contact state [C*4 + L*6] at the end of T env-steps; musc NULL without muscles */
void oracle_contact_rollout(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, const double* q, const double* qd,
                            const double* act, const double* musc, double* out) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L, C = a.C;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ra = malloc(sizeof(real) * (T * D + 1)); real* rm = malloc(sizeof(real) * (T * M + 1));
    real* o = malloc(sizeof(real) * (C * 4 + L * 6 + 1));
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < T * D; ++i) ra[i] = act[i];
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    contact_rollout_one(&a, &w, rq, rqd, ra, rm, T, dt, substeps, mm_freq, o);
    for (int i = 0; i < C * 4 + L * 6; ++i) out[i] = (double)RE(o[i]);
    free(rq); free(rqd); free(ra); free(rm); free(o);
    work_free(&w);
}

#ifdef ORACLE_COMPLEX
/* sum of g . o over the contact state [C*4 + L*6], imaginary part */
static double contact_cotangent_dot(int C, int L, const real* o, const double* g_f, const double* g_h, const double* g_body) {
    double s = 0;
    if (g_f) for (int i = 0; i < C * 3; ++i) s += g_f[i] * cimag(o[i]);
    if (g_h) for (int i = 0; i < C; ++i) s += g_h[i] * cimag(o[C * 3 + i]);
    if (g_body) for (int i = 0; i < L * 6; ++i) s += g_body[i] * cimag(o[C * 4 + i]);
    return s;
}

/* one environment: gq [Q], gqd [D] of sum(g_f . contact_f + g_h . contact_height + g_body . body_f_contact) (a NULL cotangent is
 * 0), one complex evaluation per input component */
void oracle_contact_state_gradient(const DfxModelDesc* m, double h, const double* q, const double* qd, const double* g_f,
                                   const double* g_h, const double* g_body, double* gq, double* gqd) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L, C = a.C;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* o = malloc(sizeof(real) * (C * 4 + L * 6 + 1));
    if (!(h > 0)) h = 1e-30;
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < Q; ++i) {
        rq[i] = CMPLX(q[i], h);
        contact_state_of(&a, &w, rq, rqd, o);
        gq[i] = contact_cotangent_dot(C, L, o, g_f, g_h, g_body) / h;
        rq[i] = q[i];
    }
    for (int i = 0; i < D; ++i) {
        rqd[i] = CMPLX(qd[i], h);
        contact_state_of(&a, &w, rq, rqd, o);
        gqd[i] = contact_cotangent_dot(C, L, o, g_f, g_h, g_body) / h;
        rqd[i] = qd[i];
    }
    free(rq); free(rqd); free(o);
    work_free(&w);
}

/* one environment: gq [Q], gqd [D], gact [T*D] of sum(g . contact state at the end of the rollout) */
void oracle_contact_rollout_gradient(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double h,
                                     const double* q, const double* qd, const double* act, const double* musc,
                                     const double* g_f, const double* g_h, const double* g_body,
                                     double* gq, double* gqd, double* gact) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L, C = a.C;
    int sizes[3] = {Q, D, T * D};
    const double* base[3] = {q, qd, act};
    double* outs[3] = {gq, gqd, gact};
    real* in[3];
    for (int g = 0; g < 3; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rm = malloc(sizeof(real) * (T * M + 1));
    real* o = malloc(sizeof(real) * (C * 4 + L * 6 + 1));
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 3; ++g) {
        if (!outs[g]) continue;
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            contact_rollout_one(&a, &w, rq, rqd, in[2], rm, T, dt, substeps, mm_freq, o);
            outs[g][i] = contact_cotangent_dot(C, L, o, g_f, g_h, g_body) / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 3; ++g) free(in[g]);
    free(rq); free(rqd); free(rm); free(o);
    work_free(&w);
}
#endif
