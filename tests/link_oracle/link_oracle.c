/* link_oracle.c -- the link state (include/dfx.h dfx_link_state_forward) in the C restatement of the step, TEST INFRASTRUCTURE
 * ONLY (tests/test_link_state_emu.py, tests/test_gpu_link_state.py).
 *
 * Takes the wrench oracle as it is (tests/wrench_oracle/wrench_oracle.c, which includes oracle/dflex_oracle.c; every function
 * unchanged) and adds:
 *   oracle_link_state            X_sc, X_sm (eval_rigid_fk) and v_s (eval_rigid_id) of (q, qd), reference State layouts;
 *   oracle_link_state_gradient   the complex-step gradient of sum(g . outputs) with respect to (q, qd), one environment;
 *   oracle_tether_rollout        T env-steps, each with the tether wrench f_ext = (0, k (target - X_sm.p)) formed from the state it
 *                                starts from, then the link state of the end state;
 *   oracle_tether_rollout_gradient   its complex-step gradient with respect to (q, qd, act [T*D]).
 * Built (tests/link_util.py) as the oracle is: REAL = double, or REAL = double _Complex for the complex step. */
#include "../wrench_oracle/wrench_oracle.c"

static void link_kinematics(const Art* a, const real* q, const real* qd, Work* w) {
    eval_rigid_fk(a, q, w);
    eval_rigid_id(a, qd, w);
}

static void put_xf(real* o, xf t) { o[0] = t.p.x; o[1] = t.p.y; o[2] = t.p.z; o[3] = t.q.x; o[4] = t.q.y; o[5] = t.q.z; o[6] = t.q.w; }
static void put_sv(real* o, sv v) { o[0] = v.w.x; o[1] = v.w.y; o[2] = v.w.z; o[3] = v.v.x; o[4] = v.v.y; o[5] = v.v.z; }

/* the link state of one environment as [L*7], [L*7], [L*6] reals */
static void link_state_one(const Art* a, Work* w, const real* q, const real* qd, real* Xsc, real* Xsm, real* v) {
    link_kinematics(a, q, qd, w);
    for (int i = 0; i < a->L; ++i) {
        put_xf(Xsc + i * 7, w->X_sc[i]);
        put_xf(Xsm + i * 7, w->X_sm[i]);
        put_sv(v + i * 6, w->v_s[i]);
    }
}

/* q [n*Q], qd [n*D] -> X_sc, X_sm [n*L*7], v_s [n*L*6] */
void oracle_link_state(const DfxModelDesc* m, int n, const double* q, const double* qd, double* X_sc, double* X_sm, double* v_s) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* o = malloc(sizeof(real) * L * 20);
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) rqd[i] = (real)qd[(size_t)e * D + i];
        link_state_one(&a, &w, rq, rqd, o, o + L * 7, o + L * 14);
        for (int i = 0; i < L * 7; ++i) { X_sc[(size_t)e * L * 7 + i] = (double)RE(o[i]); X_sm[(size_t)e * L * 7 + i] = (double)RE(o[L * 7 + i]); }
        for (int i = 0; i < L * 6; ++i) v_s[(size_t)e * L * 6 + i] = (double)RE(o[L * 14 + i]);
    }
    free(rq); free(rqd); free(o);
    work_free(&w);
}

/* T env-steps from (q, qd) with act [T*D], musc [T*M] (M > 0), each under the tether wrench (0, k (target_i - X_sm[i].p)) of the
 * state it starts from, then the link state of the end state into o = [X_sc | X_sm | v] (L * 20 reals).  q, qd are overwritten. */
static void tether_rollout_one(const Art* a, Work* w, real* q, real* qd, const real* act, const real* musc, const real* target,
                               real k, int T, double dt, int substeps, int mm_freq, real* o) {
    int L = a->L;
    real* f = malloc(sizeof(real) * L * 6);
    for (int t = 0; t < T; ++t) {
        eval_rigid_fk(a, q, w);
        for (int i = 0; i < L; ++i) {
            f[i * 6] = 0; f[i * 6 + 1] = 0; f[i * 6 + 2] = 0;
            f[i * 6 + 3] = k * (target[i * 3] - w->X_sm[i].p.x);
            f[i * 6 + 4] = k * (target[i * 3 + 1] - w->X_sm[i].p.y);
            f[i * 6 + 5] = k * (target[i * 3 + 2] - w->X_sm[i].p.z);
        }
        env_step_one_ext(a, w, q, qd, act + (size_t)t * a->D, a->M > 0 ? musc + (size_t)t * a->M : musc, f, dt, substeps, mm_freq);
    }
    link_state_one(a, w, q, qd, o, o + L * 7, o + L * 14);
    free(f);
}

/* one environment: the link state [L*20] (X_sc, X_sm, v) at the end of the tethered rollout; target [L*3]; musc NULL without muscles */
void oracle_tether_rollout(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double k,
                           const double* q, const double* qd, const double* act, const double* musc, const double* target, double* out) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ra = malloc(sizeof(real) * (T * D + 1)); real* rm = malloc(sizeof(real) * (T * M + 1));
    real* rt = calloc((size_t)L * 3, sizeof(real)); real* o = malloc(sizeof(real) * L * 20);
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < T * D; ++i) ra[i] = act[i];
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    for (int i = 0; i < L * 3; ++i) rt[i] = target[i];
    tether_rollout_one(&a, &w, rq, rqd, ra, rm, rt, (real)k, T, dt, substeps, mm_freq, o);
    for (int i = 0; i < L * 20; ++i) out[i] = (double)RE(o[i]);
    free(rq); free(rqd); free(ra); free(rm); free(rt); free(o);
    work_free(&w);
}

#ifdef ORACLE_COMPLEX
/* sum of g . o over the link state [L*20], imaginary part */
static double cotangent_dot(int L, const real* o, const double* g_X_sc, const double* g_X_sm, const double* g_v) {
    double s = 0;
    for (int i = 0; i < L * 7; ++i) {
        if (g_X_sc) s += g_X_sc[i] * cimag(o[i]);
        if (g_X_sm) s += g_X_sm[i] * cimag(o[L * 7 + i]);
    }
    if (g_v) for (int i = 0; i < L * 6; ++i) s += g_v[i] * cimag(o[L * 14 + i]);
    return s;
}

/* one environment: gq [Q], gqd [D] of sum(g_X_sc . X_sc + g_X_sm . X_sm + g_v . v_s) (a NULL cotangent is 0), one complex
 * evaluation per input component */
void oracle_link_state_gradient(const DfxModelDesc* m, double h, const double* q, const double* qd,
                                const double* g_X_sc, const double* g_X_sm, const double* g_v, double* gq, double* gqd) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* o = malloc(sizeof(real) * L * 20);
    if (!(h > 0)) h = 1e-30;
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < Q; ++i) {
        rq[i] = CMPLX(q[i], h);
        link_state_one(&a, &w, rq, rqd, o, o + L * 7, o + L * 14);
        gq[i] = cotangent_dot(L, o, g_X_sc, g_X_sm, g_v) / h;
        rq[i] = q[i];
    }
    for (int i = 0; i < D; ++i) {
        rqd[i] = CMPLX(qd[i], h);
        link_state_one(&a, &w, rq, rqd, o, o + L * 7, o + L * 14);
        gqd[i] = cotangent_dot(L, o, g_X_sc, g_X_sm, g_v) / h;
        rqd[i] = qd[i];
    }
    free(rq); free(rqd); free(o);
    work_free(&w);
}

/* one environment: gq [Q], gqd [D], gact [T*D] of sum(g . link state at the end of the tethered rollout) */
void oracle_tether_rollout_gradient(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double k, double h,
                                    const double* q, const double* qd, const double* act, const double* musc, const double* target,
                                    const double* g_X_sc, const double* g_X_sm, const double* g_v,
                                    double* gq, double* gqd, double* gact) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    int sizes[3] = {Q, D, T * D};
    const double* base[3] = {q, qd, act};
    double* outs[3] = {gq, gqd, gact};
    real* in[3];
    for (int g = 0; g < 3; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rm = malloc(sizeof(real) * (T * M + 1)); real* rt = calloc((size_t)L * 3, sizeof(real));
    real* o = malloc(sizeof(real) * L * 20);
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    for (int i = 0; i < L * 3; ++i) rt[i] = target[i];
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 3; ++g) {
        if (!outs[g]) continue;
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            tether_rollout_one(&a, &w, rq, rqd, in[2], rm, rt, (real)k, T, dt, substeps, mm_freq, o);
            outs[g][i] = cotangent_dot(L, o, g_X_sc, g_X_sm, g_v) / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 3; ++g) free(in[g]);
    free(rq); free(rqd); free(rm); free(rt); free(o);
    work_free(&w);
}
#endif
