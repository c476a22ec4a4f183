/* dynamics_oracle.c -- the dynamics state (include/dfx.h dfx_dynamics_state_forward) in the C restatement of the step, TEST
 * INFRASTRUCTURE ONLY (tests/test_dynamics_state_emu.py, tests/test_gpu_dynamics_state.py).
 *
 * Takes the wrench oracle as it is (tests/wrench_oracle/wrench_oracle.c, which includes oracle/dflex_oracle.c; every function
 * unchanged) and adds:
 *   oracle_dynamics_state             the first substep of an env-step up to its solve: eval_rigid_fk, eval_rigid_id,
 *                                     apply_wrench, eval_rigid_contacts, eval_muscles, eval_rigid_tau, eval_mass_matrix (w->H, no
 *                                     armature), eval_solve -> (qdd, tau, H);
 *   oracle_dynamics_state_gradient    the complex-step gradient of sum(g . outputs) with respect to (q, qd, act, musc, f_ext), one
 *                                     environment;
 *   oracle_dynamics_rollout           T env-steps (the oracle's own step), then the dynamics state of the end state, and the end
 *                                     state itself;
 *   oracle_dynamics_rollout_gradient  its complex-step gradient with respect to (q, qd, act [(T+1)*D]).
 * Built (tests/dynamics_util.py) as the oracle is: REAL = double, or REAL = double _Complex for the complex step. */
#include "../wrench_oracle/wrench_oracle.c"

/* o = [qdd (D) | tau (D) | H (D*D)] of one environment; fext [L*6] (zero: no wrench), musc [M] */
static void dynamics_state_of(const Art* a, Work* w, const real* q, const real* qd, const real* act, const real* musc,
                              const real* fext, real* o) {
    int D = a->D;
    eval_rigid_fk(a, q, w);
    eval_rigid_id(a, qd, w);
    apply_wrench(a, fext, w);
    if (a->m->ground && a->C > 0) eval_rigid_contacts(a, w);
    if (a->M > 0) eval_muscles(a, musc, w);
    eval_rigid_tau(a, q, qd, act, w);
    eval_mass_matrix(a, w);
    eval_solve(a, w);
    for (int i = 0; i < D; ++i) { o[i] = w->qdd[i]; o[D + i] = w->tau[i]; }
    for (int i = 0; i < D * D; ++i) o[2 * D + i] = w->H[i];
}

/* n environments: q [n*Q], qd [n*D], act [n*D], musc [n*M], fext [n*L*6] -> qdd [n*D], tau [n*D], H [n*D*D] */
void oracle_dynamics_state(const DfxModelDesc* m, int n, const double* q, const double* qd, const double* act, const double* musc,
                           const double* fext, double* qdd, double* tau, double* H) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ra = malloc(sizeof(real) * (D + 1)); real* rm = malloc(sizeof(real) * (M + 1));
    real* rf = malloc(sizeof(real) * (L * 6 + 1)); real* o = malloc(sizeof(real) * (2 * D + D * D + 1));
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) { rqd[i] = (real)qd[(size_t)e * D + i]; ra[i] = (real)act[(size_t)e * D + i]; }
        for (int i = 0; i < M; ++i) rm[i] = (real)musc[(size_t)e * M + i];
        for (int i = 0; i < L * 6; ++i) rf[i] = (real)fext[(size_t)e * L * 6 + i];
        dynamics_state_of(&a, &w, rq, rqd, ra, rm, rf, o);
        for (int i = 0; i < D; ++i) { qdd[(size_t)e * D + i] = (double)RE(o[i]); tau[(size_t)e * D + i] = (double)RE(o[D + i]); }
        for (int i = 0; i < D * D; ++i) H[(size_t)e * D * D + i] = (double)RE(o[2 * D + i]);
    }
    free(rq); free(rqd); free(ra); free(rm); free(rf); free(o);
    work_free(&w);
}

/* T env-steps from (q, qd) with act [T*D], musc [T*M], then o = [dynamics state (2D + D*D) under act [T] / musc [T] | q (Q) | qd (D)]
 * of the end state; act and musc hold T + 1 rows.  q, qd are overwritten. */
static void dynamics_rollout_one(const Art* a, Work* w, real* q, real* qd, const real* act, const real* musc, const real* fext, int T,
                                 double dt, int substeps, int mm_freq, real* o) {
    int D = a->D, M = a->M;
    for (int t = 0; t < T; ++t)
        env_step_one(a, w, q, qd, act + (size_t)t * D, musc + (size_t)t * M, dt, substeps, mm_freq, NULL);
    dynamics_state_of(a, w, q, qd, act + (size_t)T * D, musc + (size_t)T * M, fext, o);
    int k = 2 * D + D * D;
    for (int i = 0; i < a->Q; ++i) o[k + i] = q[i];
    for (int i = 0; i < D; ++i) o[k + a->Q + i] = qd[i];
}

/* one environment: out [2D + D*D + Q + D] */
void oracle_dynamics_rollout(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, const double* q, const double* qd,
                             const double* act, const double* musc, double* out) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L, K = 2 * D + D * D + Q + D;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ra = malloc(sizeof(real) * ((T + 1) * D + 1)); real* rm = malloc(sizeof(real) * ((T + 1) * M + 1));
    real* rf = calloc(L * 6 + 1, sizeof(real)); real* o = malloc(sizeof(real) * (K + 1));
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < (T + 1) * D; ++i) ra[i] = act[i];
    for (int i = 0; i < (T + 1) * M; ++i) rm[i] = musc[i];
    dynamics_rollout_one(&a, &w, rq, rqd, ra, rm, rf, T, dt, substeps, mm_freq, o);
    for (int i = 0; i < K; ++i) out[i] = (double)RE(o[i]);
    free(rq); free(rqd); free(ra); free(rm); free(rf); free(o);
    work_free(&w);
}

#ifdef ORACLE_COMPLEX
/* one environment: gq [Q], gqd [D], gact [D], gmusc [M], gfext [L*6] of sum(g_qdd . qdd + g_tau . tau + g_H . H) (a NULL
 * cotangent is 0; a NULL output is skipped), one complex evaluation per input component */
void oracle_dynamics_state_gradient(const DfxModelDesc* m, double h, const double* q, const double* qd, const double* act,
                                    const double* musc, const double* fext, const double* g_qdd, const double* g_tau,
                                    const double* g_H, double* gq, double* gqd, double* gact, double* gmusc, double* gfext) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int D = a.D;
    int sizes[5] = {a.Q, D, D, a.M, a.L * 6};
    const double* base[5] = {q, qd, act, musc, fext};
    double* outs[5] = {gq, gqd, gact, gmusc, gfext};
    real* in[5];
    for (int g = 0; g < 5; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* o = malloc(sizeof(real) * (2 * D + D * D + 1));
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 5; ++g) {
        if (!outs[g]) continue;
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            dynamics_state_of(&a, &w, in[0], in[1], in[2], in[3], in[4], o);
            double s = 0;
            for (int k = 0; k < D; ++k) {
                if (g_qdd) s += g_qdd[k] * cimag(o[k]);
                if (g_tau) s += g_tau[k] * cimag(o[D + k]);
            }
            if (g_H) for (int k = 0; k < D * D; ++k) s += g_H[k] * cimag(o[2 * D + k]);
            outs[g][i] = s / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 5; ++g) free(in[g]);
    free(o);
    work_free(&w);
}

/* one environment: gq [Q], gqd [D], gact [(T+1)*D] of sum(g . out) of oracle_dynamics_rollout, g [2D + D*D + Q + D] */
void oracle_dynamics_rollout_gradient(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double h,
                                      const double* q, const double* qd, const double* act, const double* musc, const double* g,
                                      double* gq, double* gqd, double* gact) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L, K = 2 * D + D * D + Q + D;
    int sizes[3] = {Q, D, (T + 1) * D};
    const double* base[3] = {q, qd, act};
    double* outs[3] = {gq, gqd, gact};
    real* in[3];
    for (int k = 0; k < 3; ++k) {
        in[k] = malloc(sizeof(real) * (sizes[k] + 1));
        for (int i = 0; i < sizes[k]; ++i) in[k][i] = base[k][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rm = malloc(sizeof(real) * ((T + 1) * M + 1)); real* rf = calloc(L * 6 + 1, sizeof(real));
    real* o = malloc(sizeof(real) * (K + 1));
    for (int i = 0; i < (T + 1) * M; ++i) rm[i] = musc[i];
    if (!(h > 0)) h = 1e-30;
    for (int k = 0; k < 3; ++k) {
        if (!outs[k]) continue;
        for (int i = 0; i < sizes[k]; ++i) {
            in[k][i] = CMPLX(base[k][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            dynamics_rollout_one(&a, &w, rq, rqd, in[2], rm, rf, T, dt, substeps, mm_freq, o);
            double s = 0;
            for (int j = 0; j < K; ++j) s += g[j] * cimag(o[j]);
            outs[k][i] = s / h;
            in[k][i] = base[k][i];
        }
    }
    for (int k = 0; k < 3; ++k) free(in[k]);
    free(rq); free(rqd); free(rm); free(rf); free(o);
    work_free(&w);
}
#endif
