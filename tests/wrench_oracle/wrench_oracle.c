/* wrench_oracle.c -- the C restatement of the step (oracle/dflex_oracle.c) with an external wrench per link, TEST
 * INFRASTRUCTURE ONLY (tests/test_external_wrench_emu.py, tests/test_gpu_external_wrench.py).
 *
 * The reference never applies State.body_f_ext_s, so there is nothing of its to restate: this file takes the oracle as it is
 * (included whole, every function unchanged) and applies include/dfx.h DfxExternalWrench's definition after its
 * eval_rigid_id -- body_f_s[i] -= (c x F + tau, F), c the link's centre of mass X_sm.p -- before the contact, muscle and tau
 * stages read body_f_s.  Built (tests/wrench_util.py) as the oracle is: REAL = double for the forward, REAL = double _Complex
 * for the complex-step gradient, with the oracle Makefile's flags. */
#include "../../oracle/dflex_oracle.c"

/* fext [L*6]: (tau, F) per link, world axes */
static void apply_wrench(const Art* a, const real* fext, Work* w) {
    for (int i = 0; i < a->L; ++i) {
        v3 tau = V(fext[i * 6], fext[i * 6 + 1], fext[i * 6 + 2]);
        v3 F = V(fext[i * 6 + 3], fext[i * 6 + 4], fext[i * 6 + 5]);
        w->f_s[i] = sv_sub(w->f_s[i], SVn(vadd(vcross(w->X_sm[i].p, F), tau), F));
    }
}

/* env_step_one (oracle/dflex_oracle.c) with the wrench held over the substeps */
static void env_step_one_ext(const Art* a, Work* w, real* q, real* qd, const real* act, const real* musc, const real* fext,
                             double dt, int substeps, int mm_freq) {
    real sub_dt = (real)(float)(dt / (double)substeps);
    real* qn = malloc(sizeof(real) * (a->Q + 1));
    real* qdn = malloc(sizeof(real) * (a->D + 1));
    for (int s = 0; s < substeps; ++s) {
        eval_rigid_fk(a, q, w);
        eval_rigid_id(a, qd, w);
        apply_wrench(a, fext, w);
        if (a->m->ground && a->C > 0) eval_rigid_contacts(a, w);
        if (a->M > 0) eval_muscles(a, musc, w);
        eval_rigid_tau(a, q, qd, act, w);
        if (s % mm_freq == 0) eval_mass_matrix(a, w);
        eval_solve(a, w);
        eval_integrate(a, q, qd, w->qdd, sub_dt, qn, qdn);
        memcpy(q, qn, sizeof(real) * a->Q);
        memcpy(qd, qdn, sizeof(real) * a->D);
    }
    free(qn); free(qdn);
}

/* oracle_step_forward with fext [n*L*6] */
void oracle_step_forward_ext(const DfxModelDesc* m, int n, int substeps, int mm_freq, double dt,
                             const double* q, const double* qd, const double* act, const double* musc, const double* fext,
                             double* q_out, double* qd_out) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ract = malloc(sizeof(real) * (D + 1)); real* rm = malloc(sizeof(real) * (M + 1));
    real* rf = malloc(sizeof(real) * L * 6);
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) { rqd[i] = (real)qd[(size_t)e * D + i]; ract[i] = (real)act[(size_t)e * D + i]; }
        for (int i = 0; i < M; ++i) rm[i] = (real)musc[(size_t)e * M + i];
        for (int i = 0; i < L * 6; ++i) rf[i] = (real)fext[(size_t)e * L * 6 + i];
        env_step_one_ext(&a, &w, rq, rqd, ract, rm, rf, dt, substeps, mm_freq);
        for (int i = 0; i < Q; ++i) q_out[(size_t)e * Q + i] = (double)RE(rq[i]);
        for (int i = 0; i < D; ++i) qd_out[(size_t)e * D + i] = (double)RE(rqd[i]);
    }
    free(rq); free(rqd); free(ract); free(rm); free(rf);
    work_free(&w);
}

#ifdef ORACLE_COMPLEX
/* oracle_exact_gradient with fext [L*6] for ONE environment and its block gfext [L*6]: the complex-step derivative of
 * loss = gq_out . q' + gqd_out . qd', one complex forward per input component */
void oracle_exact_gradient_ext(const DfxModelDesc* m, int substeps, int mm_freq, double dt, double h,
                               const double* q, const double* qd, const double* act, const double* musc, const double* fext,
                               const double* gq_out, const double* gqd_out,
                               double* gq, double* gqd, double* gact, double* gmusc, double* gfext) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M;
    int sizes[5] = {Q, D, D, M, a.L * 6};
    const double* base[5] = {q, qd, act, musc, fext};
    double* outs[5] = {gq, gqd, gact, gmusc, gfext};
    real* in[5];
    for (int g = 0; g < 5; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 5; ++g) {
        if (!outs[g]) continue;
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            env_step_one_ext(&a, &w, rq, rqd, in[2], in[3], in[4], dt, substeps, mm_freq);
            double s = 0;
            for (int k = 0; k < Q; ++k) s += gq_out[k] * cimag(rq[k]);
            for (int k = 0; k < D; ++k) s += gqd_out[k] * cimag(rqd[k]);
            outs[g][i] = s / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 5; ++g) free(in[g]);
    free(rq); free(rqd);
    work_free(&w);
}
#endif
