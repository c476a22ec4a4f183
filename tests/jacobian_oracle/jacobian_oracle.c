/* jacobian_oracle.c -- the Jacobian state (include/dfx.h dfx_jacobian_state_forward) in the C restatement of the step, TEST
 * INFRASTRUCTURE ONLY (tests/test_jacobian_state_emu.py, tests/test_gpu_jacobian_state.py).
 *
 * Takes the link oracle as it is (tests/link_oracle/link_oracle.c, which includes the wrench oracle and oracle/dflex_oracle.c;
 * every function unchanged) and adds:
 *   oracle_jacobian_state            J [L*6*D] and body_a_s [L*6] of (q, qd): eval_rigid_fk + eval_rigid_id, then J by the
 *                                    spatial_jacobian loop that opens eval_mass_matrix (restated here);
 *   oracle_jacobian_state_gradient   the complex-step gradient of sum(g_J . J + g_a . body_a_s) with respect to (q, qd);
 *   oracle_controlled_rollout        T env-steps, each under the actuation act_t = u_t + sum_l J_l^T (W_l + kappa body_a_s_l) of the
 *                                    state it starts from (a task-space wrench W [L*6] plus a bias-acceleration feedback);
 *   oracle_controlled_rollout_gradient   its complex-step gradient of sum(g_q . q_T + g_qd . qd_T) with respect to (q, qd, u).
 * Built (tests/jacobian_util.py) as the oracle is: REAL = double, or REAL = double _Complex for the complex step. */
#include "../link_oracle/link_oracle.c"

/* one environment: J [L*6*D] (row 6 i + r, column d) and body_a_s [L*6] */
static void jacobian_state_one(const Art* a, Work* w, const real* q, const real* qd, real* J, real* as) {
    int L = a->L, D = a->D;
    link_kinematics(a, q, qd, w);
    for (int k = 0; k < L * 6 * D; ++k) J[k] = 0;
    for (int i = 0; i < L; ++i) {      /* spatial_jacobian, spatial.h:691-738 (the loop of eval_mass_matrix) */
        int j = i;
        while (j != -1) {
            int d0 = a->m->joint_qd_start[j] - a->m->joint_qd_start[0], d1 = a->m->joint_qd_start[j + 1] - a->m->joint_qd_start[0];
            for (int col = d0; col < d1; ++col)
                for (int r = 0; r < 6; ++r) J[(i * 6 + r) * D + col] = sv_get(w->S_s[col], r);
            j = a->m->joint_parent[j];
        }
        put_sv(as + i * 6, w->a_s[i]);
    }
}

/* q [n*Q], qd [n*D] -> J [n*L*6*D], body_a_s [n*L*6] */
void oracle_jacobian_state(const DfxModelDesc* m, int n, const double* q, const double* qd, double* J, double* body_a_s) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rJ = malloc(sizeof(real) * (L * 6 * D + 1)); real* ra = malloc(sizeof(real) * L * 6);
    for (int e = 0; e < n; ++e) {
        for (int i = 0; i < Q; ++i) rq[i] = (real)q[(size_t)e * Q + i];
        for (int i = 0; i < D; ++i) rqd[i] = (real)qd[(size_t)e * D + i];
        jacobian_state_one(&a, &w, rq, rqd, rJ, ra);
        for (int i = 0; i < L * 6 * D; ++i) J[(size_t)e * L * 6 * D + i] = (double)RE(rJ[i]);
        for (int i = 0; i < L * 6; ++i) body_a_s[(size_t)e * L * 6 + i] = (double)RE(ra[i]);
    }
    free(rq); free(rqd); free(rJ); free(ra);
    work_free(&w);
}

/* T env-steps from (q, qd) (overwritten with the end state), actuation act_t = u_t + J(q_t)^T (W + kappa body_a_s(q_t, qd_t)) */
static void controlled_rollout_one(const Art* a, Work* w, real* q, real* qd, const real* u, const real* musc, const real* W, real kappa,
                                   int T, double dt, int substeps, int mm_freq) {
    int L = a->L, D = a->D;
    real* J = malloc(sizeof(real) * (L * 6 * D + 1)); real* as = malloc(sizeof(real) * L * 6); real* act = malloc(sizeof(real) * (D + 1));
    for (int t = 0; t < T; ++t) {
        jacobian_state_one(a, w, q, qd, J, as);
        for (int d = 0; d < D; ++d) {
            real s = u[(size_t)t * D + d];
            for (int k = 0; k < L * 6; ++k) s += J[k * D + d] * (W[k] + kappa * as[k]);
            act[d] = s;
        }
        env_step_one(a, w, q, qd, act, a->M > 0 ? musc + (size_t)t * a->M : musc, dt, substeps, mm_freq, NULL);
    }
    free(J); free(as); free(act);
}

/* one environment: the end state (q_T [Q], qd_T [D]) of the controlled rollout; u [T*D], W [L*6]; musc NULL without muscles */
void oracle_controlled_rollout(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double kappa, const double* q,
                               const double* qd, const double* u, const double* musc, const double* W, double* q_out, double* qd_out) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* ru = malloc(sizeof(real) * (T * D + 1)); real* rm = malloc(sizeof(real) * (T * M + 1)); real* rW = malloc(sizeof(real) * L * 6);
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < T * D; ++i) ru[i] = u[i];
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    for (int i = 0; i < L * 6; ++i) rW[i] = W[i];
    controlled_rollout_one(&a, &w, rq, rqd, ru, rm, rW, (real)kappa, T, dt, substeps, mm_freq);
    for (int i = 0; i < Q; ++i) q_out[i] = (double)RE(rq[i]);
    for (int i = 0; i < D; ++i) qd_out[i] = (double)RE(rqd[i]);
    free(rq); free(rqd); free(ru); free(rm); free(rW);
    work_free(&w);
}

#ifdef ORACLE_COMPLEX
/* one environment: gq [Q], gqd [D], gu [T*D] of sum(g_q . q_T + g_qd . qd_T) of the controlled rollout */
void oracle_controlled_rollout_gradient(const DfxModelDesc* m, int T, int substeps, int mm_freq, double dt, double kappa, double h,
                                        const double* q, const double* qd, const double* u, const double* musc, const double* W,
                                        const double* g_q, const double* g_qd, double* gq, double* gqd, double* gu) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, M = a.M, L = a.L;
    int sizes[3] = {Q, D, T * D};
    const double* base[3] = {q, qd, u};
    double* outs[3] = {gq, gqd, gu};
    real* in[3];
    for (int g = 0; g < 3; ++g) {
        in[g] = malloc(sizeof(real) * (sizes[g] + 1));
        for (int i = 0; i < sizes[g]; ++i) in[g][i] = base[g][i];
    }
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rm = malloc(sizeof(real) * (T * M + 1)); real* rW = malloc(sizeof(real) * L * 6);
    for (int i = 0; i < T * M; ++i) rm[i] = musc[i];
    for (int i = 0; i < L * 6; ++i) rW[i] = W[i];
    if (!(h > 0)) h = 1e-30;
    for (int g = 0; g < 3; ++g) {
        for (int i = 0; i < sizes[g]; ++i) {
            in[g][i] = CMPLX(base[g][i], h);
            memcpy(rq, in[0], sizeof(real) * Q); memcpy(rqd, in[1], sizeof(real) * D);
            controlled_rollout_one(&a, &w, rq, rqd, in[2], rm, rW, (real)kappa, T, dt, substeps, mm_freq);
            double s = 0;
            for (int k = 0; k < Q; ++k) s += g_q[k] * cimag(rq[k]);
            for (int k = 0; k < D; ++k) s += g_qd[k] * cimag(rqd[k]);
            outs[g][i] = s / h;
            in[g][i] = base[g][i];
        }
    }
    for (int g = 0; g < 3; ++g) free(in[g]);
    free(rq); free(rqd); free(rm); free(rW);
    work_free(&w);
}

static double jacobian_cotangent_dot(int n_J, int n_a, const real* J, const real* as, const double* g_J, const double* g_a) {
    double s = 0;
    if (g_J) for (int i = 0; i < n_J; ++i) s += g_J[i] * cimag(J[i]);
    if (g_a) for (int i = 0; i < n_a; ++i) s += g_a[i] * cimag(as[i]);
    return s;
}

/* one environment: gq [Q], gqd [D] of sum(g_J . J + g_a . body_a_s) (a NULL cotangent is 0), one complex evaluation per input */
void oracle_jacobian_state_gradient(const DfxModelDesc* m, double h, const double* q, const double* qd, const double* g_J,
                                    const double* g_a, double* gq, double* gqd) {
    Art a = make_art(m);
    Work w = work_alloc(&a);
    int Q = a.Q, D = a.D, L = a.L;
    real* rq = malloc(sizeof(real) * (Q + 1)); real* rqd = malloc(sizeof(real) * (D + 1));
    real* rJ = malloc(sizeof(real) * (L * 6 * D + 1)); real* ra = malloc(sizeof(real) * L * 6);
    if (!(h > 0)) h = 1e-30;
    for (int i = 0; i < Q; ++i) rq[i] = q[i];
    for (int i = 0; i < D; ++i) rqd[i] = qd[i];
    for (int i = 0; i < Q; ++i) {
        rq[i] = CMPLX(q[i], h);
        jacobian_state_one(&a, &w, rq, rqd, rJ, ra);
        gq[i] = jacobian_cotangent_dot(L * 6 * D, L * 6, rJ, ra, g_J, g_a) / h;
        rq[i] = q[i];
    }
    for (int i = 0; i < D; ++i) {
        rqd[i] = CMPLX(qd[i], h);
        jacobian_state_one(&a, &w, rq, rqd, rJ, ra);
        gqd[i] = jacobian_cotangent_dot(L * 6 * D, L * 6, rJ, ra, g_J, g_a) / h;
        rqd[i] = qd[i];
    }
    free(rq); free(rqd); free(rJ); free(ra);
    work_free(&w);
}
#endif
