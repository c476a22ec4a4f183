// dfx_env_dev.h -- device code of the env layer around the simulation step (observation, reward, termination, masked
// re-initialisation and their adjoints; reference envs/ant.py:266-307, humanoid.py:314-368, snu_humanoid.py:378-432,
// hopper.py:170-268, cheetah.py:160-244, cartpole_swing_up.py:120-187), in two granularities:
//   * per ENVIRONMENT (walker_eval / planar_eval, their adjoints, *_transition_*_env): one call = one environment.  What the
//     stand-alone env kernels run (dfx_env.cu: one thread per environment, rows in global memory);
//   * per TILE (tile_transition_forward / _backward, at the end of the file): the transition of the E environments of a tile
//     kernel's CTA as the epilogue of the simulation launch / the prologue of the adjoint launch (dfx_env_step_*), staged in
//     the scratch tile -- the same per-environment functions, instantiated on strided shared-memory pointers (SP).
// Hence the template pointer types (QP / QDP: stepped state, OP: outputs, IP: adjoint inputs): global rows or scratch slots.
// Plain (not __restrict__) pointers on purpose: in the fused launch the rows were written by other threads of the same CTA
// (ordinary coherent accesses on either side of a CTA barrier, never the read-only path).
#pragma once

#include "../../include/dfx.h"
#include "dfx_math.h"

namespace dfx {

constexpr int kMaxObs = 96;     // largest walker observation: Humanoid 76 (checked on the host before the launch)

template <class QP, class QDP>
__device__ __forceinline__ void walker_features(const DfxWalkerParams& p, QP q, QDP qd,
                                                V3& pos, Q4& rot, V3& ang, V3& lin, V3& tt, float& tn, V3& tdir,
                                                Q4& tq, V3& up, V3& heading) {
    pos = ld3(q);
    rot = ld4(q + 3);
    ang = ld3(qd);
    lin = ld3(qd + 3) - cross(pos, ang);   // twist at the world origin -> velocity of the torso origin
    tt = V3{p.target[0] - pos.x, 0.0f, p.target[2] - pos.z};
    tn = fmaxf(sqrtf(dot(tt, tt)), 1e-9f);
    tdir = tt * (1.0f / tn);
    tq = qmul(rot, ld4(p.inv_start_rot));
    up = qrot(tq, ld3(p.basis_up));
    heading = qrot(tq, ld3(p.basis_heading));
}

__device__ __forceinline__ float height_reward(const DfxWalkerParams& p, float h, float* dh) {
    if (p.height_mode == 0) { *dh = 1.0f; return h - p.termination_height; }
    if (p.height_mode == 2) { *dh = 0.0f; return 0.0f; }
    // clip(h - (term + tol), -1, tol); r<0 -> -200 r^2 ; r>0 -> scale*r        (humanoid.py:348-351)
    float x = h - (p.termination_height + p.termination_tolerance);
    float r = fminf(fmaxf(x, -1.0f), p.termination_tolerance);
    float dr = (x >= -1.0f && x <= p.termination_tolerance) ? 1.0f : 0.0f;   // torch.clip: gradient 1 inside, incl. the ends
    if (r < 0.0f) { *dh = -400.0f * r * dr; return -200.0f * r * r; }
    if (r > 0.0f) { *dh = p.height_rew_scale * dr; return p.height_rew_scale * r; }
    *dh = dr;
    return r;
}

// observation (always) and, when want_reward, reward + reset flag of ONE environment; `progress` is the step
// counter AFTER this step.  `ae` == nullptr stands for all-zero actions (a freshly reset environment).
template <class QP, class QDP, class OP>
__device__ __forceinline__ void walker_eval(const DfxWalkerParams& p, QP qe, QDP qde,
                                            const float* ae, long long progress, bool want_reward,
                                            OP o, float* r_out, long long* rs_out) {
    V3 pos, ang, lin, tt, tdir, up, heading;
    Q4 rot, tq;
    float tn;
    walker_features(p, qe, qde, pos, rot, ang, lin, tt, tn, tdir, tq, up, heading);
    int k = 0;
    o[k++] = pos.y;
    o[k++] = rot.x; o[k++] = rot.y; o[k++] = rot.z; o[k++] = rot.w;
    o[k++] = lin.x; o[k++] = lin.y; o[k++] = lin.z;
    o[k++] = ang.x; o[k++] = ang.y; o[k++] = ang.z;
    bool bad = false;
    for (int i = 7; i < p.num_q; ++i) o[k++] = qe[i];
    for (int i = 6; i < p.num_qd; ++i) o[k++] = p.joint_vel_scale * qde[i];
    const float up_y = up.y, hproj = dot(heading, tdir);
    o[k++] = up_y;
    o[k++] = hproj;
    float act_sq = 0.0f, act_abs = 0.0f;
    for (int i = 0; i < p.num_act; ++i) {
        const float a = ae ? ae[i] : 0.0f;
        if (p.obs_has_actions) o[k++] = a;
        act_sq += a * a;
        act_abs += fabsf(a);
    }
    if (!want_reward) return;
    float dh;
    const float hr = height_reward(p, pos.y, &dh);
    float r = lin.x + 0.1f * up_y + hproj;
    if (p.height_mode != 2) r += hr;
    r += (p.action_penalty_abs ? act_abs : act_sq) * p.action_penalty;
    long long rs = 0;
    if (p.early_termination && pos.y < p.termination_height) rs = 1;
    if (progress > (long long)p.episode_length - 1) rs = 1;
    if (p.check_invalid) {
        for (int i = 0; i < p.num_q; ++i) bad |= !isfinite(qe[i]) || fabsf(qe[i]) > 1e6f;
        for (int i = 0; i < p.num_qd; ++i) bad |= !isfinite(qde[i]) || fabsf(qde[i]) > 1e6f;
        for (int i = 0; i < p.num_obs; ++i) bad |= !isfinite(o[i]);
        if (bad) { rs = 1; if (p.zero_reward_on_invalid) r = 0.0f; }
    }
    *r_out = r;
    *rs_out = rs;
}

// adjoint of walker_eval for ONE environment: cotangents go (obs, nullable), go2 (a second observation cotangent
// that is added to the first, nullable), gr (reward) -> gqe, gqde (overwritten), gae (nullable)
// (IP: where the inputs live -- global rows, or the staged shared-memory copies of the fused launch; has_go / has_go2 / has_gae:
//  whether that array is present at all)
template <class IP, class OP>
__device__ __forceinline__ void walker_eval_adj(const DfxWalkerParams& p, IP qe, IP qde, IP ae, IP go, bool has_go,
                                                IP go2, bool has_go2, float gr, bool has_rew,
                                                OP gqe, OP gqde, OP gae, bool has_gae) {
    V3 pos, ang, lin, tt, tdir, up, heading;
    Q4 rot, tq;
    float tn;
    walker_features(p, qe, qde, pos, rot, ang, lin, tt, tn, tdir, tq, up, heading);
    if (p.check_invalid && p.zero_reward_on_invalid && has_rew) {
        bool bad = false;
        for (int i = 0; i < p.num_q; ++i) bad |= !isfinite(qe[i]) || fabsf(qe[i]) > 1e6f;
        for (int i = 0; i < p.num_qd; ++i) bad |= !isfinite(qde[i]) || fabsf(qde[i]) > 1e6f;
        if (bad) gr = 0.0f;
    }
    float dh;
    height_reward(p, pos.y, &dh);
    int k = 0;
    auto G = [&](int idx) { return (has_go ? go[idx] : 0.0f) + (has_go2 ? go2[idx] : 0.0f); };
    // cotangents of the features
    float a_posy = G(0) + (p.height_mode != 2 ? gr * dh : 0.0f);
    Q4 a_rot = Q4{G(1), G(2), G(3), G(4)};
    V3 a_lin = V3{G(5) + gr, G(6), G(7)};
    V3 a_ang = V3{G(8), G(9), G(10)};
    k = 11;
    for (int i = 7; i < p.num_q; ++i) gqe[i] = G(k++);
    for (int i = 6; i < p.num_qd; ++i) gqde[i] = p.joint_vel_scale * G(k++);
    const float a_upy = G(k) + 0.1f * gr; ++k;
    const float a_h = G(k) + gr; ++k;
    if (has_gae) {
        for (int i = 0; i < p.num_act; ++i) {
            const float a = ae[i];
            float g = p.obs_has_actions ? G(k + i) : 0.0f;
            g += gr * p.action_penalty * (p.action_penalty_abs ? (a < 0.0f ? -1.0f : (a > 0.0f ? 1.0f : 0.0f)) : 2.0f * a);
            gae[i] = g;
        }
    }
    // hproj = heading . tdir
    V3 a_heading = tdir * a_h;
    V3 a_tdir = heading * a_h;
    // tdir = tt / tn, tn = max(|tt|, eps)
    V3 a_tt = a_tdir * (1.0f / tn);
    if (sqrtf(dot(tt, tt)) > 1e-9f) a_tt -= tdir * (dot(a_tdir, tdir) / tn);
    V3 a_pos = V3{-a_tt.x, a_posy, -a_tt.z};
    // up = R(tq) b1 ; heading = R(tq) b0
    Q4 a_tq = qrot_adj_q(tq, ld3(p.basis_up), V3{0.0f, a_upy, 0.0f});
    a_tq += qrot_adj_q(tq, ld3(p.basis_heading), a_heading);
    // tq = rot * inv_start
    a_rot += qmul_adj_a(ld4(p.inv_start_rot), a_tq);
    // lin = v - pos x ang
    V3 a_v = a_lin;
    V3 nl = -a_lin;
    cross_adj(pos, ang, nl, a_pos, a_ang);
    gqe[0] = a_pos.x; gqe[1] = a_pos.y; gqe[2] = a_pos.z;
    gqe[3] = a_rot.x; gqe[4] = a_rot.y; gqe[5] = a_rot.z; gqe[6] = a_rot.w;
    gqde[0] = a_ang.x; gqde[1] = a_ang.y; gqde[2] = a_ang.z;
    gqde[3] = a_v.x; gqde[4] = a_v.y; gqde[5] = a_v.z;
}

// ---- the whole env transition after the simulation step, for ONE environment e:
//   progress+1 -> observation, reward, termination (obs_before_reset) -> masked re-initialisation of a
//   terminated environment (state <- start state, last actions <- 0, progress <- 0) -> observation of the
//   state the next step starts from.  Replaces, per env.step(), ~35 small PyTorch ops (torch.where masks, clones,
//   counters) and, in backward, their autograd nodes.
template <class QP, class QDP>
__device__ __forceinline__ void walker_transition_forward_env(const DfxWalkerParams& p, int e, QP qe, QDP qde,      // (qe, qde: this environment's rows)
                                                              const float* actions, const long long* progress,
                                                              const float* start_q, const float* start_qd,
                                                              float* obs_before, float* rew, long long* reset,
                                                              float* q_next, float* qd_next, float* actions_next,
                                                              long long* progress_next, float* obs_next) {
    const float* ae = actions + (size_t)e * p.num_act;
    float* ob = obs_before + (size_t)e * p.num_obs;
    float* on = obs_next + (size_t)e * p.num_obs;
    const long long pr = progress[e] + 1;
    float r = 0.0f;
    long long rs = 0;
    // the observation is formed in a thread-local buffer (L1-resident local memory) and written out once: forming it in
    // place in global memory put a store -> load round trip through L2 on the critical path of this latency-bound code
    // (the validity check and the pass-through to obs_next both read it back)
    float o[kMaxObs];
    walker_eval(p, qe, qde, ae, pr, true, o, &r, &rs);
    rew[e] = r;
    reset[e] = rs;
    progress_next[e] = rs ? 0 : pr;
    float* qn = q_next + (size_t)e * p.num_q;
    float* qdn = qd_next + (size_t)e * p.num_qd;
    float* an = actions_next + (size_t)e * p.num_act;
    for (int i = 0; i < p.num_obs; ++i) ob[i] = o[i];
    if (rs) {
        const float* sq = start_q + (size_t)e * p.num_q;
        const float* sqd = start_qd + (size_t)e * p.num_qd;
        for (int i = 0; i < p.num_q; ++i) qn[i] = sq[i];
        for (int i = 0; i < p.num_qd; ++i) qdn[i] = sqd[i];
        for (int i = 0; i < p.num_act; ++i) an[i] = 0.0f;
        float r2; long long rs2;
        walker_eval(p, sq, sqd, nullptr, 0, false, o, &r2, &rs2);
    } else {
        for (int i = 0; i < p.num_q; ++i) qn[i] = qe[i];
        for (int i = 0; i < p.num_qd; ++i) qdn[i] = qde[i];
        for (int i = 0; i < p.num_act; ++i) an[i] = ae[i];
    }
    for (int i = 0; i < p.num_obs; ++i) on[i] = o[i];
}

// cotangents of (obs_before, rew, q_next, qd_next, actions_next, obs_next), any of them NULL == 0, -> gq, gqd, gact of
// environment e.  A terminated environment passes nothing through its re-initialised outputs.
__device__ __forceinline__ void walker_transition_backward_env(const DfxWalkerParams& p, int e, const float* q, const float* qd,
                                                               const float* actions, const long long* reset,
                                                               const float* g_obs_before, const float* g_rew,
                                                               const float* g_q_next, const float* g_qd_next,
                                                               const float* g_actions_next, const float* g_obs_next,
                                                               float* gq, float* gqd, float* gact) {
    const bool live = reset[e] == 0;
    float* gqe = gq + (size_t)e * p.num_q;
    float* gqde = gqd + (size_t)e * p.num_qd;
    float* gae = gact ? gact + (size_t)e * p.num_act : nullptr;
    walker_eval_adj(p, q + (size_t)e * p.num_q, qd + (size_t)e * p.num_qd, actions + (size_t)e * p.num_act,
                    g_obs_before + (size_t)e * p.num_obs, g_obs_before != nullptr,
                    g_obs_next + (size_t)e * p.num_obs, live && g_obs_next != nullptr,
                    g_rew ? g_rew[e] : 0.0f, g_rew != nullptr, gqe, gqde, gae, gae != nullptr);
    if (!live) return;
    if (g_q_next) { const float* g = g_q_next + (size_t)e * p.num_q;
    for (int i = 0; i < p.num_q; ++i) gqe[i] += g[i]; }
    if (g_qd_next) { const float* g = g_qd_next + (size_t)e * p.num_qd;
    for (int i = 0; i < p.num_qd; ++i) gqde[i] += g[i]; }
    if (gae && g_actions_next) { const float* g = g_actions_next + (size_t)e * p.num_act;
    for (int i = 0; i < p.num_act; ++i) gae[i] += g[i]; }
}

// ---- planar envs (Hopper, HalfCheetah: observation = [q[1:], qd]; CartPole swing-up: [x, xd, sin th, cos th, thd]):
// the same transition as walker_transition_*, reference envs/hopper.py:170-268, envs/cheetah.py:160-244,
// envs/cartpole_swing_up.py:120-187
template <class QP, class QDP, class OP>
__device__ __forceinline__ void planar_eval(const DfxPlanarParams& p, QP qe, QDP qde,
                                            const float* ae, long long progress, bool want_reward,
                                            OP o, float* r_out, long long* rs_out) {
    float act_sq = 0.0f;
    for (int i = 0; i < p.num_act; ++i) { const float a = ae ? ae[i] : 0.0f; act_sq += a * a; }
    if (p.kind == 2) {                      // CartPole
        const float x = qe[0], th = qe[1], xd = qde[0], thd = qde[1];
        o[0] = x; o[1] = xd; o[2] = sinf(th); o[3] = cosf(th); o[4] = thd;
        if (!want_reward) return;
        const float t = atan2f(sinf(th), cosf(th));                  // normalize_angle
        *r_out = -(t * t) * p.pole_angle_penalty - (thd * thd) * p.pole_velocity_penalty - (x * x) * p.cart_position_penalty
                 - (xd * xd) * p.cart_velocity_penalty - act_sq * p.action_penalty;
        *rs_out = (progress > (long long)p.episode_length - 1) ? 1 : 0;
        return;
    }
    int k = 0;
    for (int i = 1; i < p.num_q; ++i) o[k++] = qe[i];
    for (int i = 0; i < p.num_qd; ++i) o[k++] = qde[i];
    if (!want_reward) return;
    const float vx = qde[0];                // o[num_q - 1]
    long long rs = (progress > (long long)p.episode_length - 1) ? 1 : 0;
    if (p.kind == 0) {                      // Hopper
        const float h0 = qe[1], ang = qe[2];
        float h = fminf(fmaxf(h0 - (p.termination_height + p.termination_height_tolerance), -1.0f), 0.3f);
        if (h < 0.0f) h = -200.0f * h * h;
        if (h > 0.0f) h = p.height_rew_scale * h;
        const float angle_reward = 1.0f * (-(ang * ang) / (p.termination_angle * p.termination_angle) + 1.0f);
        *r_out = vx + h + angle_reward + act_sq * p.action_penalty;
        if (p.early_termination && h0 < p.termination_height) rs = 1;
    } else {                                // HalfCheetah
        *r_out = vx + act_sq * p.action_penalty;
    }
    *rs_out = rs;
}

template <class IP, class OP>
__device__ __forceinline__ void planar_eval_adj(const DfxPlanarParams& p, IP qe, IP qde, IP ae, IP go, bool has_go,
                                                IP go2, bool has_go2, float gr,
                                                OP gqe, OP gqde, OP gae, bool has_gae) {
    auto G = [&](int idx) { return (has_go ? go[idx] : 0.0f) + (has_go2 ? go2[idx] : 0.0f); };
    if (has_gae) for (int i = 0; i < p.num_act; ++i) gae[i] = (p.kind == 2 ? -1.0f : 1.0f) * gr * p.action_penalty * 2.0f * ae[i];
    if (p.kind == 2) {
        const float x = qe[0], th = qe[1], xd = qde[0], thd = qde[1];
        const float t = atan2f(sinf(th), cosf(th));
        gqe[0] = G(0) - gr * 2.0f * x * p.cart_position_penalty;
        gqe[1] = G(2) * cosf(th) - G(3) * sinf(th) - gr * 2.0f * t * p.pole_angle_penalty;     // d normalize_angle / d th = 1
        gqde[0] = G(1) - gr * 2.0f * xd * p.cart_velocity_penalty;
        gqde[1] = G(4) - gr * 2.0f * thd * p.pole_velocity_penalty;
        return;
    }
    int k = 0;
    gqe[0] = 0.0f;
    for (int i = 1; i < p.num_q; ++i) gqe[i] = G(k++);
    for (int i = 0; i < p.num_qd; ++i) gqde[i] = G(k++);
    gqde[0] += gr;
    if (p.kind == 0) {
        const float h0 = qe[1], ang = qe[2];
        const float x = h0 - (p.termination_height + p.termination_height_tolerance);
        const float h = fminf(fmaxf(x, -1.0f), 0.3f);
        const float dclip = (x >= -1.0f && x <= 0.3f) ? 1.0f : 0.0f;     // torch.clip passes the gradient on the closed interval
        float dh = dclip;                                                   // h == 0: both torch.where keep h
        if (h < 0.0f) dh = -400.0f * h * dclip;
        else if (h > 0.0f) dh = p.height_rew_scale * dclip;
        gqe[1] += gr * dh;
        gqe[2] += gr * (-2.0f * ang / (p.termination_angle * p.termination_angle));
    }
}

template <class QP, class QDP>
__device__ __forceinline__ void planar_transition_forward_env(const DfxPlanarParams& p, int e, QP qe, QDP qde,      // (qe, qde: this environment's rows)
                                                              const float* actions, const long long* progress,
                                                              const float* start_q, const float* start_qd,
                                                              float* obs_before, float* rew, long long* reset,
                                                              float* q_next, float* qd_next, float* actions_next,
                                                              long long* progress_next, float* obs_next) {
    const float* ae = actions + (size_t)e * p.num_act;
    float* ob = obs_before + (size_t)e * p.num_obs;
    float* on = obs_next + (size_t)e * p.num_obs;
    const long long pr = progress[e] + 1;
    float r = 0.0f;
    long long rs = 0;
    planar_eval(p, qe, qde, ae, pr, true, ob, &r, &rs);
    rew[e] = r;
    reset[e] = rs;
    progress_next[e] = rs ? 0 : pr;
    float* qn = q_next + (size_t)e * p.num_q;
    float* qdn = qd_next + (size_t)e * p.num_qd;
    float* an = actions_next + (size_t)e * p.num_act;
    if (rs) {
        const float* sq = start_q + (size_t)e * p.num_q;
        const float* sqd = start_qd + (size_t)e * p.num_qd;
        for (int i = 0; i < p.num_q; ++i) qn[i] = sq[i];
        for (int i = 0; i < p.num_qd; ++i) qdn[i] = sqd[i];
        for (int i = 0; i < p.num_act; ++i) an[i] = p.zero_actions_on_reset ? 0.0f : ae[i];
        float r2; long long rs2;
        planar_eval(p, sq, sqd, p.zero_actions_on_reset ? nullptr : ae, 0, false, on, &r2, &rs2);
    } else {
        for (int i = 0; i < p.num_q; ++i) qn[i] = qe[i];
        for (int i = 0; i < p.num_qd; ++i) qdn[i] = qde[i];
        for (int i = 0; i < p.num_act; ++i) an[i] = ae[i];
        for (int i = 0; i < p.num_obs; ++i) on[i] = ob[i];
    }
}

__device__ __forceinline__ void planar_transition_backward_env(const DfxPlanarParams& p, int e, const float* q, const float* qd,
                                                               const float* actions, const long long* reset,
                                                               const float* g_obs_before, const float* g_rew,
                                                               const float* g_q_next, const float* g_qd_next,
                                                               const float* g_actions_next, const float* g_obs_next,
                                                               float* gq, float* gqd, float* gact) {
    const bool live = reset[e] == 0;
    float* gqe = gq + (size_t)e * p.num_q;
    float* gqde = gqd + (size_t)e * p.num_qd;
    float* gae = gact ? gact + (size_t)e * p.num_act : nullptr;
    planar_eval_adj(p, q + (size_t)e * p.num_q, qd + (size_t)e * p.num_qd, actions + (size_t)e * p.num_act,
                    g_obs_before + (size_t)e * p.num_obs, g_obs_before != nullptr,
                    g_obs_next + (size_t)e * p.num_obs, live && g_obs_next != nullptr,
                    g_rew ? g_rew[e] : 0.0f, gqe, gqde, gae, gae != nullptr);
    // the actions survive a reset in envs that do not clear them (CartPole): their cotangent passes either way
    if (gae && g_actions_next && (live || !p.zero_actions_on_reset)) {
        const float* g = g_actions_next + (size_t)e * p.num_act;
        for (int i = 0; i < p.num_act; ++i) gae[i] += g[i];
    }
    if (!live) return;
    if (g_q_next) { const float* g = g_q_next + (size_t)e * p.num_q;
    for (int i = 0; i < p.num_q; ++i) gqe[i] += g[i]; }
    if (g_qd_next) { const float* g = g_qd_next + (size_t)e * p.num_qd;
    for (int i = 0; i < p.num_qd; ++i) gqde[i] += g[i]; }
}

// =====================================================================================
// The transition of a whole TILE of E environments by all NT threads of its CTA (dfx_tile.cu: the epilogue of the simulation
// launch and the prologue of the adjoint launch of dfx_env_step_forward / _backward).  One thread per environment alone is slow
// as an epilogue -- ~150 dependent, uncoalesced global accesses by a single warp -- so the rows are STAGED in the (dead) scratch tile: thread e < E evaluates environment e entirely in shared memory,
// and all NT threads move the rows between the tile and global memory, element k of environment e by thread k * E + e
// (conflict-free scratch accesses).  Same per-environment arithmetic as above.
// =====================================================================================
__device__ __forceinline__ bool env_zero_actions_on_reset(const DfxWalkerParams&) { return true; }
__device__ __forceinline__ bool env_zero_actions_on_reset(const DfxPlanarParams& p) { return p.zero_actions_on_reset != 0; }
template <class QP, class QDP, class OP>
__device__ __forceinline__ void env_eval(const DfxWalkerParams& p, QP qe, QDP qde, const float* ae, long long progress, bool want_reward,
                                         OP o, float* r, long long* rs) { walker_eval(p, qe, qde, ae, progress, want_reward, o, r, rs); }
template <class QP, class QDP, class OP>
__device__ __forceinline__ void env_eval(const DfxPlanarParams& p, QP qe, QDP qde, const float* ae, long long progress, bool want_reward,
                                         OP o, float* r, long long* rs) { planar_eval(p, qe, qde, ae, progress, want_reward, o, r, rs); }
template <class IP, class OP>
__device__ __forceinline__ void env_eval_adj(const DfxWalkerParams& p, IP qe, IP qde, IP ae, IP go, bool has_go, IP go2, bool has_go2,
                                             float gr, bool has_rew, OP gqe, OP gqde, OP gae) {
    walker_eval_adj(p, qe, qde, ae, go, has_go, go2, has_go2, gr, has_rew, gqe, gqde, gae, true);
}
template <class IP, class OP>
__device__ __forceinline__ void env_eval_adj(const DfxPlanarParams& p, IP qe, IP qde, IP ae, IP go, bool has_go, IP go2, bool has_go2,
                                             float gr, bool has_rew, OP gqe, OP gqde, OP gae) {
    (void)has_rew;
    planar_eval_adj(p, qe, qde, ae, go, has_go, go2, has_go2, gr, gqe, gqde, gae, true);
}

// (scratch floats per environment the staged transition needs: 2 num_obs + 1 forward, 2 num_obs + 3 (num_q + num_qd + num_act)
//  backward -- dfx_kernels.cu transition_fits() checks them against the layout on the host, else the call runs two launches)

// forward.  The stepped state is at scratch offsets q_off / qd_off of every environment; [stage_off, stage_off + 2 num_obs + 1) is free.
// (One body for both env families: only the per-environment evaluation depends on the parameter struct.  The row loops are not
//  unrolled: this code runs once per launch from a cold instruction cache, and each iteration is one dependent load -> store anyway.)
template <int NT, int E>
__device__ __forceinline__ void tile_transition_forward(int kind, const DfxEnvTransition& t, const float* used, float* tile_base,
                                                        int q_off, int qd_off, int stage_off, int N) {
    const int tid = (int)threadIdx.x, env0 = (int)blockIdx.x * E;
    const bool walker = kind == 1;
    const int nq = walker ? t.walker.num_q : t.planar.num_q, nd = walker ? t.walker.num_qd : t.planar.num_qd;
    const int na = walker ? t.walker.num_act : t.planar.num_act, no = walker ? t.walker.num_obs : t.planar.num_obs;
    const bool zero_act = walker ? env_zero_actions_on_reset(t.walker) : env_zero_actions_on_reset(t.planar);
    const int ob = stage_off, on = ob + no, rsf = on + no;
    if (tid < E && env0 + tid < N) {
        const int env = env0 + tid;
        const SP se{tile_base + tid};
        const float* ae = used + (size_t)env * na;
        const float* ae0 = zero_act ? (const float*)nullptr : ae;
        const float* sq = t.start_q + (size_t)env * nq;
        const float* sqd = t.start_qd + (size_t)env * nd;
        const long long pr = t.progress[env] + 1;
        float r = 0.0f, r2;
        long long rs = 0, rs2;
        if (walker) {
            env_eval(t.walker, se + q_off, se + qd_off, ae, pr, true, se + ob, &r, &rs);
            if (rs) env_eval(t.walker, sq, sqd, ae0, 0, false, se + on, &r2, &rs2);     // observation of the state it restarts from
        } else {
            env_eval(t.planar, se + q_off, se + qd_off, ae, pr, true, se + ob, &r, &rs);
            if (rs) env_eval(t.planar, sq, sqd, ae0, 0, false, se + on, &r2, &rs2);
        }
        t.rew[env] = r;
        t.reset[env] = rs;
        t.progress_next[env] = rs ? 0 : pr;
        sp_int(se + rsf)[0] = (int)rs;
    }
    __syncthreads();
    const int nenv = (N - env0) < E ? (N - env0) : E;
#pragma unroll 1
    for (int j = tid; j < E * no; j += NT) {
        const int e = j % E, k = j / E;
        if (e >= nenv) continue;
        const SP se{tile_base + e};
        const size_t row = (size_t)(env0 + e) * no + k;
        const float v = se[ob + k];
        t.obs_before[row] = v;
        t.obs_next[row] = sp_int(se + rsf)[0] ? se[on + k] : v;
    }
#pragma unroll 1
    for (int j = tid; j < E * (nq + nd + na); j += NT) {       // q_next, qd_next, actions_next
        const int e = j % E;
        int k = j / E;
        if (e >= nenv) continue;
        const SP se{tile_base + e};
        const bool rs = sp_int(se + rsf)[0] != 0;
        if (k < nq) {
            const size_t row = (size_t)(env0 + e) * nq + k;
            t.q_next[row] = rs ? t.start_q[row] : se[q_off + k];
        } else if (k < nq + nd) {
            k -= nq;
            const size_t row = (size_t)(env0 + e) * nd + k;
            t.qd_next[row] = rs ? t.start_qd[row] : se[qd_off + k];
        } else {
            k -= nq + nd;
            const size_t row = (size_t)(env0 + e) * na + k;
            t.actions_next[row] = (rs && zero_act) ? 0.0f : used[row];
        }
    }
}

// backward.  The whole scratch tile is free (the step adjoint has not started); [0, env_stage_floats_backward()) is used.
template <int NT, int E>
__device__ __forceinline__ void tile_transition_backward(int kind, const DfxEnvTransitionAdj& t, float* tile_base, int N) {
    const int tid = (int)threadIdx.x, env0 = (int)blockIdx.x * E;
    const int nenv = (N - env0) < E ? (N - env0) : E;
    const bool walker = kind == 1;
    const int nq = walker ? t.walker.num_q : t.planar.num_q, nd = walker ? t.walker.num_qd : t.planar.num_qd;
    const int na = walker ? t.walker.num_act : t.planar.num_act, no = walker ? t.walker.num_obs : t.planar.num_obs;
    // staged inputs (8 rows per environment), then the outputs (3)
    const float* src[8] = {t.g_obs_before, t.g_obs_next, t.g_q_next, t.g_qd_next, t.g_actions_next, t.q_sim, t.qd_sim, t.used};
    const int width[8] = {no, no, nq, nd, na, nq, nd, na};
    int off[9];
    off[0] = 0;
#pragma unroll
    for (int a = 0; a < 8; ++a) off[a + 1] = off[a] + width[a];
    const int g1 = off[0], g2 = off[1], gq = off[2], gd = off[3], ga = off[4], qs = off[5], ds = off[6], us = off[7];
    const int oq = off[8], od = oq + nq, oa = od + nd;
#pragma unroll 1
    for (int a = 0; a < 8; ++a) {
        const float* sa = src[a];
        if (!sa) continue;
        const int w = width[a], d0 = off[a];
#pragma unroll 1
        for (int j = tid; j < E * w; j += NT) {
            const int e = j % E, k = j / E;
            if (e < nenv) SP{tile_base + e}[d0 + k] = sa[(size_t)(env0 + e) * w + k];
        }
    }
    __syncthreads();
    if (tid < E && tid < nenv) {
        const int env = env0 + tid;
        const SP se{tile_base + tid};
        const bool live = t.reset[env] == 0;
        const bool has1 = t.g_obs_before != nullptr, has2 = live && t.g_obs_next != nullptr, has_rew = t.g_rew != nullptr;
        const float gr = has_rew ? t.g_rew[env] : 0.0f;
        bool act_pass;
        if (walker) {
            env_eval_adj(t.walker, se + qs, se + ds, se + us, se + g1, has1, se + g2, has2, gr, has_rew, se + oq, se + od, se + oa);
            act_pass = live || !env_zero_actions_on_reset(t.walker);
        } else {
            env_eval_adj(t.planar, se + qs, se + ds, se + us, se + g1, has1, se + g2, has2, gr, has_rew, se + oq, se + od, se + oa);
            act_pass = live || !env_zero_actions_on_reset(t.planar);
        }
        // what passes through the (not re-initialised) next state and actions
        if (t.g_actions_next && act_pass) {
#pragma unroll 1
            for (int i = 0; i < na; ++i) se[oa + i] += se[ga + i];
        }
        if (live && t.g_q_next) {
#pragma unroll 1
            for (int i = 0; i < nq; ++i) se[oq + i] += se[gq + i];
        }
        if (live && t.g_qd_next) {
#pragma unroll 1
            for (int i = 0; i < nd; ++i) se[od + i] += se[gd + i];
        }
    }
    __syncthreads();
#pragma unroll 1
    for (int j = tid; j < E * (nq + nd + na); j += NT) {       // -> gq_sim, gqd_sim, g_used
        const int e = j % E;
        int k = j / E;
        if (e >= nenv) continue;
        const float v = SP{tile_base + e}[oq + k];              // (oq, od, oa are adjacent)
        if (k < nq) t.gq_sim[(size_t)(env0 + e) * nq + k] = v;
        else if (k < nq + nd) t.gqd_sim[(size_t)(env0 + e) * nd + (k - nq)] = v;
        else t.g_used[(size_t)(env0 + e) * na + (k - nq - nd)] = v;
    }
    __syncthreads();
}

}  // namespace dfx
