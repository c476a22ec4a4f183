/* dfx.h -- C ABI of the H100-native (sm_90a) differentiable articulated rigid-body step.
 *
 * This is the drop-in boundary underneath `dflex.sim.SemiImplicitIntegrator.forward`
 * (reference NVlabs/DiffRL dflex/dflex/sim.py:2182).  In the reference that call fans out into
 * 10-11 generated kernels per substep, each exported from one pybind module as
 *     <kernel>_{cpu,cuda}_forward (int dim, torch::Tensor...)
 *     <kernel>_{cpu,cuda}_backward(int dim, inputs..., outputs..., adj_inputs..., adj_outputs...)
 * (reference dflex/dflex/adjoint.py:1247-1291: raw data_ptr() casts, default stream, no error
 * returns, a null/empty adjoint tensor meaning "skip").  Here the whole env-step (all substeps)
 * is ONE forward entry point and ONE backward entry point over plain device pointers:
 *
 *   dfx_step_forward   replaces  SimulateFunc.forward  (sim.py:2097-2123): substeps x
 *                      { eval_rigid_fk :1681, eval_rigid_id :1845, eval_rigid_contacts_art :1137,
 *                        eval_muscles :1245, eval_rigid_tau :1896, [eval_rigid_jacobian :1950,
 *                        eval_rigid_mass :1999, eval_dense_gemm_batched x2 :2023,
 *                        eval_dense_cholesky_batched :2031], eval_dense_solve_batched :2047,
 *                        eval_rigid_integrate :2052 }
 *   dfx_step_backward  replaces  SimulateFunc.backward (sim.py:2127-2154) / Tape.replay
 *                      (adjoint.py:2153-2199): the *_backward twins of the kernels above.
 *
 * All pointers are DEVICE pointers unless stated otherwise; all calls are stream-ordered on
 * `stream` (a cudaStream_t passed as void*), never synchronise the host, and return a
 * cudaError_t value as int (0 == cudaSuccess).  Thread-compatible: one stream per caller.
 * No torch types appear in any signature.
 */
#ifndef DFX_H_
#define DFX_H_

#ifdef __cplusplus
extern "C" {
#endif

/* External wrench on the links, per environment (the _ex twins of the step entries below; a NULL DfxExternalWrench* is no
 * wrench, and those calls run exactly the code of the entries without _ex).  f_ext [N, L, 6], device, fp32: row (e, i) is
 * (tau, F), angular part first as in dflex spatial vectors -- F a force in world axes applied AT LINK i's CENTRE OF MASS,
 * tau a pure torque in world axes (the convention of MuJoCo's xfrc_applied).  It is held constant over the env-step's
 * substeps, as the actuation.  In the step it enters where gravity does:  body_f_s = f_b - (c x (m g + F) + tau, m g + F),
 * c = the link's centre of mass.  The backward entries take the SAME f_ext as the forward call and overwrite g_f_ext
 * [N, L, 6] (NULL: skip) with its cotangent; f_ext == NULL with a non-NULL struct is cudaErrorInvalidValue.  The external-
 * wrench kernels keep 6 L (forward) / 12 L (backward) more floats of scratch per environment: dfx_launch_plan(pack, 2 | bwd,
 * ...) tells whether they still fit.  Flag bit 6 (64) of dfx_set_flags has no external-wrench kernels (cudaErrorNotSupported). */
typedef struct DfxExternalWrench {
    const float* f_ext;
    float* g_f_ext;
} DfxExternalWrench;

/* Static description of ONE articulation (HOST pointers; copied during dfx_pack_create).
 * Field names and layouts are those of the reference Model (dflex/dflex/model.py:1646-1879,
 * collide() :424-515) restricted to a single environment, with link / shape indices made
 * local to that environment.  All environments of a batch share this description. */
typedef struct DfxModelDesc {
    int link_count;      /* L */
    int dof_count;       /* D  = len(joint_qd)  per env */
    int coord_count;     /* Q  = len(joint_q)   per env */
    int contact_count;   /* C */
    int muscle_count;    /* M */
    int waypoint_count;  /* W  = len(muscle_links) per env */
    int shape_count;     /* rows of shape_materials */
    int ground;          /* model.ground */
    float gravity[3];

    const int* joint_type;          /* [L]   0 prismatic, 1 revolute, 2 ball, 3 fixed, 4 free (model.py:35-39) */
    const int* joint_parent;        /* [L]   local parent link or -1 */
    const int* joint_q_start;       /* [L+1] with closing sentinel (model.py:1757) */
    const int* joint_qd_start;      /* [L+1] */
    const float* joint_X_pj;        /* [L,7] p then q(xyzw) */
    const float* joint_X_cm;        /* [L,7] */
    const float* joint_axis;        /* [L,3] */
    const float* body_I_m;          /* [L,6,6] blockdiag(I_c, m*1) (util.py:340-349) */
    const float* joint_target_ke;   /* [L] */
    const float* joint_target_kd;   /* [L] */
    const float* joint_limit_ke;    /* [L] */
    const float* joint_limit_kd;    /* [L] */
    const float* joint_target;      /* [Q] */
    const float* joint_limit_lower; /* [Q] */
    const float* joint_limit_upper; /* [Q] */
    const float* joint_armature;    /* [D] */

    const int* contact_body0;       /* [C] local link index */
    const float* contact_point0;    /* [C,3] */
    const float* contact_dist;      /* [C] */
    const int* contact_material;    /* [C] local shape index into shape_materials */
    const float* shape_materials;   /* [shape_count,4] ke, kd, kf, mu (model.py:964) */

    const int* muscle_start;        /* [M+1] */
    const int* muscle_links;        /* [W] local link index */
    const float* muscle_points;     /* [W,3] */
} DfxModelDesc;

typedef struct dfx_pack dfx_pack_t;

/* Optional per-substep derived state of the LAST substep of a forward call, in the reference's
 * State layouts (model.py:360-388); any pointer may be NULL.  Device pointers, env-major. */
typedef struct DfxDerived {
    float* body_X_sc;  /* [N*L,7] */
    float* body_X_sm;  /* [N*L,7] */
    float* joint_S_s;  /* [N*D,6] */
    float* body_v_s;   /* [N*L,6] */
    float* body_a_s;   /* [N*L,6] */
    float* body_f_s;   /* [N*L,6] */
    float* body_ft_s;  /* [N*L,6] */
    float* joint_tau;  /* [N*D]   */
    float* joint_qdd;  /* [N*D]   */
    float* H;          /* [N,D,D] joint-space inertia of the last mass-matrix update */
    float* L;          /* [N,D,D] its Cholesky factor */
} DfxDerived;

enum {
    DFX_QUERY_LINKS = 0,
    DFX_QUERY_DOFS = 1,
    DFX_QUERY_COORDS = 2,
    DFX_QUERY_CONTACTS = 3,
    DFX_QUERY_MUSCLES = 4,
    DFX_QUERY_FWD_SCRATCH_FLOATS = 5, /* shared-memory floats per environment, forward */
    DFX_QUERY_BWD_SCRATCH_FLOATS = 6, /* shared-memory floats per environment, backward */
    DFX_QUERY_TREE_DEPTH = 7,
    DFX_QUERY_TAPE_ROW_FLOATS = 8,    /* floats per (substep, environment) tape row */
    DFX_QUERY_TAPE_TILE = 9,          /* 0: tape blocks are [block][env][n]; E = 8 / 16 / 32: [block][tile of E envs][n][E] (tile kernels) */
    DFX_QUERY_TAPE_BF16 = 10,         /* 1: the middle of every tape row (the forward intermediates) is stored as bf16 */
    DFX_QUERY_TAPE_ROW_UNITS = 11,    /* 4-byte units per (substep, environment) row IN THE TAPE (== row floats unless bf16) */
    DFX_QUERY_JOINT_MASK = 12         /* bit t set: some link has joint type t (0 prismatic, 1 revolute, 2 ball, 3 fixed, 4 free) */
};

/* Build the device-resident pack for CUDA device `device` (>= 0).  Returns NULL on failure and
 * writes a message into err (if err != NULL). */
dfx_pack_t* dfx_pack_create(const DfxModelDesc* desc, int device, char* err, int err_len);
void dfx_pack_destroy(dfx_pack_t* pack);
int dfx_pack_query(const dfx_pack_t* pack, int what);

/* Update the pack's gravity / ground flag (envs assign model.gravity and model.ground after
 * finalize, reference envs/ant.py:132-133). */
int dfx_pack_set_gravity(dfx_pack_t* pack, float gx, float gy, float gz, int ground);

/* Number of floats of tape one forward call writes for `num_envs` environments:
 *   substeps * N * (Q + 8 D + 32 L)             per substep: the (q, qd) entering it + the forward
 *                                               intermediates the adjoint reads back instead of recomputing
 * + ceil(substeps / mm_freq) * N * D * D        H^-1 of every mass-matrix update           */
long long dfx_tape_floats(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq);

/* One env-step: `substeps` semi-implicit substeps of dt/substeps with the actuation held
 * constant (sim.py:2104-2113); the joint-space inertia is refactorised when i % mm_freq == 0.
 * dt is a double because the reference divides the Python float dt by substeps before the
 * value is narrowed to fp32 at the kernel boundary (sim.py:2113).
 *   q [N*Q], qd [N*D], act [N*D], musc [N*M] (NULL when M == 0)   inputs (not modified)
 *   q_out [N*Q], qd_out [N*D]                                      outputs (may alias the inputs)
 *   tape     NULL => no-grad mode (dflex.config.no_grad, sim.py:2201-2207)
 *   derived  NULL or a struct of optional dumps                                              */
int dfx_step_forward(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                     const float* q, const float* qd, const float* act, const float* musc,
                     float* q_out, float* qd_out, float* tape, const DfxDerived* derived,
                     void* stream);

/* Adjoint of dfx_step_forward.  gq_out/gqd_out are the cotangents of (q_out, qd_out) (NULL == 0);
 * gq, gqd, gact, gmusc receive (are overwritten with) the cotangents of the inputs; any of
 * them may be NULL to skip the write (the reference's "empty tensor => skip", adjoint.h:336-346). */
int dfx_step_backward(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                      const float* act, const float* musc, const float* tape,
                      const float* gq_out, const float* gqd_out,
                      float* gq, float* gqd, float* gact, float* gmusc, void* stream);
/* the two above with an external wrench (DfxExternalWrench; NULL: none) */
int dfx_step_forward_ex(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                        const float* q, const float* qd, const float* act, const float* musc,
                        float* q_out, float* qd_out, float* tape, const DfxDerived* derived,
                        void* stream, const DfxExternalWrench* wrench);
int dfx_step_backward_ex(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                         const float* act, const float* musc, const float* tape,
                         const float* gq_out, const float* gqd_out,
                         float* gq, float* gqd, float* gact, float* gmusc, void* stream, const DfxExternalWrench* wrench);

/* ---- fused env epilogue (SURVEY.md section 8f-1): observation + reward + termination flags of the free-root
 * walker envs and its adjoint, replacing ~35 PyTorch ops per env.step (reference envs/ant.py:266-307,
 * envs/humanoid.py:314-368, envs/snu_humanoid.py:378-432).  One thread per environment. */
typedef struct DfxWalkerParams {
    int num_q, num_qd, num_act, num_obs;
    int obs_has_actions;        /* Ant, Humanoid: observation ends with the actions; SNU: no */
    int height_mode;            /* 0: h - termination_height (Ant); 1: clipped quadratic (Humanoid); 2: none (SNU) */
    int action_penalty_abs;     /* 0: sum a^2 ; 1: sum |a| (SNU) */
    int early_termination;      /* reset when h < termination_height */
    int check_invalid;          /* reset on NaN / Inf / |x| > 1e6 (Humanoid, SNU) */
    int zero_reward_on_invalid; /* reward of an invalid environment is 0 (Humanoid: envs/humanoid.py:369, SNU: envs/snu_humanoid.py) */
    int episode_length;
    float joint_vel_scale, termination_height, termination_tolerance, height_rew_scale, action_penalty;
    float target[3];            /* targets + start_pos */
    float inv_start_rot[4];
    float basis_heading[3], basis_up[3];
} DfxWalkerParams;

/* q [n*num_q], qd [n*num_qd], actions [n*num_act], progress [n] (int64) -> obs [n*num_obs], and when rew != NULL
 * rew [n], reset [n] (int64, 0/1). */
int dfx_walker_obs_forward(const DfxWalkerParams* p, int n, const float* q, const float* qd, const float* actions,
                           const long long* progress, float* obs, float* rew, long long* reset, void* stream);
/* cotangents g_obs [n*num_obs] (NULL == 0), g_rew [n] (NULL == 0) -> gq, gqd (overwritten), gact (NULL: skip). */
int dfx_walker_obs_backward(const DfxWalkerParams* p, int n, const float* q, const float* qd, const float* actions,
                            const float* g_obs, const float* g_rew, float* gq, float* gqd, float* gact, void* stream);

/* ---- the whole env transition after the simulation step (reference envs/ant.py:156-190: progress counter,
 * calculateObservations, calculateReward, reset of the terminated environments, observation of the new state),
 * with the reset done by mask so that nothing synchronises with the host.  `progress` is the counter BEFORE this
 * step.  start_q [n*num_q], start_qd [n*num_qd]: the state a terminated environment restarts from.
 * Outputs: obs_before [n*num_obs] (the reference's extras["obs_before_reset"]), rew [n], reset [n] (int64 0/1),
 * q_next, qd_next, actions_next [n*num_act] (zeroed where reset), progress_next [n], obs_next [n*num_obs]. */
int dfx_walker_transition_forward(const DfxWalkerParams* p, int n, const float* q, const float* qd, const float* actions,
                                  const long long* progress, const float* start_q, const float* start_qd,
                                  float* obs_before, float* rew, long long* reset, float* q_next, float* qd_next,
                                  float* actions_next, long long* progress_next, float* obs_next, void* stream);
/* cotangents of the six differentiable outputs (NULL == 0) -> gq, gqd (overwritten), gact (NULL: skip). */
int dfx_walker_transition_backward(const DfxWalkerParams* p, int n, const float* q, const float* qd, const float* actions,
                                   const long long* reset, const float* g_obs_before, const float* g_rew,
                                   const float* g_q_next, const float* g_qd_next, const float* g_actions_next,
                                   const float* g_obs_next, float* gq, float* gqd, float* gact, void* stream);

/* ---- the same transition for the planar envs: kind 0 Hopper (envs/hopper.py:170-268), 1 HalfCheetah (envs/cheetah.py:160-244)
 * -- observation [q[1:], qd] -- and 2 CartPole swing-up (envs/cartpole_swing_up.py:120-187: [x, xd, sin th, cos th, thd]). */
typedef struct DfxPlanarParams {
    int num_q, num_qd, num_act, num_obs;
    int kind;                    /* 0 Hopper, 1 HalfCheetah, 2 CartPole swing-up */
    int early_termination;       /* Hopper: reset when the height drops below termination_height */
    int zero_actions_on_reset;   /* the env keeps a copy of the actions and clears it on reset (not CartPole) */
    int episode_length;
    float termination_height, termination_height_tolerance, termination_angle, height_rew_scale;
    float action_penalty;        /* Hopper / HalfCheetah: reward += penalty * sum a^2; CartPole: reward -= penalty * sum a^2 */
    float pole_angle_penalty, pole_velocity_penalty, cart_position_penalty, cart_velocity_penalty;
} DfxPlanarParams;
int dfx_planar_transition_forward(const DfxPlanarParams* p, int n, const float* q, const float* qd, const float* actions,
                                  const long long* progress, const float* start_q, const float* start_qd,
                                  float* obs_before, float* rew, long long* reset, float* q_next, float* qd_next,
                                  float* actions_next, long long* progress_next, float* obs_next, void* stream);
int dfx_planar_transition_backward(const DfxPlanarParams* p, int n, const float* q, const float* qd, const float* actions,
                                   const long long* reset, const float* g_obs_before, const float* g_rew,
                                   const float* g_q_next, const float* g_qd_next, const float* g_actions_next,
                                   const float* g_obs_next, float* gq, float* gqd, float* gact, void* stream);

/* ---- policy output -> actuation (reference envs/ant.py:156-166, envs/snu_humanoid.py:283-296):
 * used[e, j] = clip(raw[e, j], -1, 1) * pre_scale + pre_bias ;  drive[e, offset + j] = (used[e, j] * drive_scale) * strength[j],
 * every other entry of the [n, width] drive rows zero (joint_act, or the muscle activations with offset 0). */
int dfx_action_map_forward(int n, int num_act, int width, int offset, float pre_scale, float pre_bias, float drive_scale,
                           const float* strength, const float* raw, float* used, float* drive, void* stream);
/* g_used [n*num_act] (NULL == 0), g_drive [n*width] (NULL == 0) -> g_raw [n*num_act]. */
int dfx_action_map_backward(int n, int num_act, int width, int offset, float pre_scale, float drive_scale, const float* strength,
                            const float* raw, const float* g_used, const float* g_drive, float* g_raw, void* stream);

/* ---- the simulation step with the action map folded in (saves the two action-map launches per env.step()):
 * the step kernels form joint_act (or, map.is_muscle, the muscle activations) from the raw policy output while loading it,
 * write `used` (= the env's `actions`: clip(raw) * pre_scale + pre_bias) and, in the adjoint, turn the actuation cotangent
 * into the cotangent of the raw policy output -- same arithmetic as dfx_action_map_forward / _backward.
 * `act_other`: the array the map does NOT drive (joint_act of a muscle model; NULL = zeros). */
typedef struct {
    int num_act;         /* policy outputs per environment */
    int offset;          /* first driven entry of a joint_act / muscle-activation row */
    int is_muscle;       /* 0: drives joint_act [n, D]; 1: drives the muscle activations [n, M] */
    float pre_scale, pre_bias, drive_scale;
    const float* strength;   /* [num_act], device */
} DfxActionMap;
int dfx_step_forward_mapped(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                            const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                            float* used, float* q_out, float* qd_out, float* tape, void* stream);
/* cotangents of (q_out, qd_out, used; any NULL == 0) -> gq, gqd, g_raw */
int dfx_step_backward_mapped(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                             const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                             const float* gq_out, const float* gqd_out, const float* g_used,
                             float* gq, float* gqd, float* g_raw, void* stream);
int dfx_step_forward_mapped_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                               const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                               float* used, float* q_out, float* qd_out, float* tape, void* stream, const DfxExternalWrench* wrench);
int dfx_step_backward_mapped_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                                const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                                const float* gq_out, const float* gqd_out, const float* g_used,
                                float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* wrench);

/* ---- env.step() as ONE launch (SURVEY.md section 8f-1: "fuse into the step epilogue (and its adjoint)"; reference
 * envs/ant.py:156-190 = the action map, SemiImplicitIntegrator.forward and the transition, ~40 PyTorch kernels + one per
 * generated dflex kernel).  Exactly dfx_step_forward_mapped followed by dfx_walker_transition_forward /
 * dfx_planar_transition_forward on its outputs (q_sim, qd_sim, used) -- the same per-environment code, states / flags / counters
 * identical, observations and rewards to a few ulp (the two compilations may contract a*b - c*d differently) -- but the
 * tile kernels run the transition of a tile's environments as the EPILOGUE of the simulation launch (the first E threads of
 * the CTA, one environment each), and its adjoint as the PROLOGUE of the adjoint launch: one launch per env.step() forward, one
 * backward.  Articulations without a tile kernel run the two launches back to back inside the call. */
typedef struct DfxEnvTransition {
    int kind;                           /* 1: walker (`walker` is read), 2: planar (`planar` is read) */
    DfxWalkerParams walker;
    DfxPlanarParams planar;
    const long long* progress;          /* [n] step counter BEFORE this step */
    const float* start_q;               /* [n*Q], [n*D]: the state a terminated environment restarts from */
    const float* start_qd;
    float* obs_before;                  /* outputs, as in dfx_walker_transition_forward */
    float* rew;
    long long* reset;
    float* q_next;
    float* qd_next;
    float* actions_next;
    long long* progress_next;
    float* obs_next;
} DfxEnvTransition;
/* q_sim [n*Q], qd_sim [n*D]: the state right after the simulation step (before the masked re-initialisation; the adjoint
 * reads it back); used [n*num_act]: the env's `actions` (required). */
int dfx_env_step_forward(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                         const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                         float* used, float* q_sim, float* qd_sim, float* tape, const DfxEnvTransition* tr, void* stream);
int dfx_env_step_forward_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                            const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                            float* used, float* q_sim, float* qd_sim, float* tape, const DfxEnvTransition* tr, void* stream,
                            const DfxExternalWrench* wrench);
typedef struct DfxEnvTransitionAdj {
    int kind;
    DfxWalkerParams walker;
    DfxPlanarParams planar;
    const float* q_sim;                 /* saved by the forward call */
    const float* qd_sim;
    const float* used;
    const long long* reset;
    const float* g_obs_before;          /* cotangents of the six differentiable transition outputs (NULL == 0) */
    const float* g_rew;
    const float* g_q_next;
    const float* g_qd_next;
    const float* g_actions_next;
    const float* g_obs_next;
    float* gq_sim;                      /* workspace [n*Q], [n*D], [n*num_act]: the cotangents of (q_sim, qd_sim, used) on their */
    float* gqd_sim;                     /* way from the transition adjoint into the step adjoint (overwritten)                   */
    float* g_used;
} DfxEnvTransitionAdj;
/* -> gq, gqd, g_raw (overwritten), as dfx_step_backward_mapped */
int dfx_env_step_backward(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                          const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                          const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream);
int dfx_env_step_backward_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                             const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                             const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* wrench);

/* ---- recompute adjoint: backward WITHOUT a stored tape.  The forward then runs with tape == NULL (the no-grad launch) and
 * keeps nothing; each adjoint entry below re-runs the env-step's forward from its input state (q, qd) and actuation into a
 * workspace that holds ONE env-step's tape, then runs the adjoint of its stored-tape twin on it.  The forward is deterministic
 * (fixed-point scatter-adds), so the recomputed tape is the stored tape bit for bit and so are the cotangents: memory
 * O(one env-step) instead of O(horizon), for one extra forward per env-step in the backward.
 *
 * Workspace: dfx_recompute_workspace_floats(pack, n, substeps, mm_freq) floats, device memory, contents on entry ignored.  On
 * return it holds the recomputed tape in the tape's layout at offset 0 (dfx_tape_floats(pack, n, substeps, mm_freq) floats),
 * then the end state of the recomputed forward: q_out [n*Q] at offset dfx_tape_floats(...), qd_out [n*D] right after it.
 * It may be reused by the next call on the same stream.
 *
 * Tile kernels: ONE launch (the forward into the workspace and the adjoint in the same CTA).  Lane-group kernels, the A/B
 * variants of dfx_set_flags bit 6 and env-steps whose transition adjoint cannot be staged in the tile: the forward launch, then
 * the stored-tape entry on the workspace.  Arguments as the twin, with `tape` replaced by q [n*Q], qd [n*D] (the inputs of the
 * forward call, not modified) and `workspace`; a NULL q, qd or workspace is cudaErrorInvalidValue. */
long long dfx_recompute_workspace_floats(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq);
int dfx_step_backward_recompute(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                                const float* q, const float* qd, const float* act, const float* musc, float* workspace,
                                const float* gq_out, const float* gqd_out,
                                float* gq, float* gqd, float* gact, float* gmusc, void* stream);
int dfx_step_backward_mapped_recompute(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                                       const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                       float* workspace, const float* gq_out, const float* gqd_out, const float* g_used,
                                       float* gq, float* gqd, float* g_raw, void* stream);
int dfx_env_step_backward_recompute(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                                    const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                    float* workspace, const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream);
/* the three recompute entries with an external wrench (DfxExternalWrench: the f_ext of the forward call; NULL: none) */
int dfx_step_backward_recompute_ex(const dfx_pack_t* pack, int num_envs, int substeps, int mm_freq, double dt,
                                   const float* q, const float* qd, const float* act, const float* musc, float* workspace,
                                   const float* gq_out, const float* gqd_out,
                                   float* gq, float* gqd, float* gact, float* gmusc, void* stream, const DfxExternalWrench* wrench);
int dfx_step_backward_mapped_recompute_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                                          const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                          float* workspace, const float* gq_out, const float* gqd_out, const float* g_used,
                                          float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* wrench);
int dfx_env_step_backward_recompute_ex(const dfx_pack_t* pack, int n, int substeps, int mm_freq, double dt,
                                       const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                       float* workspace, const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream,
                                       const DfxExternalWrench* wrench);

/* ---- link state: the pose and velocity of every link of (q, qd), differentiable -- the kinematics of one substep on its own
 * (reference eval_rigid_fk sim.py:1681 and the velocity half of eval_rigid_id sim.py:1845), in the layouts of the reference State
 * fields (model.py:360-388):
 *   body_X_sc [n*L*7]  link frame in world: position, quaternion xyzw;
 *   body_X_sm [n*L*7]  centre-of-mass frame X_sc * X_cm (its position is where DfxExternalWrench applies the force);
 *   body_v_s  [n*L*6]  spatial twist (w, v_o) in world axes, v_o the velocity of the body-fixed point at the world origin:
 *                      the centre of mass moves with v_o + w x X_sm.p.
 * Quaternions in q are used as given (not renormalised), so the adjoint has the component along |q|, as the step's.  The backward
 * recomputes the kinematics from (q, qd) and keeps nothing between the calls.  Both run on the kernel family the step entries use
 * for the pack, in the step's scratch layouts: an articulation the step fits, these fit.  Stream-ordered, no host synchronisation. */
/* link poses / velocities of (q, qd), reference State layouts; any output NULL: skip */
int dfx_link_state_forward(const dfx_pack_t* pack, int n, const float* q, const float* qd,
                           float* body_X_sc, float* body_X_sm, float* body_v_s, void* stream);
/* cotangents (NULL == 0) -> gq [n*Q], gqd [n*D] (overwritten; NULL: skip) */
int dfx_link_state_backward(const dfx_pack_t* pack, int n, const float* q, const float* qd,
                            const float* g_X_sc, const float* g_X_sm, const float* g_v_s,
                            float* gq, float* gqd, void* stream);

/* ---- contact state: what the ground does to the links at (q, qd), differentiable -- the step's penalty ground-contact model
 * (reference eval_rigid_contacts_art sim.py:1137) evaluated at the given state, which is exactly what the first substep of an
 * env-step from it applies.  All fp32, world axes, env-major:
 *   contact_f       [n*C*3]  force the ground exerts on the link at contact point k, in the Model's contact order (Model.collide,
 *                            contact_body0); zero for a point that does not penetrate, and for every point when the ground is off
 *                            (dfx_pack_set_gravity);
 *   contact_height  [n*C]    signed height of point k above the plane, (X_sc p0).y - contact_dist: negative when penetrating (the c
 *                            of the contact model), computed whether the ground is on or not;
 *   body_f_contact  [n*L*6]  per link, (tau, F) summed over its points: F = sum f_k, tau = sum (p_k - X_sm.p) x f_k, p_k the point
 *                            after the contact_dist shift (where the step applies it) -- the DfxExternalWrench convention, so it can
 *                            be passed back as f_ext unchanged.
 * Sign: inside the step the contact model's ftot is added into body_f_s, where it acts like the gravity and external terms that
 * f = f_b - (...) subtracts, so the physical force on the link is -ftot (upward when penetrating): that is what contact_f holds.
 * The backward recomputes the kinematics from (q, qd) and keeps nothing between the calls; the force's cotangent reaches (q, qd)
 * only through penetrating points, the height's through every point.  Both run on the kernels dfx_link_state_* use; every sum is
 * taken in a fixed order by one thread, so both are bit-reproducible.  With C == 0 the kernels still run when there is an output:
 * body_f_contact and the gradients are written as zero.  Stream-ordered, no host synchronisation. */
/* contact forces / heights / link wrenches of (q, qd); any output NULL: skip (all NULL: no launch, returns 0) */
int dfx_contact_state_forward(const dfx_pack_t* pack, int n, const float* q, const float* qd,
                              float* contact_f, float* contact_height, float* body_f_contact, void* stream);
/* cotangents (NULL == 0) -> gq [n*Q], gqd [n*D] (overwritten; NULL: skip; both NULL: no launch, returns 0) */
int dfx_contact_state_backward(const dfx_pack_t* pack, int n, const float* q, const float* qd,
                               const float* g_contact_f, const float* g_contact_height, const float* g_body_f_contact,
                               float* gq, float* gqd, void* stream);

/* ---- dynamics state: joint accelerations, joint forces and mass matrix of (q, qd, act, musc, f_ext), differentiable -- what the
 * first substep of an env-step from the state computes before it integrates (reference SemiImplicitIntegrator._simulate:
 * eval_rigid_tau, eval_crba, eval_solve).  All fp32, env-major, in the Model's dof order:
 *   joint_tau  [n*D]    State.joint_tau, the right-hand side of the solve: -S^T f of each joint's subtree (gravity, Coriolis and
 *                       centrifugal terms, ground contacts, muscles and the external wrench), plus the PD drive to target, plus act,
 *                       plus the joint-limit spring and damper; -f for a free joint.  NOT the actuator effort alone;
 *   H          [n*D*D]  joint-space inertia J^T M J, row-major, symmetric, WITHOUT the armature;
 *   joint_qdd  [n*D]    (H + diag(armature))^-1 joint_tau.
 * H is always built from the given q (substep 0 of an env-step always refactorises).  act [n*D], musc [n*M] (required when M > 0),
 * f_ext [n*L*6] in the DfxExternalWrench convention (NULL: no wrench).  The values are the derived dumps (DfxDerived joint_tau, H,
 * joint_qdd) of a one-substep env-step from the same inputs, bit for bit.
 *
 * Backward: g_qdd, g_tau, g_H (NULL == 0; g_H need not be symmetric -- only g_H + g_H^T enters) -> gq [n*Q], gqd [n*D],
 * gact [n*D], gmusc [n*M], g_f_ext [n*L*6] (overwritten; NULL: skip).  It re-runs a one-substep env-step from the inputs into
 * `workspace` (device memory, dfx_dynamics_workspace_floats(pack, n) floats -- dfx_recompute_workspace_floats(pack, n, 1, 1) when
 * the pack's tape is fp32 -- contents on entry ignored; its rows are fp32 whatever dfx_set_tape_dtype says) and runs the adjoint of
 * that substep's dynamics on it, seeded with the cotangents and without the integrator: nothing is kept between the calls.
 * Launches: forward one; backward one on the tile kernels (the forward into the workspace and the adjoint in the same CTA), two on
 * the lane-group kernels (dfx_step_forward_ex into the workspace, then the adjoint).  Both run on the kernel family the step
 * entries use (flag bit 6 of dfx_set_flags: the default tile kernels) and are bit-reproducible.  A NULL q, qd, act or workspace
 * (backward), or a NULL musc when M > 0, is cudaErrorInvalidValue; with every output NULL there is no launch and 0 is returned.
 * Stream-ordered, no host synchronisation. */
long long dfx_dynamics_workspace_floats(const dfx_pack_t* pack, int n);
int dfx_dynamics_state_forward(const dfx_pack_t* pack, int n, const float* q, const float* qd, const float* act, const float* musc,
                               const float* f_ext, float* joint_qdd, float* joint_tau, float* H, void* stream);
int dfx_dynamics_state_backward(const dfx_pack_t* pack, int n, const float* q, const float* qd, const float* act, const float* musc,
                                const float* f_ext, float* workspace, const float* g_qdd, const float* g_tau, const float* g_H,
                                float* gq, float* gqd, float* gact, float* gmusc, float* g_f_ext, void* stream);

/* ---- Jacobian state: the link Jacobians and bias accelerations of (q, qd), differentiable.  At a state of n environments (fp32,
 * environment-major):
 *   J        [n*L*6*D]  the reference's per-articulation model.J block (spatial_jacobian, spatial.h:691-738): row 6 i + r, column d
 *                       at (6 i + r) * D + d.  Column d of link i's rows is the motion subspace S_s[d] of dof d (the reference's
 *                       joint_S_s: a spatial (w, v_o) twist in world axes) when dof d belongs to link i or to one of its ancestors,
 *                       and exactly 0 otherwise.  So body_v_s[i] = J[i] qd (dfx_link_state_forward), and the columns of a free
 *                       joint are the identity for every link of its tree.  Quaternions in q are used as given, as the link state.
 *   body_a_s [n*L*6]    the reference State's body_a_s (eval_rigid_fk / eval_rigid_id, sim.py:1763): each link's spatial
 *                       acceleration with q'' = 0, i.e. J-dot qd, in the same (w, v_o) convention.  The full link acceleration is
 *                       J q'' + body_a_s, with q'' from dfx_dynamics_state_forward.
 * Point Jacobians.  A point p fixed to link i (e.g. its centre of mass, X_sm.p of the link state) moves with v_o + w x p, where
 * (w, v_o) = body_v_s[i].  With J_w the rows 0-2 and J_v the rows 3-5 of link i's block:
 *   dp/dt   = (J_v - [p]x J_w) qd,
 *   d2p/dt2 = (J_v - [p]x J_w) q'' + b,   b = body_a_s[i].v + body_a_s[i].w x p + w x (v_o + w x p),
 * b being the point's bias acceleration: the spatial acceleration a = (a_w, a_v) gives a point the acceleration
 * a_v + a_w x p + w x dp/dt, and the last term is the w x (w x p)-type term of the spatial convention.
 * Gradients: J depends on q only (its cotangent reaches gq); body_a_s on (q, qd).  The backward recomputes the kinematics from
 * (q, qd) and keeps nothing between the calls.  Both run on the kernel family the step entries use, in the step's scratch layouts (an
 * articulation the step fits, these fit), one launch each, and are bit-reproducible.  A NULL q or qd is cudaErrorInvalidValue; a
 * NULL output is skipped, a NULL cotangent is zero; with every output NULL there is no launch and 0 is returned.  Stream-ordered, no
 * host synchronisation. */
int dfx_jacobian_state_forward(const dfx_pack_t* pack, int n, const float* q, const float* qd, float* J, float* body_a_s, void* stream);
/* cotangents g_J [n*L*6*D], g_a_s [n*L*6] (NULL == 0) -> gq [n*Q], gqd [n*D] (overwritten; NULL: skip) */
int dfx_jacobian_state_backward(const dfx_pack_t* pack, int n, const float* q, const float* qd, const float* g_J, const float* g_a_s,
                                float* gq, float* gqd, void* stream);

/* Launch configuration knob: lanes cooperating on one environment (8, 16 or 32; 0 = auto). */
int dfx_set_group_size(int lanes);
/* Tuning flags (default 9; for A/B timing and tests).  Lane-group kernels: bit 1 (2) = extra CTA-wide barriers between
 * phases (instruction-cache locality; no longer a gain now that the task loops synchronise the CTA anyway); bit 2 (4) =
 * generic kernels instead of the size-specialised ones; bit 3 (8) = CTA-wide task loops for thin / sparse phases.
 * Bit 7 (128): tile kernels do not prefetch the next tape row into L2 during the adjoint (A/B timing).
 * Bit 6 (64): tile kernels of the large articulations use level-by-level tree recursions instead of path / subtree passes.
 * Bit 5 (32), read when a pack is CREATED: keep an articulation that has a tile kernel on the
 * lane-group kernels (the two families lay the tape out differently, DFX_QUERY_TAPE_TILE). */
int dfx_set_flags(int flags);
/* Tape storage, read when a pack is CREATED (tile kernels; ignored by the lane-group kernels): 0 (default) = fp32;
 * 1 = the link velocities, bias accelerations and total link wrenches a row carries for the adjoint (v, a, f_tot: 18 L of the
 * row's floats) are stored as bf16; the state (q, qd), q'', the link transforms and the motion subspace stay fp32 (they carry
 * positions: contact depths are millimetres of metre-sized numbers).  Cuts the tape by 20 % (Humanoid: 182 -> 144 KB per
 * env-step); arithmetic stays fp32.  The reference has no counterpart (it rejects fp16,
 * dflex/dflex/adjoint.py:1985); the gradient tolerance against the fp32 oracle is stated in tests/tolerances.py. */
int dfx_set_tape_dtype(int bf16);
/* Tile width knob, read when a pack is CREATED: 0 (default) = the widest tile kernel that exists for the articulation
 * (32 environments per CTA for Ant / Hopper / HalfCheetah / CartPole, 8 for the two humanoids); 8, 16 or 32 = only a
 * kernel of that width (an articulation without one falls back to the lane-group kernels).  For A/B timing and tests. */
int dfx_set_tile_envs(int envs);
/* Launch geometry the step kernel would use for this pack (host arithmetic, no GPU needed); `backward`: bit 0 the adjoint,
 * bit 1 (2) the external-wrench kernels (DfxExternalWrench).  out[1] == 0: that kernel does not fit one CTA's shared memory.
 * out[0] lanes per environment, out[1] environments per CTA, out[2] CTAs per SM (shared-memory / register bound),
 * out[3] dynamic shared memory per CTA in bytes, out[4] scratch floats per environment, out[5] bytes of the staged pack + CTA task list. */
int dfx_launch_plan(const dfx_pack_t* pack, int backward, int out[6]);
/* Number of kernels this library has launched since load (bench.py's gpu_launches claim). */
long long dfx_launch_count(void);
const char* dfx_version(void);
/* sizeof() of the parameter structs as THIS library was compiled (a binding's struct mirrors can check themselves against it):
 * 0 DfxModelDesc, 1 DfxDerived, 2 DfxWalkerParams, 3 DfxPlanarParams, 4 DfxActionMap, 5 DfxEnvTransition, 6 DfxEnvTransitionAdj,
 * 7 DfxExternalWrench;
 * anything else: -1. */
int dfx_abi_sizeof(int which);
/* Joint types the size-specialised tile kernels of an articulation with these sizes are COMPILED for (a bit mask as in
 * DFX_QUERY_JOINT_MASK; 31 = no tile kernel of these sizes, the run-time-generic lane-group kernels take every type).  A pack whose
 * links have any other joint type stays on the lane-group kernels (DFX_QUERY_TAPE_TILE == 0). */
int dfx_tile_joint_mask(int L, int D, int Q, int C, int M);

#ifdef __cplusplus
}
#endif
#endif /* DFX_H_ */
