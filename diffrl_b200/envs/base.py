"""``DFlexEnv`` and the shared step / reset / trajectory machinery of the differentiable envs.

Interface mirror of the reference ``envs/dflex_env.py:21-109`` and of the per-env boiler-plate that
every reference env repeats (``envs/ant.py:156-264``): same constructor arguments, attributes
(``obs_buf``, ``rew_buf``, ``reset_buf``, ``progress_buf``, ``actions``, ``state``, ``model``,
``integrator`` ...) and methods (``step``, ``reset``, ``clear_grad``, ``initialize_trajectory``,
``get_checkpoint``, ``calculateObservations``, ``calculateReward``), so ``algorithms/shac.py`` /
``bptt.py`` drive these classes exactly like the reference's.  Differences, all outside the numerics:

* the Model is built ONCE from a single-articulation asset and tiled (reference: one MJCF/URDF/SNU
  parse per environment in a Python loop -- minutes at 65 536 envs);
* ``gym.spaces`` is optional.
"""
import os

import numpy as np
import torch

import diffrl_b200.dflex_api as df

ASSET_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "assets")


class _Box:
    def __init__(self, low, high):
        self.low, self.high, self.shape = low, high, low.shape


class DFlexEnv:
    def __init__(self, num_envs, num_obs, num_act, episode_length, MM_caching_frequency=1, seed=0, no_grad=True,
                 render=False, device="cuda:0"):
        self.seed = seed
        self.no_grad = no_grad
        df.config.no_grad = self.no_grad
        self.episode_length = episode_length
        self.device = device
        self.visualize = render
        if render:
            raise NotImplementedError("USD rendering is outside the hot-path package; use render=False")
        self.sim_time = 0.0
        self.num_frames = 0
        self.num_environments = num_envs
        self.num_agents = 1
        self.MM_caching_frequency = MM_caching_frequency
        self.num_observations = num_obs
        self.num_actions = num_act
        self.obs_space = _Box(np.ones(num_obs) * -np.inf, np.ones(num_obs) * np.inf)
        self.act_space = _Box(np.ones(num_act) * -1.0, np.ones(num_act) * 1.0)
        dev = self.device
        self.obs_buf = torch.zeros((num_envs, num_obs), device=dev, dtype=torch.float)
        self.rew_buf = torch.zeros(num_envs, device=dev, dtype=torch.float)
        self.reset_buf = torch.ones(num_envs, device=dev, dtype=torch.long)
        self.termination_buf = torch.zeros(num_envs, device=dev, dtype=torch.long)
        self.progress_buf = torch.zeros(num_envs, device=dev, dtype=torch.long)
        self.actions = torch.zeros((num_envs, num_act), device=dev, dtype=torch.float)
        self.extras = {}

    # ---- properties of the reference interface
    def get_number_of_agents(self):
        return self.num_agents

    @property
    def observation_space(self):
        return self.obs_space

    @property
    def action_space(self):
        return self.act_space

    @property
    def num_envs(self):
        return self.num_environments

    @property
    def num_acts(self):
        return self.num_actions

    @property
    def num_obs(self):
        return self.num_observations

    def get_state(self):
        return self.state.joint_q.clone(), self.state.joint_qd.clone()

    def reset_with_state(self, init_joint_q, init_joint_qd, env_ids=None, force_reset=True):
        if env_ids is None and force_reset:
            env_ids = torch.arange(self.num_envs, dtype=torch.long, device=self.device)
        if env_ids is not None:
            self.state.joint_q = self.state.joint_q.clone()
            self.state.joint_qd = self.state.joint_qd.clone()
            self.state.joint_q.view(self.num_envs, -1)[env_ids, :] = init_joint_q.view(-1, self.num_joint_q)[env_ids, :].clone()
            self.state.joint_qd.view(self.num_envs, -1)[env_ids, :] = init_joint_qd.view(-1, self.num_joint_qd)[env_ids, :].clone()
            self.progress_buf[env_ids] = 0
            self.calculateObservations()
        return self.obs_buf

    # ---- model construction shared by all envs
    def _build_model(self, asset_name):
        """Tile the single-articulation asset to num_envs copies (bit-identical to what the reference's
        per-env parse loop produces, tests/test_envs_cpu.py)."""
        arrays = dict(np.load(os.path.join(ASSET_DIR, asset_name + ".npz")))
        self.model = df.model_from_articulation(arrays, self.num_environments, self.device, ground=self.ground,
                                                gravity=(0.0, -9.81, 0.0))
        self.integrator = df.sim.SemiImplicitIntegrator()
        self.state = self.model.state()
        return arrays

    # ---- step / reset skeleton (reference envs/ant.py:156-190 and siblings)
    def _apply_actions(self, actions):
        raise NotImplementedError

    def _nan_guard(self, actions, state=None):
        """The reference's "ugly fix": zero NaN/Inf gradients flowing into the state (humanoid.py:196-206)."""
        def hook(grad):
            return torch.nan_to_num(grad, 0.0, 0.0, 0.0)
        for t in ((self.state.joint_q, self.state.joint_qd, actions) if state is None else (state.joint_q, state.joint_qd, actions)):
            if t.requires_grad:
                t.register_hook(hook)

    nan_guard = False
    external_wrench = None     # set_external_wrench
    clone_actions = True
    # True: terminated environments are re-initialised with a mask (torch.where) instead of the reference's
    # reset_buf.nonzero() + indexed writes, so env.step() never synchronises the host with the GPU.
    sync_free_reset = True
    # True: the policy-output -> actuation map is folded into the simulation launch (dfx_step_forward_mapped)
    fused_action_map = True
    # True: the transition (progress counter, observation, reward, termination, masked re-initialisation, next observation) rides
    # inside the simulation launch as its epilogue, and its adjoint as the prologue of the adjoint launch (dfx_env_step_forward /
    # _backward): env.step() is ONE launch forward and ONE backward
    single_launch_step = True

    def set_external_wrench(self, w):
        """External wrenches on the links, applied on every following step until changed: ``w`` [num_envs, L, 6] fp32 on the
        env's device -- per link (torque, force), both in world axes, the force applied at the link's centre of mass (MuJoCo's
        ``xfrc_applied`` convention; include/dfx.h DfxExternalWrench) -- or None for none.  Differentiable: a ``w`` that
        requires grad receives the gradient of whatever the rollout's loss is.  ``GraphedRollout`` refuses an env with a
        wrench set."""
        if w is not None:
            from ..dflex_api.sim import _engine_for
            from ..engine import check_wrench
            engine = _engine_for(self.model)
            if tuple(w.shape) != (self.num_envs, engine.L, 6):
                raise ValueError("external wrench has shape %s, expected [%d, %d, 6]" % (tuple(w.shape), self.num_envs, engine.L))
            check_wrench(engine, w)
        self.external_wrench = w

    def link_state(self):
        """``diffrl_b200.link_state`` of ``self.state``, the state the next step starts from: ``LinkState(body_X_sc, body_X_sm,
        body_v_s)``, [num_envs, L, 7 / 7 / 6].  Differentiable: its gradient reaches the actions and the start state through
        whichever step op produced ``self.state``."""
        from .. import link_state
        return link_state(self.model, self.state.joint_q, self.state.joint_qd)

    def contact_state(self):
        """``diffrl_b200.contact_state`` of ``self.state``, the state the next step starts from: ``ContactState(contact_f,
        contact_height, body_f_contact)``, [num_envs, C, 3], [num_envs, C], [num_envs, L, 6].  Differentiable: its gradient reaches
        the actions and the start state through whichever step op produced ``self.state``."""
        from .. import contact_state
        return contact_state(self.model, self.state.joint_q, self.state.joint_qd)

    def jacobian_state(self):
        """``diffrl_b200.jacobian_state`` of ``self.state``, the state the next step starts from: ``JacobianState(J, body_a_s)``,
        [num_envs, L, 6, D], [num_envs, L, 6].  Differentiable: its gradient reaches the actions and the start state through
        whichever step op produced ``self.state``."""
        from .. import jacobian_state
        return jacobian_state(self.model, self.state.joint_q, self.state.joint_qd)

    def dynamics_state(self, actions):
        """``diffrl_b200.dynamics_state`` of ``self.state`` under the actuation the env's action map makes of the policy output
        ``actions`` [num_envs, num_actions] (``_action_map()`` through ``ActionMapFunction``: clipped, scaled, into joint_act or the
        muscle activations, the other one zero, as the fused step forms them) and with the env's external wrench: what the next
        ``step(actions)`` starts with.  ``DynamicsState(joint_qdd, joint_tau, H)``, [num_envs, D], [num_envs, D], [num_envs, D, D].
        Differentiable: its gradient reaches ``actions``, the wrench and, through whichever step op produced ``self.state``, the
        start state -- so a reward can penalise the torques or accelerations of the action about to be taken."""
        from .. import dynamics_state
        from ..env_ops import ActionMapFunction
        if getattr(self, "_amap", None) is None:
            self._amap = self._action_map()
            self._tparams = self._transition_params()
        width, offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = self._amap
        n = self.num_envs
        _, drive = ActionMapFunction.apply(n, width, offset, pre_scale, pre_bias, drive_scale, strength, actions.view((n, self.num_actions)))
        act = None if is_muscle else drive
        musc = drive if is_muscle else None
        return dynamics_state(self.model, self.state.joint_q, self.state.joint_qd, act, musc, self.external_wrench)

    def _attach_wrench(self, state):
        """The step reads the wrench from its input State (``body_f_ext``)."""
        if self.external_wrench is None:
            state.__dict__.pop("body_f_ext", None)
        else:
            state.body_f_ext = self.external_wrench

    def step(self, actions):
        actions = actions.view((self.num_envs, self.num_actions))
        actions = self._preprocess_actions(torch.clip(actions, -1.0, 1.0))
        if self.nan_guard:
            self._nan_guard(actions)
        self.actions = actions.clone() if self.clone_actions else actions
        self._apply_actions(actions)
        self._attach_wrench(self.state)
        self.state = self.integrator.forward(self.model, self.state, self.sim_dt, self.sim_substeps, self.MM_caching_frequency)
        self.sim_time += self.sim_dt
        self.reset_buf = torch.zeros_like(self.reset_buf)
        self.progress_buf += 1
        self.num_frames += 1
        self._observe_and_reward()
        if not self.no_grad:
            self.obs_buf_before_reset = self.obs_buf.clone()
            self.extras = {"obs_before_reset": self.obs_buf_before_reset, "episode_end": self.termination_buf}
        if self.sync_free_reset and hasattr(self, "_start_state"):
            self._reset_masked(self.reset_buf)
        else:
            env_ids = self.reset_buf.nonzero(as_tuple=False).squeeze(-1)
            if len(env_ids) > 0:
                self.reset(env_ids)
        return self.obs_buf, self.rew_buf, self.reset_buf, self.extras

    def _fused_step(self, actions):
        """env.step() through the fused env layer.  Default (``single_launch_step``): ONE launch forward and ONE backward --
        ``dfx_env_step_forward / _backward``: the policy output -> actuation map is folded into the simulation launch and the
        transition (progress counter, observation, reward, termination, masked re-initialisation, next observation) runs as
        its epilogue, the transition adjoint as the prologue of the adjoint launch.  Otherwise two launches (mapped step +
        ``dfx_walker_transition_*`` / ``dfx_planar_transition_*``; also what no-grad envs use, whose integrator works in place) or
        three (``fused_action_map = False``: ``dfx_action_map_*`` on its own).  The env provides ``_action_map()`` and
        ``_transition_params()``; results equal the op-by-op ``step`` (tests/test_gpu_envs.py)."""
        from ..env_ops import ActionMapFunction, WalkerTransitionFunction
        n = self.num_envs
        if getattr(self, "_amap", None) is None:
            self._amap = self._action_map()
            self._tparams = self._transition_params()
        width, offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = self._amap
        self._attach_wrench(self.state)
        if self.single_launch_step and self.fused_action_map and not self.no_grad:
            from ..dflex_api.sim import fused_env_step
            start_q, start_qd = self._start_state()
            # nan_guard (the reference's "ugly fix", humanoid.py:196-206: NaN / Inf gradients flowing into the state and the
            # clipped actions become 0) is applied to the op's input cotangents inside its backward
            self.state, (obs_before, self.rew_buf, self.reset_buf, self.actions, self.progress_buf, self.obs_buf) = fused_env_step(
                self.model, self.state, self.sim_dt, self.sim_substeps, self.MM_caching_frequency, actions.view((n, self.num_actions)),
                (offset, pre_scale, pre_bias, drive_scale, strength, is_muscle), self._tparams, self.progress_buf, start_q, start_qd,
                nan_guard=self.nan_guard)
            self.sim_time += self.sim_dt
            self.num_frames += 1
            self.obs_buf_before_reset = obs_before
            self.extras = {"obs_before_reset": obs_before, "episode_end": self.termination_buf}
            return self.obs_buf, self.rew_buf, self.reset_buf, self.extras
        if self.fused_action_map and not self.no_grad:
            # the action map rides inside the simulation launch (dfx_step_forward_mapped): 2 launches per step instead of 3
            from ..dflex_api.sim import fused_mapped_forward
            state_in = self.state
            self.state, used = fused_mapped_forward(self.model, state_in, self.sim_dt, self.sim_substeps, self.MM_caching_frequency,
                                                    actions.view((n, self.num_actions)),
                                                    (offset, pre_scale, pre_bias, drive_scale, strength, is_muscle))
            if self.nan_guard:
                self._nan_guard(used, state_in)
            self.actions = used
        else:
            used, drive = ActionMapFunction.apply(n, width, offset, pre_scale, pre_bias, drive_scale, strength,
                                                  actions.view((n, self.num_actions)))
            if self.nan_guard:
                self._nan_guard(used)
            self.actions = used
            if is_muscle:
                self.model.muscle_activation = drive
            else:
                self.state.joint_act = drive
            self.state = self.integrator.forward(self.model, self.state, self.sim_dt, self.sim_substeps, self.MM_caching_frequency)
        self.sim_time += self.sim_dt
        self.num_frames += 1
        start_q, start_qd = self._start_state()
        (obs_before, self.rew_buf, self.reset_buf, q_next, qd_next, self.actions, self.progress_buf,
         self.obs_buf) = WalkerTransitionFunction.apply(self._tparams, n, self.progress_buf, start_q, start_qd,
                                                        self.state.joint_q, self.state.joint_qd, self.actions)
        self.state.joint_q, self.state.joint_qd = q_next.view(-1), qd_next.view(-1)
        if not self.no_grad:
            self.obs_buf_before_reset = obs_before
            self.extras = {"obs_before_reset": obs_before, "episode_end": self.termination_buf}
        return self.obs_buf, self.rew_buf, self.reset_buf, self.extras

    def _reset_masked(self, reset_buf):
        """Re-initialise terminated environments without reading reset_buf on the host: the start state is formed
        for every row (``_start_state()``: the same distributions as ``_reset_state``) and selected by mask."""
        n = self.num_envs
        flag = reset_buf.bool()
        mask = flag.unsqueeze(-1)
        start_q, start_qd = self._start_state()
        self.state.joint_q = torch.where(mask, start_q, self.state.joint_q.view(n, -1)).view(-1)
        self.state.joint_qd = torch.where(mask, start_qd, self.state.joint_qd.view(n, -1)).view(-1)
        if self.clone_actions:
            self.actions = torch.where(mask, torch.zeros_like(self.actions), self.actions)
        self.progress_buf = torch.where(flag, torch.zeros_like(self.progress_buf), self.progress_buf)
        self.calculateObservations()

    def _observe_and_reward(self):
        self.calculateObservations()
        self.calculateReward()

    def _preprocess_actions(self, actions):
        return actions

    def reset(self, env_ids=None, force_reset=True):
        if env_ids is None and force_reset:
            env_ids = torch.arange(self.num_envs, dtype=torch.long, device=self.device)
        if env_ids is not None:
            # clone so that the in-place writes below do not touch tensors saved by autograd
            self.state.joint_q = self.state.joint_q.clone()
            self.state.joint_qd = self.state.joint_qd.clone()
            self._reset_state(env_ids)
            if self.clone_actions:
                self.actions = self.actions.clone()
                self.actions[env_ids, :] = torch.zeros((len(env_ids), self.num_actions), device=self.device, dtype=torch.float)
            self.progress_buf[env_ids] = 0
            self.calculateObservations()
        return self.obs_buf

    def clear_grad(self, checkpoint=None):
        """Cut the graph between the current state and everything before it (ant.py:230-245)."""
        with torch.no_grad():
            if checkpoint is None:
                checkpoint = self.get_checkpoint()
            q, qd = checkpoint["joint_q"].clone(), checkpoint["joint_qd"].clone()
            self.state = self.model.state()
            self.state.joint_q, self.state.joint_qd = q, qd
            self.actions = checkpoint["actions"].clone()
            self.progress_buf = checkpoint["progress_buf"].clone()

    def initialize_trajectory(self):
        self.clear_grad()
        self.calculateObservations()
        return self.obs_buf

    def get_checkpoint(self):
        return {"joint_q": self.state.joint_q.clone(), "joint_qd": self.state.joint_qd.clone(),
                "actions": self.actions.clone(), "progress_buf": self.progress_buf.clone()}

    def render(self, mode="human"):
        return None

    def _invalid_state_mask(self):
        """Envs whose observation / state went NaN, Inf or > 1e6 (humanoid.py:361-366)."""
        q = self.state.joint_q.view(self.num_environments, -1)
        qd = self.state.joint_qd.view(self.num_environments, -1)
        bad = (~torch.isfinite(self.obs_buf)).any(-1) | (~torch.isfinite(q)).any(-1) | (~torch.isfinite(qd)).any(-1)
        return bad | (q.abs() > 1e6).any(-1) | (qd.abs() > 1e6).any(-1)
