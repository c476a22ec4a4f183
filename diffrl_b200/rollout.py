"""CUDA-graphed differentiable rollouts.

``env.step`` is launch-bound once the simulation kernels take a few hundred microseconds: a 32-step SHAC
rollout issues ~1 500 small launches (sim step, fused epilogue, masked reset, autograd bookkeeping) from
Python.  ``GraphedRollout`` captures ``horizon`` env-steps, the loss and its backward pass into ONE CUDA
graph (the env layer is sync-free: masked resets, no ``nonzero()``), including the host->device copy of
the actions and the device->host copies of the loss and the action gradients, and replays it:

    roll = GraphedRollout(env, horizon=32)
    loss, grad_actions = roll(host_actions)        # host_actions: pinned [horizon, num_envs, num_actions]

Capture is exercised for all six envs (tests/test_gpu_envs.py).  Anything the rollout touches must be free of autograd
leaves created on another stream (e.g. a grad-requiring reset state): the engine would synchronise with that stream
and invalidate the capture.

Each call starts from the env's current state (``env.state.joint_q/qd``, ``progress_buf``, last actions)
and leaves the env at the end of the rollout with the graph cut (as ``env.clear_grad()`` would), so
consecutive calls chain like SHAC's short-horizon windows (reference algorithms/shac.py:169-292).
"""
import torch


class GraphedRollout:
    def __init__(self, env, horizon, reward_weight=None, warmup=2):
        if torch.device(env.device).type != "cuda":
            raise RuntimeError("GraphedRollout needs a CUDA environment")
        if env.no_grad:
            raise RuntimeError("GraphedRollout differentiates the rollout: construct the env with no_grad=False")
        if getattr(env, "external_wrench", None) is not None:
            raise RuntimeError("GraphedRollout does not capture external wrenches: call env.set_external_wrench(None) first")
        if not getattr(env, "sync_free_reset", False) or not hasattr(env, "_start_state"):
            raise RuntimeError("%s resets through reset_buf.nonzero(), which cannot be captured" % type(env).__name__)
        self.env, self.T = env, int(horizon)
        dev = torch.device(env.device)
        n, a = env.num_envs, env.num_actions
        self.device = dev
        # static inputs
        self.actions = torch.zeros((self.T, n, a), device=dev, requires_grad=True)
        self.q0 = env.state.joint_q.detach().clone()
        self.qd0 = env.state.joint_qd.detach().clone()
        self.progress0 = env.progress_buf.clone()
        self.prev_actions = env.actions.detach().clone()
        self.weight = None if reward_weight is None else reward_weight.to(dev)
        # pinned host mirrors of the outputs
        self.host_grad = torch.empty((self.T, n, a), dtype=torch.float32).pin_memory()
        self.host_loss = torch.empty((), dtype=torch.float32).pin_memory()
        self.host_actions = torch.empty((self.T, n, a), dtype=torch.float32).pin_memory()
        self.graph = None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.actions.grad = None
        self.graph = torch.cuda.CUDAGraph()
        import gc
        gc.collect()                      # nothing device-synchronising (e.g. a dead engine's cudaFree) may run mid-capture
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(self.graph):
                self._body()
        finally:
            if gc_was_enabled:
                gc.enable()
        torch.cuda.synchronize(dev)
        # The captured body ended by pointing the env at `final_*` tensors of the graph's private pool, and capture runs
        # no kernels: those were never written.  Put the env back where it was when the rollout was built, so that the
        # first roll(actions) really "starts from the env's current state" (q0 / qd0 / progress0 / prev_actions still
        # hold it: the warm-up bodies only read them).
        env.state = env.model.state()
        env.state.joint_q, env.state.joint_qd = self.q0.clone(), self.qd0.clone()
        env.progress_buf, env.actions = self.progress0.clone(), self.prev_actions.clone()
        with torch.no_grad():
            env.calculateObservations()

    def _body(self):
        env = self.env
        with torch.no_grad():
            self.actions.copy_(self.host_actions, non_blocking=True)
        # start from the static state buffers, graph cut (== env.clear_grad() on those values)
        env.state = env.model.state()
        env.state.joint_q = self.q0.clone()
        env.state.joint_qd = self.qd0.clone()
        env.progress_buf = self.progress0.clone()
        env.actions = self.prev_actions.clone()
        env.calculateObservations()
        obs_l, rew_l, done_l = [], [], []
        for t, a_t in enumerate(self.actions.unbind(0)):   # unbind: ONE stack in backward instead of T zero-filled selects
            obs, rew, done, _ = env.step(a_t)
            obs_l.append(obs); rew_l.append(rew); done_l.append(done)
        rew_all = torch.stack(rew_l)                       # one reduction for the whole window
        # (always through an explicit weight tensor: the cotangent of a bare .sum() is a stride-0 expand, which every step's
        #  transition adjoint would have to materialise with a copy kernel of its own; the product's cotangent is one dense [T, N]
        #  tensor whose per-step slices are contiguous views)
        if self.weight is None:
            self.weight = torch.ones_like(rew_all)
        loss = (rew_all * self.weight).sum()
        self.actions.grad = None
        loss.backward()
        self.obs, self.rew, self.done = torch.stack(obs_l).detach(), rew_all.detach(), torch.stack(done_l)
        self.loss = loss.detach()
        self.final_q = env.state.joint_q.detach()
        self.final_qd = env.state.joint_qd.detach()
        self.final_progress = env.progress_buf
        self.final_actions = env.actions.detach()
        self.host_grad.copy_(self.actions.grad, non_blocking=True)
        self.host_loss.copy_(self.loss, non_blocking=True)
        # leave nothing on the env that keeps this body's autograd graph alive: the next body (the captured one after
        # the warm-ups) must build a fresh AccumulateGrad node for self.actions on ITS stream -- a stale node makes the
        # engine synchronise with the warm-up stream, which invalidates a capture
        env.state.joint_q, env.state.joint_qd = self.final_q, self.final_qd
        env.actions = self.final_actions
        env.obs_buf, env.rew_buf = env.obs_buf.detach(), env.rew_buf.detach()
        env.extras = {}
        musc = getattr(env.model, "muscle_activation", None)
        if musc is not None and musc.requires_grad:
            env.model.muscle_activation = musc.detach()
        if hasattr(env, "obs_buf_before_reset"):
            env.obs_buf_before_reset = env.obs_buf_before_reset.detach()
        del loss, rew_all, obs_l, rew_l, done_l

    def __call__(self, host_actions=None, sync=True):
        """Replay the captured rollout.  ``host_actions``: [T, N, A] tensor, copied into the pinned staging buffer
        ``self.host_actions`` the graph's H2D copy reads; pass None after writing the actions into
        ``self.host_actions`` directly (saves the host-side copy).  Returns (loss, grad_actions) as pinned host
        tensors (valid after the sync)."""
        env = self.env
        if host_actions is not None and host_actions is not self.host_actions:
            self.host_actions.copy_(host_actions)
        with torch.no_grad():
            # chain from where the env currently is
            self.q0.copy_(env.state.joint_q.detach().view(-1))
            self.qd0.copy_(env.state.joint_qd.detach().view(-1))
            self.progress0.copy_(env.progress_buf)
            self.prev_actions.copy_(env.actions.detach())
        self.graph.replay()
        # leave the env at the end of the rollout, detached
        env.state = env.model.state()
        env.state.joint_q, env.state.joint_qd = self.final_q, self.final_qd
        env.progress_buf, env.actions = self.final_progress, self.final_actions
        if sync:
            torch.cuda.current_stream(self.device).synchronize()
        return self.host_loss, self.host_grad
