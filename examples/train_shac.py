#!/usr/bin/env python
"""Short-Horizon Actor-Critic (SHAC) on the H100-native differentiable simulator -- example trainer.

The reference's ``algorithms/shac.py`` runs unchanged on the drop-in ``dflex`` package (INTEGRATION.md); this
file is an independently written, vectorised restatement of the same algorithm (Xu et al., ICLR 2022;
hyper-parameters of ``examples/cfg/shac/ant.yaml`` by default) whose per-step bookkeeping is sync-free
(masks instead of ``done.nonzero()`` + per-env Python loops, reference shac.py:223-289), so that a rollout never
waits on the host.  It exists to show end to end that the fused kernels' gradients train a policy and to
exercise the env-sharded multi-GPU path:

    python examples/train_shac.py --env AntEnv --num-envs 64 --max-epochs 2000
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_shac.py --num-envs 65536

Under torchrun each rank simulates ``num_envs / world_size`` environments and the actor / critic gradients and
the observation-normaliser moments are all-reduced (one NCCL all-reduce per rollout for the actor).
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import diffrl_b200.envs as envs  # noqa: E402
from diffrl_b200.parallel import allreduce_gradients, allreduce_moments  # noqa: E402

MM = {"AntEnv": 16, "HumanoidEnv": 48, "SNUHumanoidEnv": 8, "CartPoleSwingUpEnv": 4, "HopperEnv": 16, "CheetahEnv": 16}
PRESETS = {   # examples/cfg/shac/*.yaml of the reference (actor / critic learning rates are separate there)
    "AntEnv": dict(actor=[128, 64, 32], critic=[64, 64], lr=2e-3, critic_lr=2e-3, alpha=0.2, betas=(0.7, 0.95), epochs=2000, num_envs=64),
    "HumanoidEnv": dict(actor=[256, 128], critic=[128, 128], lr=2e-3, critic_lr=5e-4, alpha=0.995, betas=(0.7, 0.95), epochs=2000, num_envs=64),
    "SNUHumanoidEnv": dict(actor=[512, 256], critic=[256, 256], lr=2e-3, critic_lr=5e-4, alpha=0.995, betas=(0.7, 0.95), epochs=2000, num_envs=64),
    "HopperEnv": dict(actor=[128, 64, 32], critic=[64, 64], lr=2e-3, critic_lr=2e-4, alpha=0.2, betas=(0.7, 0.95), epochs=2000, num_envs=256),
    "CheetahEnv": dict(actor=[128, 64, 32], critic=[64, 64], lr=2e-3, critic_lr=2e-3, alpha=0.2, betas=(0.7, 0.95), epochs=2000, num_envs=64),
    "CartPoleSwingUpEnv": dict(actor=[64, 64], critic=[64, 64], lr=1e-2, critic_lr=1e-3, alpha=0.2, betas=(0.7, 0.95), epochs=500, num_envs=64),
}


def mlp(sizes, out_gain=np.sqrt(2), init_orthogonal=True):
    layers = []
    for i in range(len(sizes) - 1):
        lin = nn.Linear(sizes[i], sizes[i + 1])
        if init_orthogonal:
            nn.init.orthogonal_(lin.weight, gain=out_gain)
            nn.init.constant_(lin.bias, 0.0)
        layers.append(lin)
        if i < len(sizes) - 2:
            layers += [nn.ELU(), nn.LayerNorm(sizes[i + 1])]
    return nn.Sequential(*layers)


class Actor(nn.Module):
    """Gaussian policy with state-independent log-std (reference models/actor.py ActorStochasticMLP)."""

    def __init__(self, obs_dim, act_dim, units):
        super().__init__()
        self.mu = mlp([obs_dim] + units + [act_dim], init_orthogonal=False)
        self.logstd = nn.Parameter(torch.full((act_dim,), -1.0))

    def forward(self, obs, deterministic=False):
        mu = self.mu(obs)
        return mu if deterministic else mu + torch.randn_like(mu) * self.logstd.exp()


class RunningMeanStd:
    """Running moments kept in device tensors and updated IN PLACE (so that a captured CUDA graph sees them)."""

    def __init__(self, shape, device):
        self.mean = torch.zeros(shape, device=device)
        self.var = torch.ones(shape, device=device)
        self.count = torch.full((), 1e-4, device=device)

    @torch.no_grad()
    def update(self, x):
        n, m, v = allreduce_moments(x.shape[0], x.mean(0), x.var(0, unbiased=False))
        delta, tot = m - self.mean, self.count + n
        self.var.copy_((self.var * self.count + v * n + delta.square() * self.count * n / tot) / tot)
        self.mean.add_(delta * n / tot)
        self.count.copy_(tot)

    def frozen(self):
        """A snapshot (the statistics entering a rollout)."""
        f = RunningMeanStd.__new__(RunningMeanStd)
        f.mean, f.var, f.count = self.mean.clone(), self.var.clone(), self.count.clone()
        return f

    def normalize(self, x):
        return (x - self.mean) / torch.sqrt(self.var + 1e-5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="AntEnv", choices=sorted(PRESETS))
    ap.add_argument("--num-envs", type=int, default=0, help="total over all ranks (default: the reference's setting)")
    ap.add_argument("--max-epochs", type=int, default=0)
    ap.add_argument("--steps-num", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--log-interval", type=int, default=50)
    ap.add_argument("--out", default="")
    ap.add_argument("--profile-epochs", type=int, default=0,
                    help="time the phases of the last K epochs with CUDA events (eager mode): rollout forward, backward, the actor "
                         "all-reduce, the critic phase and its 64 all-reduces; written to --out as 'epoch_split_ms'")
    ap.add_argument("--graph", type=int, default=-1,
                    help="1: capture one whole training iteration (rollout, backward, actor step, critic training) in ONE "
                         "CUDA graph and replay it per epoch; 0: eager; default: on for single-GPU runs")
    args = ap.parse_args()
    cfg = PRESETS[args.env]

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.distributed.init_process_group("nccl", device_id=dev)
    total_envs = args.num_envs or cfg["num_envs"]
    n = total_envs // world
    max_epochs = args.max_epochs or cfg["epochs"]
    T, gamma, lam = args.steps_num, 0.99, 0.95
    torch.manual_seed(args.seed)              # identical initial weights on every rank
    np.random.seed(args.seed)

    env = getattr(envs, args.env)(num_envs=n, device=str(dev), seed=args.seed + rank, episode_length=1000, no_grad=False,
                                  stochastic_init=True, MM_caching_frequency=MM[args.env])
    obs_dim, act_dim, ep_len = env.num_obs, env.num_actions, env.episode_length
    actor = Actor(obs_dim, act_dim, cfg["actor"]).to(dev)
    critic = mlp([obs_dim] + cfg["critic"] + [1]).to(dev)
    target_critic = copy.deepcopy(critic)
    torch.manual_seed(args.seed + 1000 * (rank + 1))   # different exploration noise / resets per rank
    use_graph = (world == 1) if args.graph < 0 else bool(args.graph)
    # (a tensor lr can change under a captured graph)
    a_opt = torch.optim.Adam(actor.parameters(), lr=torch.tensor(cfg["lr"], device=dev) if use_graph else cfg["lr"],
                             betas=cfg["betas"], capturable=use_graph)
    c_opt = torch.optim.Adam(critic.parameters(), lr=torch.tensor(cfg["critic_lr"], device=dev) if use_graph else cfg["critic_lr"],
                             betas=cfg["betas"], capturable=use_graph)
    obs_rms = RunningMeanStd((obs_dim,), dev)

    obs_buf = torch.zeros((T, n, obs_dim), device=dev)
    rew_buf, done_mask, next_vals = (torch.zeros((T, n), device=dev) for _ in range(3))
    fin_ret, fin_cnt = torch.zeros((), device=dev), torch.zeros((), device=dev)
    actor_loss_s = torch.zeros((), device=dev)
    history, t_start = [], time.time()
    env.clear_grad()
    env.reset()
    # everything carried from one iteration to the next lives in static tensors that are updated in place, so that the
    # same code runs eagerly and as a replayed CUDA graph
    carry = {"q": env.state.joint_q.detach().clone(), "qd": env.state.joint_qd.detach().clone(),
             "progress": env.progress_buf.clone(), "actions": env.actions.detach().clone(),
             "ep_ret": torch.zeros(n, device=dev), "ep_len": torch.zeros(n, device=dev)}

    class Split:
        """CUDA-event stopwatch of the phases of an iteration: mark(name) closes the segment that started at the previous mark."""
        def __init__(self):
            self.on, self.marks, self.total, self.count = False, [], {}, 0

        def mark(self, name):
            if self.on:
                ev = torch.cuda.Event(enable_timing=True)
                ev.record()
                self.marks.append((name, ev))

        def close(self):
            if not self.on or not self.marks:
                return
            torch.cuda.synchronize()
            for (_, e0), (name, e1) in zip(self.marks[:-1], self.marks[1:]):
                self.total[name] = self.total.get(name, 0.0) + e0.elapsed_time(e1)
            self.marks, self.count = [], self.count + 1

    split = Split()

    def train_iteration():
        # ---------------------------------------------------------------- actor: short-horizon rollout
        split.mark("start")
        a_opt.zero_grad(set_to_none=True)
        frozen = obs_rms.frozen()                         # normalise with the statistics entering the rollout
        env.state = env.model.state()                     # == env.initialize_trajectory() on the carried state
        env.state.joint_q, env.state.joint_qd = carry["q"].clone(), carry["qd"].clone()
        env.progress_buf, env.actions = carry["progress"].clone(), carry["actions"].clone()
        env.calculateObservations()
        obs = env.obs_buf
        ep_ret, ep_len_cnt = carry["ep_ret"].clone(), carry["ep_len"].clone()
        obs_rms.update(obs)
        obs = frozen.normalize(obs)
        rew_acc = torch.zeros(n, device=dev)
        disc = torch.ones(n, device=dev)
        actor_loss = torch.zeros((), device=dev)
        for i in range(T):
            obs_buf[i] = obs.detach()
            obs, rew, done, extra = env.step(torch.tanh(actor(obs)))
            obs_rms.update(obs)
            obs = frozen.normalize(obs)
            done_b = done.bool()
            ep_len_cnt = ep_len_cnt + 1
            ep_ret = ep_ret + rew.detach()
            before = extra["obs_before_reset"]
            v = target_critic(obs).squeeze(-1)
            v_term = target_critic(frozen.normalize(before)).squeeze(-1)
            invalid = (~torch.isfinite(before)).any(-1) | (before.abs() > 1e6).any(-1)
            early = ep_len_cnt < ep_len                    # terminated before the time limit -> no bootstrap
            nv = torch.where(done_b, torch.where(early | invalid, torch.zeros_like(v), v_term), v)
            rew_acc = rew_acc + disc * rew
            if i < T - 1:
                actor_loss = actor_loss + torch.where(done_b, -rew_acc - gamma * disc * nv, torch.zeros_like(nv)).sum()
            else:
                actor_loss = actor_loss + (-rew_acc - gamma * disc * nv).sum()
            disc = torch.where(done_b, torch.ones_like(disc), disc * gamma)
            rew_acc = torch.where(done_b, torch.zeros_like(rew_acc), rew_acc)
            with torch.no_grad():
                rew_buf[i] = rew
                done_mask[i] = done_b.float() if i < T - 1 else 1.0
                next_vals[i] = nv
                fin_ret.add_((ep_ret * done_b).sum())
                fin_cnt.add_(done_b.sum())
                ep_ret = torch.where(done_b, torch.zeros_like(ep_ret), ep_ret)
                ep_len_cnt = torch.where(done_b, torch.zeros_like(ep_len_cnt), ep_len_cnt)
        actor_loss = actor_loss / (T * n * world)          # global batch normalisation (reference shac.py:291)
        split.mark("rollout_forward")
        actor_loss.backward()
        split.mark("rollout_backward")
        allreduce_gradients(list(actor.parameters()), average=False)     # the one collective per rollout
        split.mark("actor_allreduce")
        torch.nn.utils.clip_grad_norm_(actor.parameters(), 1.0)
        a_opt.step()
        split.mark("actor_step")
        with torch.no_grad():
            actor_loss_s.copy_(actor_loss.detach())
            carry["q"].copy_(env.state.joint_q.detach().view(-1)); carry["qd"].copy_(env.state.joint_qd.detach().view(-1))
            carry["progress"].copy_(env.progress_buf); carry["actions"].copy_(env.actions.detach())
            carry["ep_ret"].copy_(ep_ret); carry["ep_len"].copy_(ep_len_cnt)
        # ---------------------------------------------------------------- critic: TD(lambda) targets
        with torch.no_grad():
            Ai, Bi, lm = (torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.ones(n, device=dev))
            targets = torch.zeros((T, n), device=dev)
            for i in reversed(range(T)):
                lm = lm * lam * (1.0 - done_mask[i]) + done_mask[i]
                Ai = (1.0 - done_mask[i]) * (lam * gamma * Ai + gamma * next_vals[i] + (1.0 - lm) / (1.0 - lam) * rew_buf[i])
                Bi = gamma * (next_vals[i] * done_mask[i] + Bi * (1.0 - done_mask[i])) + rew_buf[i]
                targets[i] = (1.0 - lam) * Ai + lm * Bi
            flat_obs, flat_tgt = obs_buf.view(-1, obs_dim), targets.view(-1)
        batch = flat_obs.shape[0] // 4
        for _ in range(16):
            perm = torch.rand(flat_obs.shape[0], device=dev).argsort()       # (graph-capturable random permutation)
            for b in range(4):
                idx = perm[b * batch:(b + 1) * batch]
                c_opt.zero_grad(set_to_none=True)
                loss_c = (critic(flat_obs[idx]).squeeze(-1) - flat_tgt[idx]).square().mean()
                loss_c.backward()
                for p in critic.parameters():
                    p.grad.nan_to_num_(0.0, 0.0, 0.0)
                split.mark("critic_compute")
                allreduce_gradients(list(critic.parameters()), average=True)      # 64 per epoch (reference shac.py:463-476), one flat buffer each
                split.mark("critic_allreduce")
                torch.nn.utils.clip_grad_norm_(critic.parameters(), 1.0)
                c_opt.step()
        with torch.no_grad():
            for p, pt in zip(critic.parameters(), target_critic.parameters()):
                pt.mul_(cfg["alpha"]).add_((1.0 - cfg["alpha"]) * p)
        split.mark("critic_compute")

    graph, warm_epochs = None, 3
    for epoch in range(max_epochs):
        for opt, base in ((a_opt, cfg["lr"]), (c_opt, cfg["critic_lr"])):      # linear schedule, each from its own base (shac.py:420-431)
            lr = (1e-5 - base) * epoch / max_epochs + base
            for group in opt.param_groups:
                if use_graph:
                    group["lr"].fill_(lr)
                else:
                    group["lr"] = lr
        split.on = (not use_graph) and args.profile_epochs > 0 and epoch >= max_epochs - args.profile_epochs
        if not use_graph:
            train_iteration()
            split.close()
        elif epoch < warm_epochs:         # warm-up on a side stream, as the capture will run on one
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                train_iteration()
            torch.cuda.current_stream(dev).wait_stream(side)
        else:
            if graph is None:             # the first iterations ran eagerly (allocator / optimizer state warm-up)
                import gc
                torch.cuda.synchronize()
                gc.collect()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    train_iteration()
            graph.replay()
        # ---------------------------------------------------------------- logging (one host sync per interval)
        if (epoch + 1) % args.log_interval == 0 or epoch == max_epochs - 1:
            stats = torch.stack([fin_ret, fin_cnt])
            if world > 1:
                torch.distributed.all_reduce(stats)
            ret = float(stats[0] / stats[1].clamp(min=1))
            steps = (epoch + 1) * T * n * world
            if rank == 0:
                rec = {"epoch": epoch + 1, "env_steps": steps, "mean_episode_return": ret, "episodes": int(stats[1]),
                       "actor_loss": float(actor_loss_s), "wall_s": round(time.time() - t_start, 1),
                       "env_steps_per_s_training": round(steps / (time.time() - t_start))}
                history.append(rec)
                print(json.dumps(rec), flush=True)
            fin_ret.zero_(); fin_cnt.zero_()
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            rec = {"env": args.env, "num_envs": total_envs, "world": world, "cuda_graph": bool(use_graph), "history": history}
            if split.count:
                rec["epoch_split_ms"] = {k: v / split.count for k, v in split.total.items()}
                rec["epoch_split_ms"]["epochs_timed"] = split.count
                rec["epoch_split_note"] = ("rank 0, CUDA events: rollout_forward = %d x (policy + env.step + critic bootstrap), rollout_backward = "
                                           "loss.backward(), actor_allreduce = the ONE policy-gradient all-reduce of the rollout, critic_allreduce = "
                                           "sum of the 64 per-minibatch critic all-reduces" % T)
            json.dump(rec, f, indent=1)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
