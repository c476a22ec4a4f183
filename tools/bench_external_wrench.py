"""Cost of the external wrench (include/dfx.h DfxExternalWrench): kernel-path throughput of differentiable rollouts with and
without a wrench, in both adjoint modes.

    python tools/bench_external_wrench.py [--steps K] [--warmup W]

Prints ONE JSON line: the device (card name and power limit, read in the same run) and, for Ant 4096 x 32 and Humanoid 8192 x 32,
env-steps/s of the kernel path -- the engine's forward over the horizon, then the adjoints in reverse (tape mode: the stored-tape
adjoint; recompute mode: no tape, dfx_step_backward_recompute) -- without a wrench and with a random one on every link, timed with
CUDA events over K rollouts after W warm-up rollouts.  Nothing is written to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import MM_FREQ, SUBSTEPS  # noqa: E402
from bench_recompute import device_info  # noqa: E402

CONFIGS = [("AntEnv", 4096, 32), ("HumanoidEnv", 8192, 32)]


def rollout_rate(env_name, n, T, wrench, mode, steps, warmup):
    import torch
    import diffrl_b200.envs as envs
    env = getattr(envs, env_name)(num_envs=n, no_grad=True, device="cuda:0")
    from diffrl_b200.dflex_api.sim import _engine_for
    eng = _engine_for(env.model)
    S, mm, dt = SUBSTEPS[env_name], MM_FREQ[env_name], env.sim_dt
    g = torch.Generator(device="cuda:0").manual_seed(0)
    q0, qd0 = env.state.joint_q.detach().clone(), env.state.joint_qd.detach().clone()
    act = 0.1 * torch.randn((T, n * eng.D), device="cuda:0", generator=g)
    f = (5.0 * torch.randn((n, eng.L, 6), device="cuda:0", generator=g)) if wrench else None
    gq_T, gqd_T = torch.ones_like(q0), torch.ones_like(qd0)

    def one():
        q, qd, saved = q0, qd0, []
        for t in range(T):
            q_in, qd_in = q, qd
            q, qd, tape, _ = eng.forward(q, qd, act[t], None, S, mm, dt, want_tape=(mode == "tape"), f_ext=f)
            saved.append((q_in, qd_in, tape))
        gq, gqd = gq_T, gqd_T
        for t in reversed(range(T)):
            q_in, qd_in, tape = saved[t]
            if mode == "tape":
                r = eng.backward(act[t], None, tape, gq, gqd, S, mm, dt, f_ext=f)
            else:
                r = eng.backward_recompute(q_in, qd_in, act[t], None, gq, gqd, S, mm, dt, f_ext=f)
            gq, gqd = r[0], r[1]
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        one()
    t1.record()
    torch.cuda.synchronize()
    sec = t0.elapsed_time(t1) / 1e3
    del env, eng
    torch.cuda.empty_cache()
    return n * T * steps / sec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    out = {"device": device_info(), "unit": "env-steps/s, kernel path (forward over the horizon + adjoints in reverse)", "configs": {}}
    for env_name, n, T in CONFIGS:
        for mode in ("tape", "recompute"):
            key = "%s_%dx%d_%s" % (env_name, n, T, mode)
            plain = rollout_rate(env_name, n, T, False, mode, a.steps, a.warmup)
            wr = rollout_rate(env_name, n, T, True, mode, a.steps, a.warmup)
            out["configs"][key] = {"no_wrench": round(plain), "wrench": round(wr), "wrench_cost_pct": round(100 * (plain / wr - 1), 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
