"""Tape vs recompute adjoint (diffrl_b200.set_adjoint_mode): throughput and peak device memory of differentiable rollouts.

    python tools/bench_recompute.py [--steps K] [--warmup W]

Prints ONE JSON line:
  device         card name and power limit, read in the same run;
  configs        Ant 4096 x 32, Humanoid 8192 x 32, SNU 4096 x 128 in both modes: the kernel path (engine forward over the horizon,
                 then the adjoints in reverse) and GraphedRollout end to end (H2D actions, env.step x T, loss.backward, D2H), in
                 env-steps/s, with torch.cuda.max_memory_allocated per rollout above what was allocated before it;
  long           Ant / SNU 4096 x 1000 in recompute mode only, with the tape that tape mode would need (dfx_tape_floats) marked
                 "does not fit" -- those runs are not attempted;
  fused          the one-launch recompute adjoint against its two-launch equivalent (the forward into a tape, then the stored-tape
                 adjoint), per env-step, on Ant 4096 and Humanoid 8192.
Nothing is written to the tree."""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import MM_FREQ, SUBSTEPS  # noqa: E402


def device_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "total_memory_gb": round(torch.cuda.get_device_properties(0).total_memory / 1e9, 1)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        info["smi_name"], info["power_limit"] = [x.strip() for x in out.split(",")]
    except Exception as exc:       # (no nvidia-smi: the card name above still identifies the device)
        info["power_limit"] = "unknown (%s)" % type(exc).__name__
    return info


def _free():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _timed(fn, steps, warmup):
    """(ms per call, peak bytes above the allocation before the first timed call) -- host clock around synchronised calls."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps, torch.cuda.max_memory_allocated() - base


def make_env(name, N, T):
    import torch
    import diffrl_b200.envs as envs
    torch.manual_seed(1234)
    return getattr(envs, name)(num_envs=N, device="cuda:0", render=False, seed=0, stochastic_init=False, no_grad=False,
                               MM_caching_frequency=MM_FREQ[name], episode_length=max(1000, T))


def kernel_inputs(env, name, T):
    """Actuation of T env-steps (joint_act, or muscle activations for SNU) and the start state."""
    import torch
    from diffrl_b200.dflex_api.sim import _engine_for
    eng = _engine_for(env.model)
    N = env.num_envs
    g = torch.Generator(device="cuda:0").manual_seed(1)
    env.clear_grad(); env.reset()
    acts, muscs = [], []
    for _ in range(T):
        a = torch.rand((N, env.num_actions), generator=g, device="cuda:0") * 2 - 1
        if eng.M:
            acts.append(torch.zeros(N * eng.D, device="cuda:0"))
            muscs.append(((a * 0.5 + 0.5).view(-1) * env.muscle_strengths).contiguous())
        else:
            env.state.joint_act.zero_()
            env._apply_actions(a)
            acts.append(env.state.joint_act.detach().clone())
            muscs.append(None)
    return eng, env.state.joint_q.detach().clone(), env.state.joint_qd.detach().clone(), acts, muscs


def kernel_rollout_fn(eng, name, dt, q0, qd0, acts, muscs, mode):
    import torch
    S, mm, dt_ = SUBSTEPS[name], MM_FREQ[name], dt
    T = len(acts)
    gq0, gqd0 = torch.ones_like(q0).view(-1), torch.ones_like(qd0).view(-1)

    def run():
        q, qd, keep = q0, qd0, []
        for t in range(T):
            q1, qd1, tape, _ = eng.forward(q, qd, acts[t], muscs[t], S, mm, dt_, want_tape=(mode == "tape"))
            keep.append(tape if mode == "tape" else (q, qd))
            q, qd = q1, qd1
        gq, gqd = gq0, gqd0
        for t in reversed(range(T)):
            if mode == "tape":
                gq, gqd, _, _ = eng.backward(acts[t], muscs[t], keep[t], gq, gqd, S, mm, dt_)
            else:
                gq, gqd, _, _ = eng.backward_recompute(keep[t][0], keep[t][1], acts[t], muscs[t], gq, gqd, S, mm, dt_)
            keep[t] = None
        return gq
    return run


def measure(name, N, T, mode, steps, warmup, e2e=True):
    import torch
    import diffrl_b200
    from diffrl_b200.rollout import GraphedRollout
    rec = {"env": name, "N": N, "T": T, "mode": mode}
    diffrl_b200.set_adjoint_mode(mode)
    try:
        env = make_env(name, N, T)
        eng, q0, qd0, acts, muscs = kernel_inputs(env, name, T)
        rec["tape_gb_per_rollout"] = round(T * eng.tape_floats(SUBSTEPS[name], MM_FREQ[name]) * 4 / 1e9, 2)
        rec["workspace_mb"] = round(int(eng.lib.dfx_recompute_workspace_floats(eng.pack, N, SUBSTEPS[name], MM_FREQ[name])) * 4 / 1e6, 1)
        ms, peak = _timed(kernel_rollout_fn(eng, name, env.sim_dt, q0, qd0, acts, muscs, mode), steps, warmup)
        rec.update(kernel_env_steps_per_s=round(N * T / (ms / 1e3)), kernel_ms=round(ms, 2), kernel_peak_gb=round(peak / 1e9, 3))
        del acts, muscs
        _free()
        if e2e:
            env.clear_grad(); env.reset(); env.initialize_trajectory()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            roll = GraphedRollout(env, T, warmup=1)
            roll.host_actions.copy_(torch.rand(roll.host_actions.shape, generator=torch.Generator().manual_seed(3)) * 2 - 1)
            build_peak = torch.cuda.max_memory_allocated() - base

            def replay():
                env.clear_grad(); env.reset()
                roll(None, sync=True)
            ms, _ = _timed(replay, steps, max(1, warmup))
            rec.update(e2e_env_steps_per_s=round(N * T / (ms / 1e3)), e2e_ms=round(ms, 2), e2e_peak_gb=round(build_peak / 1e9, 3),
                       e2e_loss=float(roll.host_loss))
            del roll
    finally:
        diffrl_b200.set_adjoint_mode("tape")
    del env, eng
    _free()
    return rec


def fused_vs_two_launch(name, N, steps):
    """Per env-step adjoint time: the one-launch recompute adjoint vs the forward into a tape followed by the stored-tape adjoint
    (the same arithmetic in two launches), and the stored-tape adjoint alone."""
    import torch
    env = make_env(name, N, 1)
    eng, q, qd, acts, muscs = kernel_inputs(env, name, 1)
    S, mm, dt = SUBSTEPS[name], MM_FREQ[name], env.sim_dt
    act, musc = acts[0], muscs[0]
    gq, gqd = torch.ones_like(q).view(-1), torch.ones_like(qd).view(-1)
    ws = eng.recompute_workspace(S, mm)
    _, _, tape, _ = eng.forward(q, qd, act, musc, S, mm, dt)
    out = {"env": name, "N": N}
    reps = 10 * steps
    fused_ms, _ = _timed(lambda: eng.backward_recompute(q, qd, act, musc, gq, gqd, S, mm, dt, workspace=ws), reps, 3)

    def two():
        _, _, t2, _ = eng.forward(q, qd, act, musc, S, mm, dt)
        eng.backward(act, musc, t2, gq, gqd, S, mm, dt)
    two_ms, _ = _timed(two, reps, 3)
    fwd_ms, _ = _timed(lambda: eng.forward(q, qd, act, musc, S, mm, dt, want_tape=False), reps, 3)
    bwd_ms, _ = _timed(lambda: eng.backward(act, musc, tape, gq, gqd, S, mm, dt), reps, 3)
    out.update(fused_ms=round(fused_ms, 3), two_launch_ms=round(two_ms, 3), tape_adjoint_ms=round(bwd_ms, 3), nograd_forward_ms=round(fwd_ms, 3),
               fused_speedup=round(two_ms / fused_ms, 3),
               # a rollout step costs forward + adjoint: tape mode (taping forward ~ no-grad forward) vs recompute mode
               recompute_kernel_time_overhead=round((fwd_ms + fused_ms) / (fwd_ms + bwd_ms) - 1.0, 3))
    del env, eng, tape, ws
    _free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip-long", action="store_true")
    args = ap.parse_args()
    import torch
    from diffrl_b200.dflex_api.sim import _engine_for
    res = {"device": device_info(), "steps": args.steps, "warmup": args.warmup, "configs": [], "long": [], "fused": []}
    total = torch.cuda.get_device_properties(0).total_memory
    for name, N, T in (("AntEnv", 4096, 32), ("HumanoidEnv", 8192, 32), ("SNUHumanoidEnv", 4096, 128)):
        for mode in ("tape", "recompute"):
            res["configs"].append(measure(name, N, T, mode, args.steps, args.warmup))
            print(json.dumps(res["configs"][-1]), file=sys.stderr)
    for name, N in (("AntEnv", 4096), ("HumanoidEnv", 8192)):
        res["fused"].append(fused_vs_two_launch(name, N, args.steps))
        print(json.dumps(res["fused"][-1]), file=sys.stderr)
    if not args.skip_long:
        for name in ("AntEnv", "SNUHumanoidEnv"):
            N, T = 4096, 1000
            env = make_env(name, N, T)
            need = T * _engine_for(env.model).tape_floats(SUBSTEPS[name], MM_FREQ[name]) * 4
            del env
            _free()
            res["long"].append({"env": name, "N": N, "T": T, "mode": "tape", "tape_gb_required": round(need / 1e9, 1),
                                "device_gb": round(total / 1e9, 1), "status": "does not fit" if need > total else "fits (not run)"})
            res["long"].append(measure(name, N, T, "recompute", 1, 0))
            print(json.dumps(res["long"][-1]), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
