"""Cost of the dynamics state (include/dfx.h dfx_dynamics_state_forward / _backward) next to one env-step.

    python tools/bench_dynamics_state.py [--launches K] [--warmup W] [--settle T]

Prints ONE JSON line: the device (card name and power limit, read in the same run) and, for Ant 4096, Humanoid 8192 and SNU 4096
on their default kernels, the time per launch through the C ABI (microseconds, CUDA events over K back-to-back launches after W
warm-up launches; issued from a host loop, and replayed from one CUDA graph -- the kernels' own time) of
  * the dynamics-state forward (all three outputs) and its backward (all three cotangents, all five gradients; one launch on the
    tile kernels, two on the lane groups);
  * one env-step forward with a tape and its stored-tape backward, at the env's own (substeps, mm_freq);
and the dynamics state's forward + backward as a percentage of the env-step's.  The contact model and its adjoint run for
penetrating points only, so it is timed at a state in ground contact: the env's start state advanced by T env-steps (default 120)
under small random joint torques.  Nothing is written to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import MM_FREQ, SUBSTEPS  # noqa: E402
from bench_link_state import per_launch_us  # noqa: E402
from bench_recompute import device_info  # noqa: E402

CONFIGS = [("AntEnv", 4096), ("HumanoidEnv", 8192), ("SNUHumanoidEnv", 4096)]


def measure(env_name, n, launches, warmup, settle):
    """the four launches through the C ABI on preallocated buffers (one tape, reused), at the start state advanced by `settle`
    env-steps"""
    import ctypes
    import torch
    import diffrl_b200.envs as envs
    env = getattr(envs, env_name)(num_envs=n, no_grad=True, device="cuda:0")
    from diffrl_b200.dflex_api.sim import _engine_for
    eng = _engine_for(env.model)
    lib = eng.lib
    S, mm, dt = SUBSTEPS[env_name], MM_FREQ[env_name], env.sim_dt
    g = torch.Generator(device="cuda:0").manual_seed(0)
    q, qd = env.state.joint_q.detach().clone(), env.state.joint_qd.detach().clone()
    act = 0.1 * torch.randn(n * eng.D, device="cuda:0", generator=g)
    musc = 0.5 * torch.ones(n * eng.M, device="cuda:0") if eng.M else None
    shapes = ((n, eng.D), (n, eng.D), (n, eng.D, eng.D))
    X = [torch.empty(s, device="cuda:0") for s in shapes]
    gX = [torch.randn(s, device="cuda:0", generator=g) for s in shapes]
    gq, gqd = torch.empty_like(q), torch.empty_like(qd)
    f_ext = torch.zeros((n, eng.L, 6), device="cuda:0")
    g_f_ext = torch.empty_like(f_ext)
    ws = eng.dynamics_workspace()
    q_out, qd_out = torch.empty_like(q), torch.empty_like(qd)
    gact = torch.empty_like(act)
    gmusc = torch.empty_like(musc) if musc is not None else None
    ones_q, ones_qd = torch.ones_like(q), torch.ones_like(qd)
    tape = torch.empty(eng.tape_floats(S, mm), device="cuda:0")
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(settle):          # (the robots start above the ground: let them land)
        act.normal_(generator=g).mul_(0.1)
        assert lib.dfx_step_forward(eng.pack, n, S, mm, dt, p(q), p(qd), p(act), p(musc), p(q_out), p(qd_out), None, None, st()) == 0
        q.copy_(q_out)
        qd.copy_(qd_out)
    calls = {
        "dynamics_state_fwd": lambda: lib.dfx_dynamics_state_forward(eng.pack, n, p(q), p(qd), p(act), p(musc), p(f_ext),
                                                                     *(p(x) for x in X), st()),
        "dynamics_state_bwd": lambda: lib.dfx_dynamics_state_backward(eng.pack, n, p(q), p(qd), p(act), p(musc), p(f_ext), p(ws),
                                                                      *(p(x) for x in gX), p(gq), p(gqd), p(gact), p(gmusc), p(g_f_ext),
                                                                      st()),
        "env_step_fwd": lambda: lib.dfx_step_forward(eng.pack, n, S, mm, dt, p(q), p(qd), p(act), p(musc), p(q_out), p(qd_out), p(tape),
                                                     None, st()),
        "env_step_bwd": lambda: lib.dfx_step_backward(eng.pack, n, S, mm, dt, p(act), p(musc), p(tape), p(ones_q), p(ones_qd), p(gq),
                                                      p(gqd), p(gact), p(gmusc), st()),
    }
    for k, f in calls.items():
        assert f() == 0, k
    r = {}
    for mode in ("host_loop", "graphed"):
        t = {k: per_launch_us(f, launches, warmup, mode == "graphed") for k, f in calls.items()}
        r[mode] = {k + "_us": round(v, 1) for k, v in t.items()}
        r[mode]["dynamics_state_pct_of_env_step"] = round(100 * (t["dynamics_state_fwd"] + t["dynamics_state_bwd"])
                                                      / (t["env_step_fwd"] + t["env_step_bwd"]), 2)
    tile = int(lib.dfx_pack_query(eng.pack, 9))
    r["kernel"] = "tile%d" % tile if tile else "lane groups"
    r["substeps"], r["mm_freq"] = S, mm
    r["settle_env_steps"] = settle
    if eng.C:
        r["penetrating_points_frac"] = round(float((eng.contact_state(q, qd)[1] < 0).float().mean()), 3)
    del env, eng, tape, ws
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--settle", type=int, default=120)
    a = ap.parse_args()
    out = {"device": device_info(), "configs": {}}
    for env_name, n in CONFIGS:
        out["configs"]["%s_%d" % (env_name, n)] = measure(env_name, n, a.launches, a.warmup, a.settle)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
