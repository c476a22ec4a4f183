"""Cost of the Jacobian state (include/dfx.h dfx_jacobian_state_forward / _backward) next to one env-step.

    python tools/bench_jacobian_state.py [--launches K] [--warmup W]

Prints ONE JSON line: the device (card name and power limit, read in the same run) and, for Ant 4096, Humanoid 8192 and SNU 4096
on their default kernels, the time per launch through the C ABI (microseconds, CUDA events over K back-to-back launches after W
warm-up launches; issued from a host loop, and replayed from one CUDA graph -- the kernels' own time) of
  * the Jacobian-state forward (J and body_a_s) and its backward (both cotangents);
  * the same without J: the forward with body_a_s only (J NULL) and the backward with g_a_s only (g_J NULL) -- the kinematics and its
    adjoint on their own, so that the difference is what forming and storing J (reading g_J) costs;
  * one env-step forward with a tape and its stored-tape backward, at the env's own (substeps, mm_freq);
the Jacobian state's forward + backward as a percentage of the env-step's, and the bytes of J one forward writes over its graphed
time, next to the 3.35 TB/s of HBM3 bandwidth NVIDIA's data sheet gives for the H100 SXM (a data-sheet figure, not a measured
peak).  Nothing is written to the tree."""
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
DATASHEET_HBM_TBS = 3.35


def measure(env_name, n, launches, warmup):
    """the four launches through the C ABI on preallocated buffers (one tape, reused)"""
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
    J, a_s = torch.empty((n, eng.L, 6, eng.D), device="cuda:0"), torch.empty((n, eng.L, 6), device="cuda:0")
    gJ, ga = torch.randn(J.shape, device="cuda:0", generator=g), torch.randn(a_s.shape, device="cuda:0", generator=g)
    gq, gqd = torch.empty_like(q), torch.empty_like(qd)
    q_out, qd_out = torch.empty_like(q), torch.empty_like(qd)
    gact = torch.empty_like(act)
    gmusc = torch.empty_like(musc) if musc is not None else None
    ones_q, ones_qd = torch.ones_like(q), torch.ones_like(qd)
    tape = torch.empty(eng.tape_floats(S, mm), device="cuda:0")
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    calls = {
        "jacobian_state_fwd": lambda: lib.dfx_jacobian_state_forward(eng.pack, n, p(q), p(qd), p(J), p(a_s), st()),
        "jacobian_state_bwd": lambda: lib.dfx_jacobian_state_backward(eng.pack, n, p(q), p(qd), p(gJ), p(ga), p(gq), p(gqd), st()),
        "jacobian_state_fwd_without_J": lambda: lib.dfx_jacobian_state_forward(eng.pack, n, p(q), p(qd), None, p(a_s), st()),
        "jacobian_state_bwd_without_g_J": lambda: lib.dfx_jacobian_state_backward(eng.pack, n, p(q), p(qd), None, p(ga), p(gq), p(gqd),
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
        r[mode]["jacobian_state_pct_of_env_step"] = round(100 * (t["jacobian_state_fwd"] + t["jacobian_state_bwd"])
                                                          / (t["env_step_fwd"] + t["env_step_bwd"]), 2)
    j_bytes = J.numel() * 4
    r["J_bytes_per_forward"] = j_bytes
    r["J_store_TBps_over_graphed_forward"] = round(j_bytes / (r["graphed"]["jacobian_state_fwd_us"] * 1e-6) / 1e12, 3)
    r["J_store_share_of_datasheet_3.35TBps"] = round(r["J_store_TBps_over_graphed_forward"] / DATASHEET_HBM_TBS, 3)
    tile = int(lib.dfx_pack_query(eng.pack, 9))
    r["kernel"] = "tile%d" % tile if tile else "lane groups"
    r["substeps"], r["mm_freq"] = S, mm
    del env, eng, tape, J, gJ
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    out = {"device": device_info(), "configs": {}}
    for env_name, n in CONFIGS:
        out["configs"]["%s_%d" % (env_name, n)] = measure(env_name, n, a.launches, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
