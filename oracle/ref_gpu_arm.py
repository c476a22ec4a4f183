"""The reference's OWN implementation driven through its stock public API -- the baselines bench.py reports.

BENCH / TEST INFRASTRUCTURE ONLY.  Runs in its own interpreter (the name ``dflex`` must resolve to the reference's
package, not to this repo's) on the git-ignored install made by ``oracle/install_reference.py`` under
``baseline/_ref`` (it travels to the GPU box; ``/root/reference`` does not exist there).

    python oracle/ref_gpu_arm.py --env AntEnv --num-envs 4096 --horizon 32 --rollouts 2 --warmup 1 [--device cuda:0|cpu]

``--device cuda:0``: the reference's CUDA codegen path (``dflex/dflex/adjoint.py:1247-1262`` launch templates), rebuilt
for sm_90 with the ONE flag edit at ``adjoint.py:1861`` (``compute_35`` -> ``compute_90``) -- SURVEY.md section 8d's
"second bar", the only pre-existing GPU implementation of this path.
``--device cpu``: the reference's CPU path (a serial loop, ``adjoint.py:1271-1279``).

Workload = SURVEY.md section 8d: ``envs.<Env>(stochastic_init=False, no_grad=False, seed=0, MM_caching_frequency=YAML)``,
``clear_grad(); reset(); initialize_trajectory()``, ``horizon`` x ``env.step(U(-1,1) actions)``, ``sum(rew).backward()``.
Prints one JSON object.
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "baseline", "_ref")
MM_FREQ = {"AntEnv": 16, "HumanoidEnv": 48, "SNUHumanoidEnv": 8, "CartPoleSwingUpEnv": 4, "HopperEnv": 16, "CheetahEnv": 16}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="AntEnv")
    ap.add_argument("--num-envs", type=int, default=4096)
    ap.add_argument("--horizon", type=int, default=32)
    ap.add_argument("--rollouts", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--stamp", action="store_true", help="also report time.time() at the start / end of the timed rollouts (pool wall clock)")
    a = ap.parse_args()
    if not os.path.isdir(os.path.join(REF, "refdflex", "dflex")):
        print(json.dumps({"unavailable": "baseline/_ref missing: run `python oracle/install_reference.py` in the build container"}))
        return
    import numpy as np
    if not hasattr(np, "Inf"):
        np.Inf = np.inf
    sys.path[:0] = [os.path.join(HERE, "refshim"), os.path.join(REF, "refdflex"), REF]
    if a.device == "cpu":
        os.environ["CUDA_VISIBLE_DEVICES"] = ""
    # the reference caches its generated kernels by comparing source strings, and the source differs with / without the CUDA
    # half: always generate both, so that the ONE prebuilt kernels.so (CPU + sm_90) is reused on every box and device
    os.environ["DFLEX_FORCE_CUDA_BUILD"] = "1"
    import torch
    import dflex  # noqa: F401  (the reference's; loads its prebuilt kernels.so)
    assert os.path.realpath(dflex.__file__).startswith(os.path.realpath(REF)), dflex.__file__
    import envs
    cuda = a.device.startswith("cuda")
    if a.device == "cpu":
        torch.set_num_threads(1)
    env = getattr(envs, a.env)(num_envs=a.num_envs, device=a.device, render=False, seed=0, stochastic_init=False,
                               no_grad=False, MM_caching_frequency=MM_FREQ[a.env])
    gen = torch.Generator().manual_seed(1)
    actions = (torch.rand((a.horizon, a.num_envs, env.num_actions), generator=gen) * 2 - 1).to(a.device)

    def sync():
        if cuda:
            torch.cuda.synchronize()

    def rollout():
        env.clear_grad()
        env.reset()
        env.initialize_trajectory()
        act = actions.clone().requires_grad_()
        sync()
        t0 = time.perf_counter()
        loss = 0.0
        for t in range(a.horizon):
            obs, rew, done, _ = env.step(act[t])
            loss = loss + rew.sum()
        sync()
        t1 = time.perf_counter()
        loss.backward()
        sync()
        t2 = time.perf_counter()
        return t1 - t0, t2 - t1, float(loss), float(act.grad.abs().sum())

    for _ in range(a.warmup):
        rollout()
    tf = tb = 0.0
    t_start = time.time()
    for _ in range(a.rollouts):
        f, b, loss, gsum = rollout()
        tf += f
        tb += b
    t_end = time.time()
    steps = a.num_envs * a.horizon * a.rollouts
    out = {"impl": "reference", "device": a.device, "env": a.env, "num_envs": a.num_envs, "horizon": a.horizon,
           "rollouts": a.rollouts, "forward_s": tf, "backward_s": tb, "env_steps_per_s": steps / (tf + tb),
           "loss": loss, "grad_abs_sum": gsum, "finite": bool(np.isfinite(loss) and np.isfinite(gsum)),
           "api": "reference envs.%s.step -> reference dflex.sim.SemiImplicitIntegrator (%s codegen kernels)" % (a.env, "CUDA sm_90" if cuda else "CPU"),
           "peak_mem_gb": (torch.cuda.max_memory_allocated() / 1e9) if cuda else None}
    if a.stamp:
        out["t_start"], out["t_end"] = t_start, t_end
    print(json.dumps(out))


if __name__ == "__main__":
    main()
