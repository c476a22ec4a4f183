"""Run the reference's UNCHANGED ``algorithms/shac.py`` (from the git-ignored install ``baseline/_ref``) on either ``dflex``:

    python tools/run_ref_shac.py --dflex ours|reference --env ant --seed 0 --max-epochs 2000 --device cuda:0 --out curve.json

``--dflex ours``: this repo's drop-in package (the claim: the trainer runs unchanged on it); ``--dflex reference``: the
reference's own dflex (its CUDA codegen rebuilt for sm_90, or its CPU path with ``--device cpu``).  The training curve
(policy loss per epoch = minus the mean undiscounted return estimate the trainer logs, episode returns) is written as JSON.
Harness only: the trainer file is byte-identical to the reference's; ``oracle/refshim/torch_compat.py`` supplies the
torch >= 2 indexing behaviour it was written against.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dflex", default="ours", choices=["ours", "reference"])
    ap.add_argument("--env", default="ant", help="basename of examples/cfg/shac/<env>.yaml")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-epochs", type=int, default=0)
    ap.add_argument("--num-actors", type=int, default=0)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--logdir", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    if not hasattr(np, "Inf"):
        np.Inf = np.inf
    shim = os.path.join(ROOT, "oracle", "refshim")
    if a.dflex == "ours":
        sys.path[:0] = [ROOT, shim, REF]
    else:
        os.environ["DFLEX_FORCE_CUDA_BUILD"] = "1"
        if a.device == "cpu":
            os.environ["CUDA_VISIBLE_DEVICES"] = ""
        sys.path[:0] = [shim, os.path.join(REF, "refdflex"), REF]
    import torch
    import torch_compat  # noqa: F401
    import yaml
    import dflex
    import algorithms.shac as shac
    assert shac.__file__.startswith(REF), shac.__file__
    cfg = yaml.load(open(os.path.join(REF, "examples", "cfg", "shac", a.env + ".yaml")), Loader=yaml.SafeLoader)
    logdir = a.logdir or os.path.join("/tmp", "ref_shac_%s_%s_%d" % (a.dflex, a.env, a.seed))
    cfg["params"]["general"] = dict(device=a.device, seed=a.seed, render=False, logdir=logdir, train=True, checkpoint="Base", no_time_stamp=True)
    if a.max_epochs:
        cfg["params"]["config"]["max_epochs"] = a.max_epochs
    if a.num_actors:
        cfg["params"]["config"]["num_actors"] = a.num_actors
    agent = shac.SHAC(cfg)
    # the trainer logs through its SummaryWriter and prints; tap its meters once per epoch without touching the file
    curve = []
    orig = agent.actor_optimizer.step

    def tapped(closure=None):
        out = orig(closure)
        curve.append({"epoch": int(agent.iter_count), "env_steps": int(agent.step_count), "actor_loss": float(out.detach()) if out is not None else None,
                      "mean_policy_loss": float(agent.episode_loss_meter.get_mean()) if agent.episode_loss_meter.current_size > 0 else None,
                      "wall_s": round(time.time() - t0, 2)})
        return out

    agent.actor_optimizer.step = tapped
    t0 = time.time()
    agent.train()
    rec = {"trainer": "reference algorithms/shac.py (unchanged)", "dflex": dflex.__file__, "env": a.env, "seed": a.seed, "device": a.device,
           "num_actors": int(agent.num_envs), "epochs": int(agent.iter_count), "env_steps": int(agent.step_count), "wall_s": round(time.time() - t0, 1),
           "final_mean_policy_loss": curve[-1]["mean_policy_loss"] if curve else None, "curve": curve[:: max(1, len(curve) // 200)] + curve[-1:]}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps({k: v for k, v in rec.items() if k != "curve"}))


if __name__ == "__main__":
    main()
