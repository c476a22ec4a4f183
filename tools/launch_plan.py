"""Print the launch geometry (lanes/env, envs/CTA, CTAs/SM, shared memory) of the step kernels for the six DiffRL
articulations.  Needs a CUDA device (the pack lives in device memory)."""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from emu_util import load_golden
from diffrl_b200.modelpack import articulation_from_model
from diffrl_b200.engine import ArticulationEngine

for name in ["CartPoleSwingUpEnv", "HopperEnv", "CheetahEnv", "AntEnv", "HumanoidEnv", "SNUHumanoidEnv"]:
    d, model = load_golden(name)
    desc, _ = articulation_from_model(model, int(d["meta/num_envs"]))
    eng = ArticulationEngine(desc, 4, "cuda:0")
    for bwd in (0, 1):
        out = (ctypes.c_int * 6)()
        eng.lib.dfx_launch_plan(eng.pack, bwd, out)
        g, e, c, smem, stride, pack = list(out)
        print("%-20s %s lanes/env %2d envs/CTA %2d CTAs/SM %2d -> %3d envs/SM (%6d on 132 SMs)  smem/CTA %6d B  scratch %5d B/env  pack %5d B"
              % (name, "bwd" if bwd else "fwd", g, e, c, e * c, e * c * 148, smem, stride * 4, pack))
