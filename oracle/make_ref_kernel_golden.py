"""Store what the reference's own compiled CPU kernels (oracle/_ref, built by build() from a reference checkout) return
for the inputs of two tests, so that they run without the reference:  python oracle/make_ref_kernel_golden.py

* tests/golden/ref_kernels_random_states.npz (tests/test_oracle.py): <env>/{q0,qd0,act[,musc]} and one env-step <env>/{q,qd};
* tests/golden/SNUHumanoidEnv_bptt128.npz (tests/test_gpu_atsize.py): a 128-env-step window of the muscle humanoid on 4
  environments: q, qd [129] (state entering every step), gq, gqd, gmusc [128] (input cotangents of step t for the chain
  started with ones on the final state), jump [128] (largest change of the gradient of step t under perturbation_signs(t)),
  musc0 (pins the activation stream).
"""
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
import ref_driver  # noqa: E402
from emu_util import load_golden  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SNU, SNU_N, SNU_T = "SNUHumanoidEnv", 4, 128


def random_state_inputs(name, d, Q, D, M):
    N, n0 = 5, int(d["meta/num_envs"])
    rng = np.random.default_rng(11)
    p = "case%d/" % (int(d["meta/num_cases"]) - 1)
    pick = rng.integers(0, n0, N)
    out = dict(q0=(d[p + "q0"].reshape(n0, Q)[pick] + 1e-2 * rng.standard_normal((N, Q))).astype(np.float32),
               qd0=(d[p + "qd0"].reshape(n0, D)[pick] + 1e-1 * rng.standard_normal((N, D))).astype(np.float32),
               act=(d[p + "act"].reshape(n0, D)[pick] * rng.uniform(0.5, 1.5, (N, D))).astype(np.float32))
    if M:
        out["musc"] = (d[p + "musc"].reshape(n0, M)[pick] * rng.uniform(0.5, 1.5, (N, M))).astype(np.float32)
    return out


def snu_muscle_activations(M):
    # activation x strength range of the env (envs/snu_humanoid.py:283-296)
    g = torch.Generator().manual_seed(5)
    return [torch.rand(SNU_N * M, generator=g) * 40.0 for _ in range(SNU_T)]


def perturbation_signs(t, nq, nqd):
    # random sign patterns of 1 and 4 ulp: a switching surface of the contact / limit model nearby flips for some
    rng = np.random.default_rng(11 + t)
    return [(mag, torch.tensor(rng.choice([-1.0, 1.0], nq), dtype=torch.float32),
             torch.tensor(rng.choice([-1.0, 1.0], nqd), dtype=torch.float32)) for mag in (1.2e-7, 4.8e-7) for _ in range(6)]


def _snu_model():
    d, model = load_golden(SNU)
    arrays = dict(np.load(os.path.join(ROOT, "diffrl_b200", "assets", SNU + ".npz")))
    cfg = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    return ref_driver.RefModel(arrays, SNU_N, ground=True), cfg


def _snu_jump(job):
    t, q0, qd0, act, musc, cq, cqd = job
    rm, (S, mm, dt) = _snu_model()
    base = ref_driver.env_step(rm, q0, qd0, act, musc, dt, S, mm, gq_out=cq, gqd_out=cqd)[2]
    jump = 0.0
    for mag, sq, sqd in perturbation_signs(t, q0.numel(), qd0.numel()):
        pert = ref_driver.env_step(rm, q0 * (1.0 + mag * sq), qd0 * (1.0 + mag * sqd), act, musc, dt, S, mm, gq_out=cq, gqd_out=cqd)[2]
        jump = max(jump, float((pert[0] - base[0]).abs().max()), float((pert[1] - base[1]).abs().max()))
    return jump


def snu_window():
    rm, (S, mm, dt) = _snu_model()
    D, M = rm.D, rm.m.muscle_count // SNU_N
    muscs = snu_muscle_activations(M)
    act = torch.zeros(SNU_N * D)
    qs, qds = [rm.m.joint_q.clone()], [rm.m.joint_qd.clone()]
    for t in range(SNU_T):
        q, qd, _, _ = ref_driver.env_step(rm, qs[-1], qds[-1], act, muscs[t], dt, S, mm)
        qs.append(q.detach()); qds.append(qd.detach())
    gq_r, gqd_r = torch.ones_like(qs[-1]), torch.ones_like(qds[-1])
    gq, gqd, gm, cots = [None] * SNU_T, [None] * SNU_T, [None] * SNU_T, [None] * SNU_T
    for t in reversed(range(SNU_T)):
        cots[t] = (gq_r, gqd_r)
        g = ref_driver.env_step(rm, qs[t], qds[t], act, muscs[t], dt, S, mm, gq_out=gq_r, gqd_out=gqd_r)[2]
        gq[t], gqd[t], gm[t] = g[0].clone(), g[1].clone(), g[3].clone()
        gq_r, gqd_r = gq[t], gqd[t]
    jobs = [(t, qs[t], qds[t], act, muscs[t], cots[t][0], cots[t][1]) for t in range(SNU_T)]
    with ProcessPoolExecutor(max(1, min(16, os.cpu_count() or 1))) as pool:
        jump = list(pool.map(_snu_jump, jobs))
    st = lambda xs: torch.stack(xs).numpy().astype(np.float32)
    return dict(q=st(qs), qd=st(qds), gq=st(gq), gqd=st(gqd), gmusc=st(gm), jump=np.array(jump, np.float32),
                musc0=muscs[0].numpy())


def random_states():
    from oracle import Oracle
    out = {}
    for name in ("AntEnv", "SNUHumanoidEnv", "CartPoleSwingUpEnv"):
        d, model = load_golden(name)
        o = Oracle.from_model(model, int(d["meta/num_envs"]))
        Q, D, M = o.desc.Q, o.desc.D, o.desc.M
        inp = random_state_inputs(name, d, Q, D, M)
        S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
        arrays = dict(np.load(os.path.join(ROOT, "diffrl_b200", "assets", name + ".npz")))
        rm = ref_driver.RefModel(arrays, 5, ground=bool(d["meta/ground"]))
        t = lambda a: None if a is None else torch.tensor(a.ravel())
        rq, rqd, _, _ = ref_driver.env_step(rm, t(inp["q0"]), t(inp["qd0"]), t(inp["act"]), t(inp.get("musc")), dt, S, mm)
        for k, v in inp.items():
            out[name + "/" + k] = v
        out[name + "/q"], out[name + "/qd"] = rq.numpy(), rqd.numpy()
    return out


if __name__ == "__main__":
    if not ref_driver.available():
        raise SystemExit("oracle/_ref/kernels/kernels.so not built: run build() where a reference checkout is readable")
    np.savez_compressed(os.path.join(GOLDEN, "ref_kernels_random_states.npz"), **random_states())
    np.savez_compressed(os.path.join(GOLDEN, SNU + "_bptt128.npz"), **snu_window())
    print("wrote", GOLDEN)
