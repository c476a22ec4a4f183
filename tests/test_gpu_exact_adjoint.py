"""The CUDA step adjoint against the EXACT gradient of the oracle's fp64 forward (complex step, tests/exact_util.py): every
articulation x every kernel family that exists for it x every H-refresh pattern of exact_util.patterns, on a batch of 75
environments (not a multiple of any tile) of golden states + noise and explicit pushes into every branch of the contact and
limit model.  Each sampled environment (first tile, last tile, between) must hold every gradient block within
tolerances.exact_grad_tol; only environments on a switching surface of the fp64 branch sequence may be excluded, a few per
case, and are printed.  The exact gradients depend only on the inputs and are computed once per pattern for all families."""
import numpy as np
import pytest

from conftest import ENVS
import exact_util as X
from tolerances import EXACT_SAMPLE, exact_grad_tol

pytestmark = pytest.mark.gpu

N = 75
VARIANTS = ["auto", "tile8", "tile16", "tile32", "group8", "group16", "group32"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", ENVS)
def test_cuda_adjoint_matches_exact_gradient(name, variant):
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    from test_gpu_golden import _select
    o = X._oracle(name)
    desc, inp, idx = X.make_batch(name, N, EXACT_SAMPLE[name], seed=1)
    sub = {k: (None if v is None else v[idx]) for k, v in inp.items()}
    t = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a).ravel(), device="cuda:0")
    _select(variant)
    try:
        eng = ArticulationEngine(desc, N, "cuda:0")
        tile = int(_capi.lib().dfx_pack_query(eng.pack, 9))
        if variant.startswith("tile") and tile != int(variant[4:]):
            pytest.skip("no %s-environment tile kernel for %s" % (variant[4:], name))
        assert (tile == 0) == variant.startswith("group")
        worst_all, excluded_all = {}, 0
        for S, mm in X.patterns(name):
            dt = X.pattern_dt(name, S)
            cov = X.branch_coverage(o, sub, S, mm, dt)
            assert all(cov[b] > 0 for b in X.branches_of_model(desc)), (name, (S, mm), cov)
            ex = X.exact_gradients(name, inp, idx, S, mm, dt)
            q, qd, tape, _ = eng.forward(t(inp["q0"]), t(inp["qd0"]), t(inp["act"]), t(inp["musc"]), S, mm, dt)
            g = eng.backward(t(inp["act"]), t(inp["musc"]), tape, t(inp["gq_out"]), t(inp["gqd_out"]), S, mm, dt)
            got = [x.cpu().numpy().reshape(N, -1)[idx] for x in g if x is not None]
            what = "%s %s (%d, %d)" % (name, variant, S, mm)
            worst, excluded = X.check_against_exact(what, o, inp, idx, got, ex, exact_grad_tol(name, S), S, mm, dt,
                                                    max_excluded=max(2, len(idx) // 20))
            print(what, "worst per block:", {b: "%.1e" % v for b, v in worst.items()})
            excluded_all += len(excluded)
            for b, v in worst.items():
                key = (b, "1x1" if S == 1 else "multi")
                worst_all[key] = max(worst_all.get(key, 0.0), v)
        print("%s %s: worst over patterns %s; %d exclusions" % (name, variant, {"%s/%s" % k: "%.1e" % v for k, v in worst_all.items()}, excluded_all))
    finally:
        _select("auto")
