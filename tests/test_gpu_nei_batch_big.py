"""NEI with pending points (DESIGN.md 4.14) at production sizes and on ill-conditioned noiseless factors, against a
double-double reference.

tests/test_gpu_nei_batch.py holds the device to tests/nei_batch_oracle.py at N = 300 on well-conditioned sets.  The
fixtures here (oracle/make_nei_batch.py, tests/golden/neibatch_*.npz) take three cases of oracle/make_nei_big.py
(N = 121, 1000 and 4096; cond(K0) to about 1e10) with p = 1, 7 and 15 pending rows - the incumbent's input, rows 1e-3
from training rows and uniform rows - and hold the double-double truth of the pending fantasies, best_s', sigma0' and
NEI / LogNEI at the case's candidates, the pending rows and their 1e-7 neighbours, with the restatement's fp64 results
on the same draws as the referee.  At these sizes the pending rows are chained O(N^2) updates of L and L^-1 over up to
32 row blocks, and A' comes from S explicit-inverse solves on the grown factor.

The rules are tests/test_gpu_nei_big.py's: device error <= max(C_REF * the referee's error, FLOOR), the 1e-5 bar wherever
the referee meets it, and per-case bars pinned at about 10x the error measured on an H100 80GB HBM3 at a 700 W power
limit (in the comments).  Every case prints the device's and the referee's errors (pytest -s).
"""
import warnings

import numpy as np
import pytest

from oracle import make_illcond as MI
from oracle import make_nei_batch as NBB
from oracle import make_nei_big as NB
from test_gpu_illcond import RTOL
from test_gpu_nei_big import C_REF, FLOOR, _fmt, _value_err

pytestmark = pytest.mark.gpu

# The pending rows' fantasies come from the appended factor row l = L0^-1 k, which the row update forms with the
# explicit inverse (W k, DESIGN.md 4.11), not by substitution as the referee does: measured 5-40x the referee's error
# (2.4e-12 against 1.2e-13 on c_m25_d3, p = 1), held to 100x as sigma0, the residue of the same explicit inverse, is.
C_REF_P = dict(C_REF, F=100.0)
# Per-case bars at about 10x the measurement (comments): over every metric and p of the case (LogNEI sets it), and
# on the pending fantasies alone.
PIN = {
    "c_m25_d3": 8.4e-7,  # 8.4e-8 LogNEI, p = 7 and 15
    "b_m15_d17": 1.9e-6,  # 1.9e-7 LogNEI, p = 15
    "b_m25_c3": 3.3e-6,  # 3.3e-7 LogNEI, p = 15
}
PIN_F = {
    "c_m25_d3": 6.9e-10,  # 6.9e-11, p = 15
    "b_m15_d17": 2.4e-9,  # 2.4e-10, p = 15
    "b_m25_c3": 2.3e-9,  # 2.3e-10, p = 7 and 15
}

_FIX, _GP = {}, {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = NBB.load(name)
    return _FIX[name]


def _gp(bo, name):
    if name not in _GP:
        noisy, _, _ = NB.gp_cases(name)
        r = fixture(name)
        _GP[name] = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(noisy), alpha=noisy["alpha"],
                                                    normalize_y=True, optimizer=None).fit(r["X"], r["y"])
    return _GP[name]


def _errors(r, key, got):
    """F and best_s relative to |value| + s_y, sigma0 relative, NEI / LogNEI as tests/test_gpu_nei_big.py."""
    want, ys = r[key], float(r["y_std"])
    kind = key.split("_", 1)[1]
    if kind in ("F", "best"):
        return float(np.max(np.abs(got - want) / (np.abs(want) + ys)))
    if kind == "sd0":
        return float(np.max(np.abs(got - want) / want))
    return _value_err(kind, got, want)


@pytest.mark.parametrize("p", NBB.PS)
@pytest.mark.parametrize("name", NBB.CASES)
def test_pending_fantasies_and_values_against_truth(bo, name, p):
    r = fixture(name)
    gp = _gp(bo, name)
    n = len(r["X"])
    fant = gp.noiseless_fantasies(NBB.S, jitter=NB.JITTER, random_state=NBB.SEED, pending=r["P"][:p],
                                  extra_rows=NBB.P_MAX - p)
    assert fant.F.shape == (n + p, NBB.S)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, sd = fant.gp.predict(r["xc"], return_std=True)
    got = dict(F=fant.F[n:], best=fant.best, sd0=sd)
    for kind in ("nei", "lognei"):
        code = bo._lib.ACQ_NEI if kind == "nei" else bo._lib.ACQ_LOGNEI
        got[kind] = -bo.FusedAcquisition(code, gp, xi=NBB.XI, fantasies=fant)(r["xc"])
    dev = {k: _errors(r, f"p{p}_{k}", v) for k, v in got.items()}
    ref = {k: _errors(r, f"p{p}_{k}", r[f"sk_p{p}_{k}"]) for k in got}
    print(f"\n{name} p={p}\n  device  {_fmt(dev)}\n  referee {_fmt(ref)}")
    for k in dev:
        assert dev[k] <= max(C_REF_P[k] * ref[k], FLOOR[k]), (k, dev[k], ref[k])
        if ref[k] <= RTOL:
            assert dev[k] <= RTOL, (k, dev[k], ref[k])
    assert max(dev.values()) <= PIN[name] and dev["F"] <= PIN_F[name], (name, dev)
    # the incumbent's input is the first pending row: its fantasies can only raise best_s
    assert np.all(fant.best >= r["sk_p1_best"] - 1e-8 * (np.abs(r["sk_p1_best"]) + float(r["y_std"])))
