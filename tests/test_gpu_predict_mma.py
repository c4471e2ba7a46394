"""Phase B of the fused fp64 predict kernel on the sm_90 MMA shape (default) against the sm_80 shape m8n8k4
(B200BO_PREDICT_MMA=884) on the same fitted GPs.

Phase A (K* and K* alpha_) is shared, so mu must be bit-equal.  sigma^2 = prior - sum_i V_i^2 where only the
summation order of V = L^-1 K*^T changes, so sigma and the acquisition agree to round-off: 1e-12 relative, plus an
absolute floor of 1e-12 of the array's scale where sigma is near 0.  Selection (argmin, top-10) is identical, and a
candidate's values do not depend on the batch it is evaluated in."""
import numpy as np
import pytest
from numpy.testing import assert_allclose
from sklearn.gaussian_process.kernels import Matern

pytestmark = pytest.mark.gpu

RTOL = 1e-12


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    """The 16-warp fp64 tiled kernel for every batch size (the small-batch kernels have no phase B)."""
    monkeypatch.setenv("B200BO_PREDICT_IMPL", "dmma")
    monkeypatch.setenv("B200BO_PREDICT_WARPS", "16")
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


class _Constraints:  # duck type of bayes_opt's ConstraintModel as FusedAcquisition reads it
    def __init__(self, models, lb, ub):
        self.model, self.lb, self.ub = models, np.asarray(lb, float), np.asarray(ub, float)


def _gp(bo, X, y, ls):
    return bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=ls), alpha=1e-6, normalize_y=True,
                                           optimizer=None).fit(X, y)


def _problem(n, d, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    return X, np.sin(X.sum(1)) + 0.1 * rs.randn(n)


def _evaluate(monkeypatch, mma, gp, f, xt):
    if mma is None:
        monkeypatch.delenv("B200BO_PREDICT_MMA", raising=False)
    else:
        monkeypatch.setenv("B200BO_PREDICT_MMA", mma)
    mu, sd = gp.predict(xt, return_std=True)
    acq = f(xt)
    idx, val, top = f.argmin_topk(xt, 10)
    return dict(mu=mu, sd=sd, acq=acq, idx=idx, val=val, top=list(top))


def _close(a, b):
    scale = float(np.max(np.abs(b)))
    assert_allclose(a, b, rtol=RTOL, atol=RTOL * scale)


def _compare(new, old):
    assert np.array_equal(new["mu"], old["mu"])
    _close(new["sd"], old["sd"])
    _close(new["acq"], old["acq"])
    assert new["idx"] == old["idx"]
    assert new["top"] == old["top"]


CASES = {
    # name: N_train, d, acquisition, constraint GPs, candidates
    "c3": (4096, 16, "ei", 0, 1 << 16),
    "d32_ragged": (1500, 32, "ucb", 0, 20000),
    "ei_2con_ragged": (1000, 5, "ei", 2, 30000),
    "ucb_2con_ragged": (1000, 5, "ucb", 2, 30000),
    "poi_2con_ragged": (1000, 5, "poi", 2, 30000),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sm90_shape_matches_m8n8k4(bo, monkeypatch, case):
    from bayesianoptimization_b200 import _lib as B

    n, d, kind, ncon, m = CASES[case]
    X, y = _problem(n, d)
    gp = _gp(bo, X, y, 0.7 if d == 16 else 1.0)
    cons = None
    if ncon:
        models = [_gp(bo, X, np.cos((j + 1) * X.sum(1)), 0.6) for j in range(ncon)]
        cons = _Constraints(models, [-0.5, -0.8][:ncon], [0.7, 0.9][:ncon])
    kinds = {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI}
    f = bo.FusedAcquisition(kinds[kind], gp, cons, kappa=2.576, xi=0.01, y_max=float(y.max()))
    xt = np.random.RandomState(7).uniform(size=(m, d))
    new = _evaluate(monkeypatch, None, gp, f, xt)
    old = _evaluate(monkeypatch, "884", gp, f, xt)
    _compare(new, old)
    # the new default shape: a candidate's values do not depend on the batch (tile position, grid size)
    monkeypatch.delenv("B200BO_PREDICT_MMA", raising=False)
    for a, b in ((0, 1), (12345, 12345 + 1000), (m - 129, m)):
        mu, sd = gp.predict(xt[a:b], return_std=True)
        assert np.array_equal(mu, new["mu"][a:b])
        assert np.array_equal(sd, new["sd"][a:b])
        assert np.array_equal(f(xt[a:b]), new["acq"][a:b])
