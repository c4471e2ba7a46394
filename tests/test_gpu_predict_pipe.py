"""Phase B data paths of the 16-warp fp64 predict kernel (B200BO_PREDICT_PIPE) on the same fitted GPs.

`bulk` (bulk copies on an mbarrier ring, L^-1 multicast across CTA pairs), `bulk_nomc` (the same without clusters)
and `cpasync` (per-thread cp.async under CTA barriers) stage the same operands into the same shared-memory layout and
run the same MMAs in the same order, so mu, sigma, the acquisition and the selection (argmin, top-10) are bit-equal.
The cases cover both candidate-register paths (d <= 16 and d = 17), constraint GPs, a training size that is not a
multiple of 128, tile counts that are odd, below the grid and one past a multiple of it, and the streamed host batches
whose per-CTA selection lists carry over from launch to launch."""
import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

pytestmark = pytest.mark.gpu

PIPES = ("cpasync", "bulk_nomc", "bulk")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    """The 16-warp fp64 tiled kernel on m16n8k4 for every batch size (the small-batch kernels have no phase B)."""
    monkeypatch.setenv("B200BO_PREDICT_IMPL", "dmma")
    monkeypatch.setenv("B200BO_PREDICT_WARPS", "16")
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")
    monkeypatch.delenv("B200BO_PREDICT_MMA", raising=False)


class _Constraints:  # duck type of bayes_opt's ConstraintModel as FusedAcquisition reads it
    def __init__(self, models, lb, ub):
        self.model, self.lb, self.ub = models, np.asarray(lb, float), np.asarray(ub, float)


def _gp(bo, X, y, ls):
    return bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=ls), alpha=1e-6, normalize_y=True,
                                           optimizer=None).fit(X, y)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(n):
    return n * 128 - 37  # n tiles, the last one ragged


CASES = {
    # name: N_train, d, acquisition, constraint GPs, candidates (a callable of the SM count)
    "c3": (4096, 16, "ei", 0, lambda sm: 1 << 16),
    "poi_2con": (1000, 5, "poi", 2, lambda sm: 30000),
    "n_ragged_ucb": (1500, 8, "ucb", 0, lambda sm: 20000),
    "d17": (700, 17, "ei", 0, lambda sm: 25000),
    "tiles_odd_below_grid": (600, 6, "ei", 1, lambda sm: _tiles(5)),
    "tiles_one": (600, 6, "ucb", 0, lambda sm: 50),
    "tiles_grid_plus_one": (600, 6, "ei", 0, lambda sm: _tiles(2 * sm + 1)),
    "tiles_odd_above_grid": (600, 17, "poi", 1, lambda sm: _tiles(3 * sm - 1)),
}


def _evaluate(monkeypatch, pipe, gp, f, xt):
    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    mu, sd = gp.predict(xt, return_std=True)
    acq = f(xt)
    idx, val, top = f.argmin_topk(xt, 10)
    return dict(mu=mu, sd=sd, acq=acq, idx=idx, val=val, top=list(top))


def _assert_bit_equal(new, old, label):
    for key in ("mu", "sd", "acq"):
        assert np.array_equal(new[key], old[key], equal_nan=True), f"{label}: {key} differs"
    assert new["idx"] == old["idx"], label
    assert np.array_equal(np.asarray(new["val"]), np.asarray(old["val"]), equal_nan=True), label
    assert new["top"] == old["top"], label


@pytest.mark.parametrize("case", sorted(CASES))
def test_pipes_bit_equal(bo, monkeypatch, case):
    from bayesianoptimization_b200 import _lib as B

    n, d, kind, ncon, mfun = CASES[case]
    m = mfun(_sm_count())
    rs = np.random.RandomState(0)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    gp = _gp(bo, X, y, 0.7 if d == 16 else 1.0)
    cons = None
    if ncon:
        models = [_gp(bo, X, np.cos((j + 1) * X.sum(1)), 0.6) for j in range(ncon)]
        cons = _Constraints(models, [-0.5, -0.8][:ncon], [0.7, 0.9][:ncon])
    kinds = {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI}
    f = bo.FusedAcquisition(kinds[kind], gp, cons, kappa=2.576, xi=0.01, y_max=float(y.max()))
    xt = np.random.RandomState(7).uniform(size=(m, d))
    out = {p: _evaluate(monkeypatch, p, gp, f, xt) for p in PIPES}
    for p in PIPES[1:]:
        _assert_bit_equal(out[p], out["cpasync"], f"{case}: {p} vs cpasync")


def test_pipes_streamed_batches(bo, monkeypatch):
    """argmin_topk on a host batch large enough to be streamed in chunks: the per-CTA selection lists of the
    clustered launch carry over from chunk to chunk and are merged once."""
    n, d = 300, 4
    m = 3 * 8 * 128 * _sm_count()  # three chunks of kChunkTilesPerSm tiles per SM
    rs = np.random.RandomState(1)
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1))
    gp = _gp(bo, X, y, 0.5)
    from bayesianoptimization_b200 import _lib as B

    f = bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
    xt = np.random.RandomState(9).uniform(size=(m, d))
    res = {}
    for p in PIPES:
        monkeypatch.setenv("B200BO_PREDICT_PIPE", p)
        idx, val, top = f.argmin_topk(xt, 10)
        res[p] = (idx, float(val), list(top))
    assert res["bulk"] == res["cpasync"]
    assert res["bulk_nomc"] == res["cpasync"]
    monkeypatch.setenv("B200BO_CHUNKED", "0")
    monkeypatch.setenv("B200BO_PREDICT_PIPE", "cpasync")
    idx, val, top = f.argmin_topk(xt, 10)
    assert (idx, float(val), list(top)) == res["bulk"]
