"""The refine stages of selection-only pruning (B200BO_PRUNE_REFINE, DESIGN.md 4.9).

With the stages on, a pruned selection call evaluates the first tiles in bound order split across SMs by row block,
bounds the following tiles by the leading row blocks of L^-1, and evaluates what is left split the same way.  The
records (value bits and indices) must equal those of the unpruned call and of pruning without the stages: for EI, UCB
and PoI, k = 1 / 10 / 64, every covariance code with and without candidate registers, ragged batch and training sizes,
both phase-B pipes, streamed host batches, the Philox source, UCB with kappa = 100 (little prunes: the final stage
hands over to the tile kernel), and a batch with a NaN value.  At the C3 shape the stages must run (a refined count)
and send strictly fewer candidates through the full N^2 term.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

KINDS = ("ei", "ucb", "poi")
SETTINGS = (("0", "1"), ("1", "0"), ("1", "1"))  # (B200BO_PRUNE, B200BO_PRUNE_REFINE)


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED", "B200BO_PRUNE_REFINE_BLOCKS"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _acq(bo, gp, kind, y, kappa=2.576):
    from bayesianoptimization_b200 import _lib as B

    code = {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI}[kind]
    return bo.FusedAcquisition(code, gp, kappa=kappa, xi=0.01, y_max=float(np.max(y)))


def _three(monkeypatch, fn):
    """fn() unpruned, pruned without and with the refine stages: results and (evaluated, refined) of each."""
    from bayesianoptimization_b200 import _lib as B

    out, stats = [], []
    for prune, refine in SETTINGS:
        monkeypatch.setenv("B200BO_PRUNE", prune)
        monkeypatch.setenv("B200BO_PRUNE_REFINE", refine)
        out.append(fn())
        ev, tot, ref = C.c_int64(), C.c_int64(), C.c_int64()
        B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        if prune == "1":
            ms = (C.c_float * 6)()
            B.check(B.lib().b200bo_last_prune_stage_ms(ms, C.byref(ref)))
            assert all(v >= 0.0 for v in ms)
        stats.append((ev.value, ref.value))
    return out, stats


def _host(acq, x, k):
    idx, val, top = acq.argmin_topk(x, k)
    return idx, np.float64(val).view(np.int64), list(top)


def _dev(acq, xd, k, index_base=0):
    import torch

    from bayesianoptimization_b200 import _lib as B

    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), xd.shape[0], None, None, None, k,
                                        sel.data_ptr(), index_base, s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _problem(n, d, seed):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    return X, np.sin(X.sum(1)) + 0.1 * rs.randn(n)


def _gp(bo, X, y, kernel):
    return bo.B200GaussianProcessRegressor(kernel=kernel, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)


@pytest.mark.parametrize("pipe", ("bulk_nomc", "cpasync"))
def test_c3_shape_fewer_evaluated(bo, monkeypatch, pipe):
    import torch

    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    X, y = _problem(4096, 16, 0)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.7))
    acq = _acq(bo, gp, "ei", y)
    xd = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 18, 16))).cuda()
    (off, plain, refined), stats = _three(monkeypatch, lambda: _dev(acq, xd, 10))
    assert np.array_equal(off, plain) and np.array_equal(off, refined)
    assert stats[1][1] == 0 and stats[2][1] > 0, stats  # the stages ran, and only when asked
    assert stats[2][0] < stats[1][0], stats
    print(f"c3 2^18 {pipe}: evaluated {stats[1][0]} -> {stats[2][0]}, refined {stats[2][1]}")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("k", (1, 10, 64))
def test_kinds_and_k(bo, monkeypatch, kind, k):
    import torch

    X, y = _problem(1000, 6, 3)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, kind, y)
    xd = torch.from_numpy(np.random.RandomState(7).uniform(size=((1 << 17) - 37, 6))).cuda()
    (off, plain, refined), stats = _three(monkeypatch, lambda: _dev(acq, xd, k, index_base=12345))
    assert np.array_equal(off, plain) and np.array_equal(off, refined), kind
    assert stats[2][0] < xd.shape[0]


@pytest.mark.parametrize("case", sorted(KM.PREDICT))
def test_kernel_matrix_cases_streamed(bo, monkeypatch, case):
    """Every covariance code, ARD, WhiteKernel, the round transform and d > 16 (no candidate registers), as a host
    batch streamed in chunks, with copies of training points (clamped variance) and a ragged training size."""
    c = KM.PREDICT[case]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, seed=11)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    acq = _acq(bo, gp, "ei", y)
    x = np.vstack([KM.inputs(c, (1 << 18) - 128, d, rs), X[:64], X[:64] + 1e-9])
    (off, plain, refined), stats = _three(monkeypatch, lambda: _host(acq, x, 10))
    assert off == plain and off == refined, case
    print(f"{case}: evaluated {stats[1][0]} -> {stats[2][0]}, refined {stats[2][1]}")


def test_d32_large_training_set(bo, monkeypatch):
    import torch

    X, y = _problem(2100, 32, 5)
    gp = _gp(bo, X, y, Matern(nu=1.5, length_scale=1.0))
    acq = _acq(bo, gp, "ucb", y)
    xd = torch.from_numpy(np.random.RandomState(8).uniform(size=((1 << 16) + 5, 32))).cuda()
    (off, plain, refined), stats = _three(monkeypatch, lambda: _dev(acq, xd, 10))
    assert np.array_equal(off, plain) and np.array_equal(off, refined)
    assert stats[2][0] <= stats[1][0], stats


def test_ucb_kappa_100_hands_over(bo, monkeypatch):
    """sigma dominates the value: the refined bound lets more through than the final stage takes, and the tile kernel
    goes on in bound order."""
    import torch

    X, y = _problem(1500, 8, 9)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, "ucb", y, kappa=100.0)
    xd = torch.from_numpy(np.random.RandomState(10).uniform(size=(1 << 16, 8))).cuda()
    (off, plain, refined), stats = _three(monkeypatch, lambda: _dev(acq, xd, 10))
    assert np.array_equal(off, plain) and np.array_equal(off, refined)


def test_philox_source(bo, monkeypatch):
    import torch

    from bayesianoptimization_b200 import _lib as B

    X, y = _problem(1200, 5, 13)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.4))
    acq = _acq(bo, gp, "ei", y)
    lo, hi, m, k = np.zeros(5), np.ones(5), (1 << 18) + 77, 10

    def run():
        sel = torch.zeros((k + 1, 2), dtype=torch.int64, device="cuda")
        s = torch.cuda.current_stream()
        B.check(B.lib().b200bo_acq_select_philox_dev(C.byref(acq.spec), 99, B.as_dp(lo), B.as_dp(hi), m, 1000, k,
                                                     sel.data_ptr(), s.cuda_stream))
        s.synchronize()
        return sel.cpu().numpy()

    (off, plain, refined), stats = _three(monkeypatch, run)
    assert np.array_equal(off, plain) and np.array_equal(off, refined)


def test_nan_value_is_reported(bo, monkeypatch):
    """A candidate on a training point with a = 0 and sigma = 0 gives the NaN np.argmin reports first; it is never
    pruned, with or without the stages."""
    import torch

    X, y = _problem(1000, 4, 21)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    x = np.random.RandomState(22).uniform(size=(1 << 16, 4))
    x[40000] = X[int(np.argmax(y))]
    xd = torch.from_numpy(x).cuda()
    for kind in ("ei", "poi"):
        acq = _acq(bo, gp, kind, y)
        (off, plain, refined), _ = _three(monkeypatch, lambda: _dev(acq, xd, 10))
        assert np.array_equal(off, plain) and np.array_equal(off, refined), kind
