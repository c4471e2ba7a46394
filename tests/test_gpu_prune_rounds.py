"""The merged k-th key, the final rounds and the shared K* of pruning's refine stages (DESIGN.md 4.9).

The records (value bits and indices) must equal those of the unpruned call: for EI, UCB, PoI and LogEI, k = 1 / 10 /
64, every covariance code with and without candidate registers, ragged batch and training sizes, streamed host batches,
the Philox source, a batch split into launches of kPruneMaxBatch, a batch with a NaN value and UCB with kappa = 100
(the tile kernel takes over).  At the C3 shape the refine stage runs, and no candidate goes through the full N^2 term
but the lead tiles' and the level's survivors: the final stage closes the tile kernel's counter.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

SETTINGS = ("0", "1")  # B200BO_PRUNE
LEAD_TILES, PBN = 8, 128  # kLeadTiles, candidates per tile


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED", "B200BO_PRUNE_REFINE", "B200BO_PRUNE_REFINE_BLOCKS", "B200BO_PRUNE_BOUND"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _acq(bo, gp, kind, y, kappa=2.576):
    from bayesianoptimization_b200 import _lib as B

    code = {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI, "logei": B.ACQ_LOGEI}[kind]
    return bo.FusedAcquisition(code, gp, kappa=kappa, xi=0.01, y_max=float(np.max(y)))


def _all(monkeypatch, fn):
    """fn() under every setting: its results and the evaluated / refined counts of the pruned ones."""
    from bayesianoptimization_b200 import _lib as B

    out, stats = [], []
    for prune in SETTINGS:
        monkeypatch.setenv("B200BO_PRUNE", prune)
        out.append(fn())
        ev, tot, ref = C.c_int64(), C.c_int64(), C.c_int64()
        B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        if prune == "1":
            ms = (C.c_float * 6)()
            B.check(B.lib().b200bo_last_prune_stage_ms(ms, C.byref(ref)))
            assert all(v >= 0.0 for v in ms)
        stats.append((ev.value, ref.value))
    return out, stats


def _equal(out):
    return all(np.array_equal(out[0], o) for o in out[1:])


def _host(acq, x, k):
    idx, val, top = acq.argmin_topk(x, k)
    return repr((idx, int(np.float64(val).view(np.int64)), list(top)))  # repr of a float is exact


def _dev(acq, xd, k, index_base=0):
    import torch

    from bayesianoptimization_b200 import _lib as B

    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), xd.shape[0], None, None, None, k,
                                        sel.data_ptr(), index_base, s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _philox(acq, d, m, k, seed=99, index_base=1000):
    import torch

    from bayesianoptimization_b200 import _lib as B

    lo, hi = np.zeros(d), np.ones(d)
    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_select_philox_dev(C.byref(acq.spec), seed, B.as_dp(lo), B.as_dp(hi), m, index_base,
                                                 k, sel.data_ptr(), s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _problem(n, d, seed):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    return X, np.sin(X.sum(1)) + 0.1 * rs.randn(n)


def _gp(bo, X, y, kernel):
    return bo.B200GaussianProcessRegressor(kernel=kernel, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)


def test_c3_shape_evaluates_lead_and_level_survivors(bo, monkeypatch):
    import torch

    from bayesianoptimization_b200 import _lib as B

    X, y = _problem(4096, 16, 0)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.7))
    acq = _acq(bo, gp, "ei", y)
    xd = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 20, 16))).cuda()
    out, stats = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    ms, passed, nlev = C.c_float(), (C.c_int64 * 5)(), C.c_int()
    B.check(B.lib().b200bo_last_prune_levels(C.byref(ms), passed, C.byref(nlev)))
    assert _equal(out)
    evaluated, refined = stats[1]
    assert refined > 0, stats  # the stages ran
    assert nlev.value == 1 and 0 < passed[1] < passed[0], (nlev.value, list(passed))
    # the lead tiles and the final rounds over the level's survivors; the tile kernel evaluates nothing
    assert evaluated <= LEAD_TILES * PBN + passed[1], (stats, list(passed))
    print(f"c3: evaluated {evaluated}, refined {refined}, passed {list(passed)[:2]}")


@pytest.mark.parametrize("kind", ("ei", "ucb", "poi", "logei"))
@pytest.mark.parametrize("k", (1, 10, 64))
def test_kinds_and_k(bo, monkeypatch, kind, k):
    import torch

    X, y = _problem(1000, 6, 3)  # ragged: np = 1024
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, kind, y)
    xd = torch.from_numpy(np.random.RandomState(7).uniform(size=((1 << 17) - 37, 6))).cuda()
    out, stats = _all(monkeypatch, lambda: _dev(acq, xd, k, index_base=12345))
    assert _equal(out), (kind, k)


@pytest.mark.parametrize("case", sorted(KM.PREDICT))
def test_kernel_matrix_cases_streamed(bo, monkeypatch, case):
    """Every covariance code, ARD, WhiteKernel, the round transform and d > 16 (no candidate registers), as a host
    batch streamed in chunks, with copies of training points (clamped variance)."""
    c = KM.PREDICT[case]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, seed=11)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    acq = _acq(bo, gp, "ei", y)
    x = np.vstack([KM.inputs(c, (1 << 18) - 128, d, rs), X[:64], X[:64] + 1e-9])
    out, stats = _all(monkeypatch, lambda: _host(acq, x, 10))
    assert _equal(out), case


def test_d17_large_training_set(bo, monkeypatch):
    import torch

    X, y = _problem(2100, 17, 5)
    gp = _gp(bo, X, y, Matern(nu=1.5, length_scale=1.0))
    acq = _acq(bo, gp, "ei", y)
    xd = torch.from_numpy(np.random.RandomState(8).uniform(size=((1 << 17) + 5, 17))).cuda()
    out, _ = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    assert _equal(out)


def test_ucb_kappa_100_hands_over(bo, monkeypatch):
    import torch

    X, y = _problem(1500, 8, 9)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, "ucb", y, kappa=100.0)
    xd = torch.from_numpy(np.random.RandomState(10).uniform(size=(1 << 16, 8))).cuda()
    out, _ = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    assert _equal(out)


def test_philox_source_and_split_batch(bo, monkeypatch):
    """A Philox batch of more than kPruneMaxBatch = 2^22 candidates runs as launches that continue the lists."""
    X, y = _problem(1200, 5, 13)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.4))
    acq = _acq(bo, gp, "ei", y)
    for m in ((1 << 18) + 77, (1 << 22) + 3000):
        out, _ = _all(monkeypatch, lambda: _philox(acq, 5, m, 10))
        assert _equal(out), m


def test_nan_value_is_reported(bo, monkeypatch):
    import torch

    X, y = _problem(1000, 4, 21)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    x = np.random.RandomState(22).uniform(size=(1 << 16, 4))
    x[40000] = X[int(np.argmax(y))]
    xd = torch.from_numpy(x).cuda()
    for kind in ("ei", "poi"):
        acq = _acq(bo, gp, kind, y)
        out, _ = _all(monkeypatch, lambda: _dev(acq, xd, 10))
        assert _equal(out), kind
