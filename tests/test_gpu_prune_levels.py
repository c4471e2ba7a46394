"""The refine level of pruning (DESIGN.md 4.9): the refine stage's survivors carry their running sums of squares into
a level over the next row blocks, which keys them again, and into the final stage.

The records (value bits and indices) must equal those of the unpruned call: at the C3 shape, on the ill-conditioned
production-size fixtures, for a streamed (continued) host batch, for the Philox source and at N = 1024 (one leading row
block, a level to two).  At C3 the level lets fewer candidates through than the refine stage, and no candidate goes
through the full N^2 term but the lead tiles' and the level's survivors.  Repeat calls are bit-identical, and where the
refine stage lets candidates through but the level lets none (illbig_b_m25_c3, EI), the final stage evaluates nothing
and the records still hold.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

from oracle import make_illcond as MI
from oracle import make_illcond_big as MB

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


def _levels():
    """(levels run, candidates the refine stage and each level let through) of the last pruned launch"""
    from bayesianoptimization_b200 import _lib as B

    ms, passed, n = C.c_float(), (C.c_int64 * 5)(), C.c_int()
    B.check(B.lib().b200bo_last_prune_levels(C.byref(ms), passed, C.byref(n)))
    assert ms.value >= 0.0
    return n.value, list(passed)[:n.value + 1]


def _all(monkeypatch, fn):
    """fn() under every setting: its results, and per pruned setting (evaluated, levels, passed)"""
    from bayesianoptimization_b200 import _lib as B

    out, stats = [], []
    for prune in SETTINGS:
        monkeypatch.setenv("B200BO_PRUNE", prune)
        out.append(fn())
        ev, tot = C.c_int64(), C.c_int64()
        B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
        stats.append((ev.value, *_levels()) if prune == "1" else None)
    return out, stats


def _equal(out):
    return all(np.array_equal(out[0], o) for o in out[1:])


def _dev(acq, xd, k, index_base=0):
    import torch

    from bayesianoptimization_b200 import _lib as B

    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), xd.shape[0], None, None, None, k,
                                        sel.data_ptr(), index_base, s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _host(acq, x, k):
    idx, val, top = acq.argmin_topk(x, k)
    return repr((idx, int(np.float64(val).view(np.int64)), list(top)))  # repr of a float is exact


def _c3(bo):
    from bayesianoptimization_b200 import _lib as B

    rs = np.random.RandomState(0)
    X = rs.uniform(size=(4096, 16))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(4096)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    return bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))


def test_c3_one_level_and_evaluated_bound(bo, monkeypatch):
    import torch

    acq = _c3(bo)
    xd = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 20, 16))).cuda()
    out, stats = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    print(f"\nc3 (evaluated, levels, passed) per setting: {stats}")
    assert _equal(out)
    ev, nlev, passed = stats[1]
    assert nlev == 1 and 0 < passed[1] < passed[0] <= 128 * 128, stats
    # the lead tiles and the final rounds over the level's survivors; the tile kernel evaluates nothing
    assert ev <= LEAD_TILES * PBN + passed[1], stats
    # repeat calls: bit-identical records
    monkeypatch.setenv("B200BO_PRUNE", "1")
    for _ in range(3):
        assert np.array_equal(_dev(acq, xd, 10), out[0])


def test_c3_streamed_host_batch(bo, monkeypatch):
    """A host batch goes up in chunks; every chunk's launch continues the lists and the k-th key of the last."""
    acq = _c3(bo)
    x = np.random.RandomState(1001).uniform(size=(1 << 20, 16))
    out, stats = _all(monkeypatch, lambda: _host(acq, x, 10))
    assert _equal(out), out


def test_c3_philox(bo, monkeypatch):
    import torch

    from bayesianoptimization_b200 import _lib as B

    acq = _c3(bo)
    lo, hi = np.zeros(16), np.ones(16)

    def run():
        sel = torch.zeros((11, 2), dtype=torch.int64, device="cuda")
        s = torch.cuda.current_stream()
        B.check(B.lib().b200bo_acq_select_philox_dev(C.byref(acq.spec), 12345, B.as_dp(lo), B.as_dp(hi), 1 << 20,
                                                     0, 10, sel.data_ptr(), s.cuda_stream))
        s.synchronize()
        return sel.cpu().numpy()

    out, stats = _all(monkeypatch, run)
    assert _equal(out)
    assert stats[1][1] == 1 and stats[1][2][1] < stats[1][2][0], stats


@pytest.mark.parametrize("kind", ("ucb", "ei"))
@pytest.mark.parametrize("name", sorted(MB.CASES))
def test_illcond_big(bo, monkeypatch, name, kind):
    """Eight copies of the fixture's candidates, so that the refine stage and the level see candidates."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    c, r = MB.CASES[name], MB.load(name)
    gp = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                         optimizer=None).fit(r["X"], r["y"])
    code = {"ucb": B.ACQ_UCB, "ei": B.ACQ_EI}[kind]
    acq = bo.FusedAcquisition(code, gp, kappa=MI.KAPPA, xi=MI.XI, y_max=float(np.max(r["y"])))
    xd = torch.from_numpy(np.tile(r["xt"], (8, 1))).cuda()
    out, stats = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    print(f"\n{name} {kind}: {stats}")
    assert _equal(out), (name, kind)
    if (name, kind) == ("b_m25_c3", "ei"):  # nothing survives the level: only the lead tiles are evaluated
        ev, nlev, passed = stats[1]
        assert nlev == 1 and passed[0] > 0 and passed[1] == 0 and ev == 1024, stats


def test_n1024(bo, monkeypatch):
    """N = 1024: one leading row block, a level to two."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    rs = np.random.RandomState(0)
    X = rs.uniform(size=(1024, 8))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(1024)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    acq = bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
    xd = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 20, 8))).cuda()
    out, stats = _all(monkeypatch, lambda: _dev(acq, xd, 10))
    print(f"\nn1024: {stats}")
    assert _equal(out)
    assert stats[1][1] == 1 and 0 < stats[1][2][1] <= stats[1][2][0], stats
