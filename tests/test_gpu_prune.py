"""Selection-only pruning of the 16-warp fp64 predict kernel (B200BO_PRUNE, DESIGN.md 4.9).

A selection-only call (argmin + top-k, no values materialised) of EI, UCB or PoI on one GP first bounds every
candidate's acquisition from phase-A quantities alone and then runs the N^2 term only on the tiles, in bound order,
whose best bound can still enter the top-k.  Pruned candidates provably cannot, so the records must be bit-equal to the
unpruned path: value bits and indices, for every covariance code, both candidate-register paths and d > 16, ragged
batch sizes, k = 1 / 10 / 64, a non-zero index base, the Philox source, streamed host batches of several chunks and
candidates that duplicate training points (clamped variance), and batches split into several pruned launches.  Every
bit-equality case also requires fewer candidates evaluated than given, so the pruned path is the one under test.  The
keys the device's bound pass writes (b200bo_acq_prune_bound_dev) are checked against the keys of the exact values of
the same candidates, and at the C3 shape most candidates must be skipped.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

KINDS = ("ei", "ucb", "poi")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _acq(bo, gp, kind, y):
    from bayesianoptimization_b200 import _lib as B

    code = {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI}[kind]
    return bo.FusedAcquisition(code, gp, kappa=2.576, xi=0.01, y_max=float(np.max(y)))


def _both(monkeypatch, fn):
    """fn() with pruning off, then on; returns both results and the prune stats of the second call."""
    from bayesianoptimization_b200 import _lib as B

    monkeypatch.setenv("B200BO_PRUNE", "0")
    off = fn()
    monkeypatch.setenv("B200BO_PRUNE", "1")
    on = fn()
    ev, tot = C.c_int64(), C.c_int64()
    B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
    return off, on, (ev.value, tot.value)


def _host(acq, x, k):
    idx, val, top = acq.argmin_topk(x, k)
    return idx, np.float64(val).view(np.int64), list(top)


def _dev(acq, xd, k, index_base=0):
    """b200bo_acq_eval_dev: raw (value bits, index) records."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), xd.shape[0], None, None, None, k,
                                        sel.data_ptr(), index_base, s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _c3_problem(n=4096, d=16, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    return X, np.sin(X.sum(1)) + 0.1 * rs.randn(n)


def _gp(bo, X, y, kernel):
    return bo.B200GaussianProcessRegressor(kernel=kernel, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)


def test_c3_shape_bit_equal_and_mostly_pruned(bo, monkeypatch):
    import torch

    X, y = _c3_problem()
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.7))
    acq = _acq(bo, gp, "ei", y)
    xd = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 18, 16))).cuda()
    off, on, (ev, tot) = _both(monkeypatch, lambda: _dev(acq, xd, 10))
    assert np.array_equal(off, on)
    assert tot == 1 << 18
    assert ev < 0.25 * tot, f"{ev} of {tot} candidates evaluated"
    print(f"c3 2^18: {ev} of {tot} evaluated ({ev / tot:.3%})")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("k", (1, 10, 64))
def test_kinds_and_k(bo, monkeypatch, kind, k):
    import torch

    X, y = _c3_problem(n=1000, d=6, seed=3)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, kind, y)
    xd = torch.from_numpy(np.random.RandomState(7).uniform(size=((1 << 17) - 37, 6))).cuda()
    off, on, (ev, tot) = _both(monkeypatch, lambda: _dev(acq, xd, k, index_base=12345))
    assert np.array_equal(off, on), kind
    assert off[1, 1] >= 12345
    assert tot == xd.shape[0] and ev < tot  # the pruned path is the one under test


@pytest.mark.parametrize("case", sorted(KM.PREDICT))
@pytest.mark.parametrize("kind", KINDS)
def test_kernel_matrix_cases(bo, monkeypatch, case, kind):
    """Every covariance code, ARD, WhiteKernel and the round transform; d = 17 / 33 / 40 / 64 run without DREG.
    The batch holds copies of training points (clamped variance) and a training size not a multiple of 128."""
    c = KM.PREDICT[case]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, seed=11)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    acq = _acq(bo, gp, kind, y)
    x = np.vstack([KM.inputs(c, (1 << 17) - 128, d, rs), X[:64], X[:64] + 1e-9])
    off, on, (ev, tot) = _both(monkeypatch, lambda: _host(acq, x, 10))
    assert off == on, case
    print(f"{case} {kind}: {ev} of {tot} evaluated")
    assert tot == x.shape[0] and ev < tot


def test_d32_no_dreg(bo, monkeypatch):
    import torch

    X, y = _c3_problem(n=2000, d=32, seed=5)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=1.0))
    acq = _acq(bo, gp, "ei", y)
    xd = torch.from_numpy(np.random.RandomState(9).uniform(size=(1 << 17, 32))).cuda()
    off, on, (ev, tot) = _both(monkeypatch, lambda: _dev(acq, xd, 10))
    assert np.array_equal(off, on)
    assert tot == xd.shape[0] and ev < tot


def test_philox_batch_split(bo, monkeypatch):
    """A pruned batch larger than kPruneMaxBatch (2^22) runs as consecutive launches that continue the selection."""
    X, y = _c3_problem(n=600, d=6, seed=8)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.5))
    acq = _acq(bo, gp, "ei", y)
    bounds = np.column_stack([np.zeros(6), np.ones(6)])
    m = (1 << 22) + (1 << 20) + 77

    def run():
        idx, val, bx, ti, tx = acq.argmin_topk_philox(5, bounds, m, 10, index_base=3)
        return idx, np.float64(val).view(np.int64), list(ti), bx.tobytes()

    off, on, (ev, tot) = _both(monkeypatch, run)
    assert off == on
    assert tot == m and ev < tot


@pytest.mark.parametrize("pipe", ("bulk_nomc", "cpasync"))
def test_philox_source(bo, monkeypatch, pipe):
    monkeypatch.setenv("B200BO_PREDICT_PIPE", pipe)
    X, y = _c3_problem(n=1500, d=8, seed=2)
    gp = _gp(bo, X, y, Matern(nu=1.5, length_scale=0.6))
    acq = _acq(bo, gp, "ei", y)
    bounds = np.column_stack([np.zeros(8), np.ones(8)])

    def run():
        idx, val, bx, ti, tx = acq.argmin_topk_philox(77, bounds, 150000, 10, index_base=1 << 33)
        return idx, np.float64(val).view(np.int64), list(ti), bx.tobytes(), tx.tobytes()

    off, on, (ev, tot) = _both(monkeypatch, run)
    assert off == on
    assert ev < tot


def test_streamed_host_batch(bo, monkeypatch):
    """More than two chunks: the per-CTA lists and the k-th key word carry over from chunk to chunk."""
    import torch

    X, y = _c3_problem(n=1024, d=8, seed=4)
    gp = _gp(bo, X, y, Matern(nu=2.5, length_scale=0.6))
    acq = _acq(bo, gp, "ei", y)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    m = int(2.5 * 8 * 128 * sm) + 17  # 3 chunks of 8 tiles per SM, the last one ragged
    x = np.random.RandomState(21).uniform(size=(m, 8))
    off, on, (ev, tot) = _both(monkeypatch, lambda: _host(acq, x, 10))
    assert off == on
    assert tot == m and ev < m


def _order_keys(v):
    """key_nan_last of select.cuh: the order of (value, NaN last) as uint64."""
    v = np.where(v == 0.0, 0.0, v)
    u = v.view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    return np.where(np.isnan(v), np.uint64(0xFFFFFFFFFFFFFFFF), key)


BOUND_CASES = [(c, kind) for c in sorted(KM.PREDICT) for kind in KINDS] + [("c3", kind) for kind in KINDS]


@pytest.mark.parametrize("case,kind", BOUND_CASES)
def test_device_bound_below_exact(bo, case, kind):
    """The keys the bound pass writes (b200bo_acq_prune_bound_dev) are never above the key of the exact closure value
    of the same candidate (b200bo_acq_eval_dev with d_acq_neg), training copies and near-duplicates included; key 0
    marks exactly the candidates of the never-prune rule; max |K*_i| matches sklearn.  Also reports how far the
    computed sum of squares of the explicit inverse falls below max K*_i^2 / K_ii, against kPruneVarEps = 1e-8."""
    import torch

    from bayesianoptimization_b200 import _lib as B
    from test_prune_cpu import VAR_EPS, never_prune

    if case == "c3":
        X, y = _c3_problem()
        d, kern = 16, Matern(nu=2.5, length_scale=0.7)
        rs = np.random.RandomState(1000)
        cand = rs.uniform(size=(1 << 16, d))
    else:
        c = KM.PREDICT[case]
        n, d = c["n"], c["d"]
        X, y, rs = KM.problem(c, n, d, seed=11)
        kern = KM.kernel(c, d)
        cand = KM.inputs(c, 4000, d, rs)
    gp = bo.B200GaussianProcessRegressor(kernel=kern, alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
    acq = _acq(bo, gp, kind, y)
    x = np.vstack([cand, X[:64], X[:64] + 1e-9])
    m = x.shape[0]
    xd = torch.from_numpy(x).cuda()
    acq_o, mu, sd, kmax = (torch.empty(m, dtype=torch.float64, device="cuda") for _ in range(4))
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), m, acq_o.data_ptr(), mu.data_ptr(), sd.data_ptr(),
                                  0, None, 0, s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(acq.spec), xd.data_ptr(), m, key.data_ptr(), kmax.data_ptr(),
                                         s.cuda_stream))
    s.synchronize()
    exact, mu, sd, kmax = (t.cpu().numpy() for t in (acq_o, mu, sd, kmax))
    key = key.cpu().numpy().view(np.uint64)
    bad = key > _order_keys(exact)
    assert not bad.any(), f"{bad.sum()} bound keys above the exact key, e.g. row {np.flatnonzero(bad)[0]}"
    y_max = float(np.max(y))
    expect0 = never_prune(kind, mu, np.zeros(m), y_max, 0.01)
    assert np.array_equal(key == 0, expect0), (np.sum(key == 0), np.sum(expect0))
    assert np.allclose(kmax, np.max(np.abs(gp.kernel_(x, X)), axis=1), rtol=1e-12, atol=1e-300)
    kdiag = gp.kernel_(X[:1])[0, 0] + 1e-6
    prior = gp.kernel_.diag(x[:1])[0]
    live = sd > 0
    colsq = prior - (sd[live] / float(gp._y_train_std)) ** 2
    overshoot = float(np.max((kmax[live] ** 2 / kdiag - colsq) / prior))
    print(f"{case} {kind}: max (max K*^2/Kii - computed sum V^2) / prior = {overshoot:.3e}")
    assert overshoot <= VAR_EPS
