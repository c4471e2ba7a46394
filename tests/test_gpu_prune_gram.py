"""The Gram bound pass of selection pruning (predict_bound_gram_kernel, DESIGN.md 4.9) against the exact path.

The pass computes the candidate-to-training distances on the fp64 tensor pipe in the Gram form and keys every
candidate from an interval [mu_lo, mu_hi] of its mean and a lower bound of max |k*_i|.  On every covariance with a
bounded dk/d(r^2) (all but Matern-0.5), at C3 and on the ill-conditioned fixtures, with training copies and
near-duplicates in the batch (b200bo_acq_prune_bound_gram_dev):
  * its key is never above the key of the exact value (b200bo_acq_eval_dev);
  * mu_lo <= mu <= mu_hi with the exact path's mu;
  * kmax_lb <= the direct pass's max |k*_i| (b200bo_acq_prune_bound_dev);
  * the distance between the Gram mu and the exact mu, as a share of the interval half width, is printed;
  * at C3 it prunes within 1 % as many candidates as the direct pass.
"""
import ctypes as C

import numpy as np
import pytest

import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

KINDS = ("ei", "ucb", "poi")
U = 2.0 ** -53


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED", "B200BO_PRUNE"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _order_keys(v):
    v = np.where(v == 0.0, 0.0, v)
    u = v.view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    return np.where(np.isnan(v), np.uint64(0xFFFFFFFFFFFFFFFF), key)


def _run(acq, x):
    """exact values and mu, direct keys and max |k|, Gram keys, (mu_lo, mu_hi) and kmax_lb"""
    import torch

    from bayesianoptimization_b200 import _lib as B

    m = x.shape[0]
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device="cuda")  # noqa: E731
    acq_o, mu, sd, kmax, kmax_lb, mu_iv = f64(m), f64(m), f64(m), f64(m), f64(m), f64((m, 2))
    key_d = torch.empty(m, dtype=torch.int64, device="cuda")
    key_g = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), m, acq_o.data_ptr(), mu.data_ptr(), sd.data_ptr(),
                                  0, None, 0, s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(acq.spec), xd.data_ptr(), m, key_d.data_ptr(), kmax.data_ptr(),
                                         s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_gram_dev(C.byref(acq.spec), xd.data_ptr(), m, key_g.data_ptr(),
                                              mu_iv.data_ptr(), kmax_lb.data_ptr(), s.cuda_stream))
    s.synchronize()
    out = {k: t.cpu().numpy() for k, t in dict(exact=acq_o, mu=mu, kmax=kmax, kmax_lb=kmax_lb, mu_iv=mu_iv).items()}
    out["key_d"] = key_d.cpu().numpy().view(np.uint64)
    out["key_g"] = key_g.cpu().numpy().view(np.uint64)
    return out


def _check(name, gp, acq, x):
    r = _run(acq, x)
    y_std, y_mean = float(gp._y_train_std), float(gp._y_train_mean)
    bad = r["key_g"] > _order_keys(r["exact"])
    assert not bad.any(), f"{name}: {bad.sum()} Gram keys above the exact key, e.g. row {np.flatnonzero(bad)[0]}"
    mu_n = (r["mu"] - y_mean) / y_std  # normalised units, as the interval: compare with a data-unit rounding slack
    lo, hi = r["mu_iv"][:, 0], r["mu_iv"][:, 1]
    slack = 4 * U * (np.abs(mu_n) + abs(y_mean) / y_std)
    fin = np.isfinite(lo) & np.isfinite(hi)
    assert np.all(lo[fin] <= mu_n[fin] + slack[fin]) and np.all(mu_n[fin] <= hi[fin] + slack[fin]), name
    assert np.all(r["kmax_lb"] <= r["kmax"]), name
    half = 0.5 * (hi - lo)
    print(f"{name}: median dmu {np.median(half[fin]):.3e}, max {np.max(half[fin]):.3e}; "
          f"max |mu~ - mu| / dmu {np.max(np.abs(0.5 * (lo + hi) - mu_n)[fin] / np.maximum(half[fin], 1e-300)):.3e}")
    return r


CASES = [(c, kind) for c in sorted(KM.PREDICT) if KM.PREDICT[c]["kern"] != "m05" for kind in KINDS]


@pytest.mark.parametrize("case,kind", CASES)
def test_kernel_matrix_cases(bo, case, kind):
    c = KM.PREDICT[case]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, seed=11)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    acq = bo.FusedAcquisition(_code(kind), gp, kappa=2.576, xi=0.01, y_max=float(np.max(y)))
    x = np.vstack([KM.inputs(c, 4000, d, rs), X[:64], X[:64] + 1e-9])
    _check(f"{case} {kind}", gp, acq, x)


def _code(kind):
    from bayesianoptimization_b200 import _lib as B

    return {"ei": B.ACQ_EI, "ucb": B.ACQ_UCB, "poi": B.ACQ_POI}[kind]


def _ill_cases():
    import test_gpu_illcond as TI

    return TI, [n for n in TI.CASES if "m05" not in n]


@pytest.mark.parametrize("kind", KINDS)
def test_illcond_fixtures(bo, kind):
    TI, names = _ill_cases()
    for name in names:
        r = TI.fixture(name)
        gp = TI._gp(bo, name)
        acq = TI._acq(bo, gp, kind, r)
        X = r["X"]
        x = np.vstack([r["xt"], X[:64], X[:64] + 1e-9,
                       np.random.RandomState(3).uniform(size=(1 << 12, X.shape[1]))])
        _check(f"{name} {kind}", gp, acq, x)


def test_c3_tightness(bo):
    """At C3, the Gram keys prune about as many candidates as the direct keys: of the 2^18 candidates, the count at
    or below the final k-th key is within 1 % of the direct pass's count."""
    from sklearn.gaussian_process.kernels import Matern

    rs = np.random.RandomState(0)
    X = rs.uniform(size=(4096, 16))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(4096)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    acq = bo.FusedAcquisition(_code("ei"), gp, xi=0.01, y_max=float(np.max(y)))
    x = np.vstack([np.random.RandomState(1000).uniform(size=((1 << 18) - 128, 16)), X[:64], X[:64] + 1e-9])
    r = _check("c3 ei", gp, acq, x)
    kth = np.sort(_order_keys(r["exact"]))[9]
    nd, ng = int(np.sum(r["key_d"] <= kth)), int(np.sum(r["key_g"] <= kth))
    print(f"c3: candidates at or below the 10th key: direct {nd}, Gram {ng}")
    assert ng <= max(nd * 1.01, nd + 1)
