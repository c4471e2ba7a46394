"""The fp32 Gram bound pass of selection pruning (predict_bound_gram_kernel<COV, true>, DESIGN.md 4.9).

The pass takes r~^2 from the same fp64 DMMA Gram product as the fp64 Gram pass and evaluates the covariance in fp32
(rsqrtf, exp2f and FMA-pipe arithmetic), with a margin derived per row as u k~ (R + Q z~) (u = 2^-24) plus the Gram
distance term.  Checked here:
  * the device covariance (b200bo_cov_f32_dev), exhaustively over every fp32 argument from 0 up past the clamp, against
    an fp64 evaluation of the formula, within the per-row error the margin assumes;
  * on every kernel-matrix case with a bounded Lip, on the ill-conditioned fixtures (the fp32 pass forced, and the pass
    B200BO_PRUNE_BOUND=auto picks) and at C3: keys <= exact keys, mu_lo <= mu <= mu_hi, kmax_lb <= the direct max;
  * at C3 the fp32 keys let through no more than 3 % more candidates than the fp64 Gram keys;
  * auto picks the fp64 pass on illbig_b_rbf_long (A1 = 1.1e10) and the fp32 pass at C3.
"""
import ctypes as C

import numpy as np
import pytest

import kernel_matrix_cases as KM
from test_gpu_prune_gram import KINDS, U, _code, _order_keys

pytestmark = pytest.mark.gpu

# (family, nu) codes of include/b200bo.h per covariance code, and CovF32's clamp, R and Q (predict16.cuh)
COVS = {"m15": (1, 2300.0, 24.0, 8.0), "m25": (2, 1400.0, 32.0, 8.0), "rbf": (3, 166.0, 12.0, 4.0)}
U32 = 2.0 ** -24
MU_SUM_R = 6.0  # the part of R for the fp32 mu partial, not for the covariance itself
PASS_F64, PASS_F32 = 1, 2


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED", "B200BO_PRUNE", "B200BO_PRUNE_BOUND"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _family_nu(code):
    from bayesianoptimization_b200 import _lib as B

    return {1: (B.KERNEL_MATERN, B.NU_15), 2: (B.KERNEL_MATERN, B.NU_25), 3: (B.KERNEL_RBF, B.NU_25)}[code]


@pytest.mark.parametrize("cov", sorted(COVS))
def test_cov_f32_exhaustive(bo, cov):
    """Every fp32 r^2 from +0 to twice the clamp: |k~ - k(s)| <= u k~ (R - 6 + Q z~) + 1e-30, s the clamped argument."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    code, r2max, R, Q = COVS[cov]
    fam, nu = _family_nu(code)
    L, s = B.lib(), torch.cuda.current_stream()
    hi = int(np.float32(2 * r2max).view(np.int32))
    chunk = 1 << 26
    k = torch.empty(chunk, dtype=torch.float32, device="cuda")
    z = torch.empty(chunk, dtype=torch.float32, device="cuda")
    worst = 0.0
    for b0 in range(0, hi + 1, chunk):
        n = min(chunk, hi + 1 - b0)
        bits = torch.arange(b0, b0 + n, dtype=torch.int32, device="cuda")
        r2 = bits.view(torch.float32)
        B.check(L.b200bo_cov_f32_dev(fam, nu, r2.data_ptr(), n, k.data_ptr(), z.data_ptr(), s.cuda_stream))
        sc = r2.double().clamp(2.0 ** -100, r2max)
        if code == 3:
            ref = torch.exp(-0.5 * sc)
        else:
            zz = torch.sqrt(sc) * (5.0 ** 0.5 if code == 2 else 3.0 ** 0.5)
            ref = (1.0 + zz + zz * zz / 3.0 if code == 2 else 1.0 + zz) * torch.exp(-zz)
        kd, zd = k[:n].double(), z[:n].double()
        bound = U32 * kd * ((R - MU_SUM_R) + Q * zd) + 1e-30
        err = (kd - ref).abs()
        assert bool(torch.isfinite(kd).all()), cov
        bad = err > bound
        assert not bool(bad.any()), (cov, float(r2[bad.nonzero()[0, 0]]))
        worst = max(worst, float((err / bound).max()))
        del bits, r2, sc, ref, kd, zd, err, bound
    print(f"{cov}: largest error / assumed bound {worst:.3f}")


def _run(bo, acq, x, pass_=PASS_F32):
    """exact values and mu, direct keys and max |k|, keys, (mu_lo, mu_hi) and kmax_lb of the fp32 (or fp64) Gram pass"""
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
    entry = L.b200bo_acq_prune_bound_gram32_dev if pass_ == PASS_F32 else L.b200bo_acq_prune_bound_gram_dev
    B.check(entry(C.byref(acq.spec), xd.data_ptr(), m, key_g.data_ptr(), mu_iv.data_ptr(), kmax_lb.data_ptr(),
                  s.cuda_stream))
    s.synchronize()
    out = {k: t.cpu().numpy() for k, t in dict(exact=acq_o, mu=mu, kmax=kmax, kmax_lb=kmax_lb, mu_iv=mu_iv).items()}
    out["key_d"] = key_d.cpu().numpy().view(np.uint64)
    out["key_g"] = key_g.cpu().numpy().view(np.uint64)
    return out


def _check(bo, name, gp, acq, x, pass_=PASS_F32):
    r = _run(bo, acq, x, pass_)
    y_std, y_mean = float(gp._y_train_std), float(gp._y_train_mean)
    bad = r["key_g"] > _order_keys(r["exact"])
    assert not bad.any(), f"{name}: {bad.sum()} keys above the exact key, e.g. row {np.flatnonzero(bad)[0]}"
    mu_n = (r["mu"] - y_mean) / y_std
    lo, hi = r["mu_iv"][:, 0], r["mu_iv"][:, 1]
    slack = 4 * U * (np.abs(mu_n) + abs(y_mean) / y_std)
    fin = np.isfinite(lo) & np.isfinite(hi)
    assert np.all(lo[fin] <= mu_n[fin] + slack[fin]) and np.all(mu_n[fin] <= hi[fin] + slack[fin]), name
    assert np.all(r["kmax_lb"] <= r["kmax"]), name
    half = 0.5 * (hi - lo)
    print(f"{name}: median dmu {np.median(half[fin]):.3e}, max {np.max(half[fin]):.3e}; "
          f"max |mu~ - mu| / dmu {np.max(np.abs(0.5 * (lo + hi) - mu_n)[fin] / np.maximum(half[fin], 1e-300)):.3e}")
    return r


def _pass(acq):
    import torch

    from bayesianoptimization_b200 import _lib as B

    p = C.c_int()
    B.check(B.lib().b200bo_acq_prune_bound_pass(C.byref(acq.spec), C.byref(p), torch.cuda.current_stream().cuda_stream))
    return p.value


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
    _check(bo, f"{case} {kind}", gp, acq, x)


def _ill_small():
    import test_gpu_illcond as TI

    return [(TI, n) for n in TI.CASES if "m05" not in n]


def _ill_big():
    import test_gpu_illcond_big as TB

    return [(TB, n) for n in TB.CASES if "m05" not in n]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("which", ("f32", "auto"))
def test_illcond_fixtures(bo, which, kind):
    for T, name in _ill_small() + _ill_big():
        r = T.fixture(name)
        gp = T._gp(bo, name)
        acq = T._acq(bo, gp, kind, r)
        X = r["X"]
        x = np.vstack([r["xt"], X[:64], X[:64] + 1e-9,
                       np.random.RandomState(3).uniform(size=(1 << 12, X.shape[1]))])
        p = PASS_F32 if which == "f32" else _pass(acq)
        _check(bo, f"{name} {kind} {which}->{'f32' if p == PASS_F32 else 'f64'}", gp, acq, x, p)


def _c3(bo):
    from sklearn.gaussian_process.kernels import Matern

    rs = np.random.RandomState(0)
    X = rs.uniform(size=(4096, 16))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(4096)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    return X, gp, bo.FusedAcquisition(_code("ei"), gp, xi=0.01, y_max=float(np.max(y)))


def test_c3_tightness(bo):
    """At C3, of 2^18 candidates, the fp32 keys at or below the final 10th key are at most 3 % more than the fp64
    Gram keys'."""
    X, gp, acq = _c3(bo)
    x = np.vstack([np.random.RandomState(1000).uniform(size=((1 << 18) - 128, 16)), X[:64], X[:64] + 1e-9])
    r = _check(bo, "c3 ei f32", gp, acq, x)
    g = _run(bo, acq, x, PASS_F64)
    kth = np.sort(_order_keys(r["exact"]))[9]
    nd, n64, n32 = (int(np.sum(v <= kth)) for v in (r["key_d"], g["key_g"], r["key_g"]))
    print(f"c3: candidates at or below the 10th key: direct {nd}, fp64 Gram {n64}, fp32 Gram {n32}")
    assert n32 <= max(n64 * 1.03, n64 + 1)


def test_auto_choice(bo, monkeypatch):
    import test_gpu_illcond_big as TB

    _, _, acq = _c3(bo)
    assert _pass(acq) == PASS_F32
    r = TB.fixture("b_rbf_long")
    acq_l = TB._acq(bo, TB._gp(bo, "b_rbf_long"), "ei", r)
    assert _pass(acq_l) == PASS_F64
    monkeypatch.setenv("B200BO_PRUNE_BOUND", "f32")
    assert _pass(acq_l) == PASS_F32
    monkeypatch.setenv("B200BO_PRUNE_BOUND", "f64")
    assert _pass(acq) == PASS_F64
