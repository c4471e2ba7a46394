"""Posterior accuracy on ill-conditioned, clustered training sets, against an extended-precision reference.

Late in a Bayesian-optimisation run the registered points cluster around the incumbent and cond(K) climbs towards
1/alpha.  Both fp64 computations of the posterior then carry errors of order cond(K) eps: sklearn's triangular solve
and the device's product with the explicit inverse L^-1 (DESIGN.md 4.1).  So neither is compared with the other here:
both are compared with the same operations at 50 digits (oracle/make_illcond.py, fixtures tests/golden/illcond_*.npz,
which also hold sklearn's fp64 results on the same rows), and the device is held to "no worse than sklearn":

  device error <= max(C * sklearn's error, floor),  C and the floor per metric (C_SK, FLOOR),

plus the north-star bar (1e-5 relative) wherever sklearn itself meets it, plus a per-case bar pinned at about 10x the
largest error measured over the fp64 kernel variants on an H100 80GB HBM3 at a 700 W power limit.

Metrics: mu as |dmu| / (|mu| + s_y); sigma relative, |d sigma| / sigma (every candidate's true sigma^2 is at least
about alpha * prior, tests/test_illcond_cpu.py); UCB as |d ucb| / (|mu| + kappa sigma); EI and PoI relative.  alpha_
is held twice: against the truth K^-1 y, where the fp64 rounding of K alone costs cond(K) eps in any fp64 solve, and
through its residual max |y - K alpha_| / max |y| against the device's own K, evaluated at 50 digits: that is what the
iterative refinement of the device's solve improves.  Every case prints the device's and sklearn's errors (pytest -s).
"""
import ctypes as C
import warnings

import numpy as np
import pytest
from scipy.linalg import lapack

from oracle import make_illcond as MI
from test_gpu_mes import _ENV, VARIANTS

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # north-star bar, fp64
# The device may be at most C_SK times further from the truth than sklearn, or FLOOR away.  The mean, the fit state
# and the LML come from the factor and alpha_ (iteratively refined) and are held to 10x.  sigma and the acquisitions
# come from the product with the explicit inverse: its error is of order |L^-1| |k*| eps where sklearn's triangular
# solve has |L^-1 k*| eps, and near the training points, where sigma^2 = prior - sum V^2 is a small residue, the
# measured gap reaches 25x on sigma and 90x on UCB (DESIGN.md section 2).  That gap is the bar; the per-case pins
# below keep it from growing.
C_SK = dict(mu=10.0, sd=100.0, ucb=100.0, ei=100.0, poi=100.0, L=10.0, alpha=10.0, lml=10.0, grad=10.0, res=2.0)
FLOOR = dict(mu=1e-13, sd=1e-11, ucb=1e-13, ei=1e-10, poi=1e-10, L=1e-13, alpha=1e-12, lml=1e-13, grad=5e-11,
             res=1e-15)

# Per-case bars, pinned at about 10x the error measured on an H100 80GB HBM3 at a 700 W power limit (in the comments):
# PREDICT_BAR on the fp64 predict metrics (max over mu, sigma, UCB, EI, PoI and the seven fp64 variants); FIT_BAR on
# the fit metrics (max over L and alpha_ on the four factorisation paths, the LML and its gradient).
PREDICT_BAR = {
    "c_m05_ard": 1e-7,  # 9.1e-9
    "c_m15_d17": 3.5e-5,  # 3.3e-6
    "c_m25_d2": 2.5e-5,  # 2.3e-6
    "c_m25_d3": 1.2e-6,  # 1.2e-7
    "c_rbf_d6": 2e-7,  # 1.9e-8
    "l_m15_a8": 2e-5,  # 1.8e-6
    "l_m25_ard_d5": 3.5e-6,  # 3.4e-7
    "l_m25_d4": 1.5e-7,  # 1.5e-8
    "l_rbf_a10": 2e-3,  # 1.8e-4 (sigma; sklearn's own error is 1.5e-5: neither meets the 1e-5 bar at alpha = 1e-10)
    "l_rbf_d3": 1.1e-5,  # 1.1e-6
    "t_m25_d2": 1e-7,  # 8.5e-9
}
# RES_BAR on the residual of alpha_ (max over the five factorisation paths), pinned at 2x the measurement: the metric
# is deterministic (every fit-side reduction has a fixed order), and without the refinement step of the solve it
# grows by only 2x to 7x, so a 10x pin could not see the step go.
RES_BAR = {  # measured with refinement | without it (the smallest over the paths)
    "c_m05_ard": 3e-15,  # 1.5e-15 | 3.5e-15
    "c_m15_d17": 3e-13,  # 1.4e-13 | 7.5e-12
    "c_m25_d2": 2e-14,  # 9.4e-15 | 6.2e-13
    "c_m25_d3": 1.1e-13,  # 5.3e-14 | 1.9e-12
    "c_rbf_d6": 5e-12,  # 2.5e-12 | 2.9e-11
    "l_m15_a8": 2.2e-14,  # 1.1e-14 | 3.1e-13
    "l_m25_ard_d5": 8e-13,  # 4.0e-13 | 1.2e-11
    "l_m25_d4": 9e-11,  # 4.5e-11 | 2.1e-10
    "l_rbf_a10": 9.2e-8,  # 4.6e-8 | 1.5e-6
    "l_rbf_d3": 2.4e-8,  # 1.2e-8 | 1.9e-7
    "t_m25_d2": 7e-14,  # 3.5e-14 | 3.2e-13
}
FIT_BAR = {
    "c_m05_ard": 5e-11,  # 4.6e-12
    "c_m15_d17": 1e-8,  # 1.0e-9
    "c_m25_d2": 5e-9,  # 5.3e-10
    "c_m25_d3": 1.5e-8,  # 1.5e-9
    "c_rbf_d6": 8e-9,  # 8.1e-10
    "l_m15_a8": 1e-7,  # 1.0e-8
    "l_m25_ard_d5": 1.5e-8,  # 1.5e-9
    "l_m25_d4": 1.3e-8,  # 1.3e-9
    "l_rbf_a10": 6.5e-5,  # 6.4e-6
    "l_rbf_d3": 1e-6,  # 1.0e-7
    "t_m25_d2": 7.5e-9,  # 7.4e-10
}
# fp32 mode, DESIGN.md section 2: |d sigma^2| <= 1e-3 sigma^2 + 1e-4 prior s_y^2 (prior = const + noise), and the
# acquisitions within 2e-3 where sigma > 0.1 s_y.  Near the training points only the absolute term holds.
BAR32 = 1e-4
RTOL32 = 2e-3

CASES = sorted(c for c in MI.CASES if c != "a_m25_d3")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


_FIX = {}


def fixture(name):
    if name not in _FIX:
        with np.load(MI.fixture_path(name)) as z:
            _FIX[name] = {k: z[k] for k in z.files}
        r = _FIX[name]
        n = len(r["X"])
        L = np.zeros((n, n))
        L[np.tril_indices(n)] = r["L_packed"]
        r["L"] = L
    return _FIX[name]


def _pin(monkeypatch, variant):
    for k in _ENV + ("B200BO_PRUNE",):
        monkeypatch.delenv(k, raising=False)
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)


def _gp(bo, name, precision="fp64"):
    c = MI.CASES[name]
    r = fixture(name)
    return bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                           optimizer=None, precision=precision).fit(r["X"], r["y"])


def _acq(bo, gp, kind, r):
    from bayesianoptimization_b200 import _lib as B

    code = {"ucb": B.ACQ_UCB, "ei": B.ACQ_EI, "poi": B.ACQ_POI}[kind]
    return bo.FusedAcquisition(code, gp, kappa=MI.KAPPA, xi=MI.XI, y_max=float(np.max(r["y"])))


def _errors(r, mu, sd, acq):
    """The metrics of the module docstring for one set of results (mu, sd, {kind: acquisition value})."""
    e = dict(mu=float(np.max(np.abs(mu - r["mu"]) / (np.abs(r["mu"]) + r["y_std"]))),
             sd=float(np.max(np.abs(sd - r["sd"]) / r["sd"])),
             ucb=float(np.max(np.abs(acq["ucb"] - r["acq_ucb"]) / (np.abs(r["mu"]) + MI.KAPPA * r["sd"]))))
    for k in ("ei", "poi"):
        ref = r[f"acq_{k}"]
        rel = np.abs(acq[k] - ref) / np.maximum(np.abs(ref), 1e-300)
        e[k] = float(np.max(np.where(ref > 1e-290, rel, 0.0)))
    return e


def _e32(r, sd, var):
    return float(np.max(np.abs(sd**2 - var) - 1e-3 * var)) / (r["prior"] * r["y_std"] ** 2)


def _check_fp32_acq(r, acq):
    """Where the true sigma > 0.1 s_y: each acquisition within RTOL32 of its value or of the batch's largest value (the
    whole candidate array, as the mode ranks it: an EI of 1e-75 next to one of 1e-3 is compared at the latter's scale)."""
    rows = r["sd"] > 0.1 * r["y_std"]
    print(f"  fp32 acquisition rows: {rows.sum()}")
    if not rows.any():  # long length scales: no candidate is that uncertain
        return
    for k in ("ucb", "ei", "poi"):
        # floor 1e-12: where every EI is ~1e-75 (z ~ -18), z^2 amplifies fp32's sigma error into O(1) relative ones
        scale = max(float(np.max(np.abs(r[f"acq_{k}"]))), 1e-12)
        np.testing.assert_allclose(acq[k][rows], r[f"acq_{k}"][rows], rtol=RTOL32, atol=RTOL32 * scale, err_msg=k)


def _sk_errors(r):
    return _errors(r, r["sk_mu"], r["sk_sd"], {k: r[f"sk_acq_{k}"] for k in ("ucb", "ei", "poi")})


def _fmt(e):
    return " ".join(f"{k} {v:.1e}" for k, v in e.items())


def _hold(dev, sk, keys):
    """device error <= max(C_SK * sklearn's, FLOOR) and the north-star bar where sklearn meets it."""
    for k in keys:
        assert dev[k] <= max(C_SK[k] * sk[k], FLOOR[k]), (k, dev[k], sk[k])
        if sk[k] <= RTOL:
            assert dev[k] <= RTOL, (k, dev[k], sk[k])


# ---------------------------------------------------------------------------------------------------------------
# predict + acquisition through every kernel variant
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", CASES)
def test_predict_and_acquisition_against_truth(bo, monkeypatch, name, variant):
    r = fixture(name)
    fp32 = variant == "fp32"
    gp = _gp(bo, name, "fp32" if fp32 else "fp64")
    _pin(monkeypatch, variant)
    xt = r["xt"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = gp.predict(xt, return_std=True)
    acq = {k: -_acq(bo, gp, k, r)(xt) for k in ("ucb", "ei", "poi")}
    dev, sk = _errors(r, mu, sd, acq), _sk_errors(r)
    print(f"\n{name} {variant} cond {r['cond']:.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    if fp32:
        e32 = _e32(r, sd, r["var"])
        print(f"  fp32 e32 {e32:.1e}")
        assert e32 <= BAR32
        _hold(dev, sk, ("mu",))  # the mean stays fp64
        _check_fp32_acq(r, acq)
        return
    _hold(dev, sk, ("mu", "sd", "ucb", "ei", "poi"))
    if name in PREDICT_BAR:
        assert max(dev[k] for k in ("mu", "sd", "ucb", "ei", "poi")) <= PREDICT_BAR[name]


# ---------------------------------------------------------------------------------------------------------------
# selection: truth's order, pruning on/off bit-equal, bound keys below the exact keys
# ---------------------------------------------------------------------------------------------------------------
def _order_keys(v):
    v = np.where(v == 0.0, 0.0, v)
    u = v.view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    return np.where(np.isnan(v), np.uint64(0xFFFFFFFFFFFFFFFF), key)


@pytest.mark.parametrize("kind", ("ucb", "ei", "poi"))
@pytest.mark.parametrize("name", CASES)
def test_selection_against_truth_and_pruning(bo, monkeypatch, name, kind):
    import torch

    from bayesianoptimization_b200 import _lib as B

    r = fixture(name)
    gp = _gp(bo, name)
    f = _acq(bo, gp, kind, r)
    _pin(monkeypatch, "m16n8k4")
    ref = -r[f"acq_{kind}"]
    idx, val, top = f.argmin_topk(r["xt"], 10)
    # near-ties: two candidates may trade places when their true values are closer than the case's pinned bar
    want = [int(np.argmin(ref))] + list(np.argsort(ref, kind="stable")[:10])
    got = [int(idx)] + [int(t) for t in top]
    for g, w in zip(got, want):
        if g != w:
            tol = 2 * PREDICT_BAR[name] * max(abs(ref[g]), abs(ref[w]))
            assert abs(ref[g] - ref[w]) <= tol, (g, w, ref[g], ref[w], tol)
    # pruning on / off: bit-equal records, on the case's rows plus enough uniform rows for the pruned path to skip
    x = np.vstack([r["xt"], np.random.RandomState(3).uniform(size=(1 << 14, r["xt"].shape[1]))])
    out = []
    for p in ("0", "1"):
        monkeypatch.setenv("B200BO_PRUNE", p)
        i, v, t = f.argmin_topk(x, 10)
        out.append((i, np.float64(v).view(np.int64), list(t)))
    assert out[0] == out[1]
    # bound keys at or below the keys of the exact values
    m = x.shape[0]
    xd = torch.from_numpy(x).cuda()
    acq_o = torch.empty(m, dtype=torch.float64, device="cuda")
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, acq_o.data_ptr(), None, None, 0, None, 0,
                                  s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), None, s.cuda_stream))
    s.synchronize()
    bad = key.cpu().numpy().view(np.uint64) > _order_keys(acq_o.cpu().numpy())
    assert not bad.any(), f"{bad.sum()} bound keys above the exact key, e.g. row {np.flatnonzero(bad)[0]}"


# ---------------------------------------------------------------------------------------------------------------
# fit side: K, L, alpha_ through every factorisation path; LML and gradient
# ---------------------------------------------------------------------------------------------------------------
FIT_PATHS = {
    "lookahead": {},
    "serial_gemm64": {"B200BO_POTRF": "serial", "B200BO_GEMM": "64"},
    "gemm64": {"B200BO_GEMM": "64"},
    "graph0": {"B200BO_GRAPH": "0"},
    "graph1": {"B200BO_GRAPH": "1"},
}
_K = {}


def _k_truth(name):
    if name not in _K:
        r = fixture(name)
        _K[name] = np.array([[float(v) for v in row] for row in MI.kernel_matrix_mp(MI.CASES[name], r["X"])])
    return _K[name]


def _sk_K(name):
    c, r = MI.CASES[name], fixture(name)
    K = MI.sk_kernel(c)(r["X"])
    K[np.diag_indices_from(K)] += c["alpha"]
    return K


def _sk_L(name):
    from sklearn.gaussian_process import GaussianProcessRegressor

    c, r = MI.CASES[name], fixture(name)
    return GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                    optimizer=None).fit(r["X"], r["y"]).L_


def _residual(r, K, a):
    """max |y_n - K a| / max |y_n| at 50 digits, y_n the normalised targets, K the fp64 matrix the solve was given."""
    import mpmath as mp

    mp.mp.dps = MI.DPS
    y = r["y"]
    yn = (y - np.mean(y)) / np.std(y)
    am = [mp.mpf(float(v)) for v in a]
    res = max(abs(mp.mpf(float(yn[i])) - mp.fdot([mp.mpf(float(v)) for v in K[i]], am)) for i in range(len(yn)))
    return float(res) / float(np.max(np.abs(yn)))


def _fit_errors(r, L, a):
    return dict(L=float(np.max(np.abs(L - r["L"])) / np.max(np.abs(r["L"]))),
                alpha=float(np.max(np.abs(a - r["alpha_"])) / np.max(np.abs(r["alpha_"]))))


@pytest.mark.parametrize("path", list(FIT_PATHS))
@pytest.mark.parametrize("name", CASES)
def test_fit_state_against_truth(bo, monkeypatch, name, path):
    """np <= 128 (l_m15_a8, l_rbf_a10, c_m25_d3, t_m25_d2) factorises without look-ahead on every path."""
    from bayesianoptimization_b200 import _lib as B

    for k in ("B200BO_POTRF", "B200BO_GEMM", "B200BO_GRAPH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in FIT_PATHS[path].items():
        monkeypatch.setenv(k, v)
    r = fixture(name)
    n = len(r["X"])
    gp = _gp(bo, name)
    K = np.empty((n, n))
    B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_K, B.as_dp(K), n * n))
    Kt = _k_truth(name)
    e_K = float(np.max(np.abs(K - Kt) / np.abs(Kt)))
    dev = _fit_errors(r, gp.L_, gp.alpha_)
    sk = _fit_errors(r, _sk_L(name), r["sk_alpha_"])
    dev["res"] = _residual(r, K, gp.alpha_)
    sk["res"] = _residual(r, _sk_K(name), r["sk_alpha_"])
    print(f"\n{name} {path} cond {r['cond']:.1e}: K {e_K:.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    assert e_K <= 4e-16 * (1 + 2 * np.sqrt(MI.CASES[name]["d"]))  # a few ulp per entry: K is well-conditioned data
    _hold(dev, sk, ("L", "alpha", "res"))
    if name in FIT_BAR:
        assert max(dev["L"], dev["alpha"]) <= FIT_BAR[name]
    if name in RES_BAR:
        assert dev["res"] <= RES_BAR[name]


@pytest.mark.parametrize("name", CASES)
def test_lml_and_gradient_against_truth(bo, name):
    """lml_grad_tile_kernel (d <= 16) and lml_grad_kernel (c_m15_d17) at the case's theta."""
    r = fixture(name)
    gp = _gp(bo, name)
    theta = MI.sk_kernel(MI.CASES[name]).theta
    lml, grad = gp.log_marginal_likelihood(theta, eval_gradient=True)
    gs = max(float(np.max(np.abs(r["lml_grad"]))), 1.0)
    dev = dict(lml=abs(lml - r["lml"]) / abs(r["lml"]), grad=float(np.max(np.abs(grad - r["lml_grad"]))) / gs)
    sk = dict(lml=abs(r["sk_lml"] - r["lml"]) / abs(r["lml"]),
              grad=float(np.max(np.abs(r["sk_lml_grad"] - r["lml_grad"]))) / gs)
    print(f"\n{name} lml cond {r['cond']:.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    assert grad.shape == r["lml_grad"].shape
    _hold(dev, sk, ("lml", "grad"))
    if name in FIT_BAR:
        assert max(dev.values()) <= FIT_BAR[name]


@pytest.mark.parametrize("potrf", ("lookahead", "serial"))
@pytest.mark.parametrize("row", (131, 250))
def test_not_pd_pivot_equals_lapack(bo, monkeypatch, potrf, row):
    """A copy of an earlier training point at `row` with a negative diagonal jitter: the leading minor of that row is
    the first one that is not positive, inside a later 64-row block.  The device reports the same 1-based pivot as
    LAPACK's dpotrf."""
    from bayesianoptimization_b200 import _lib as B

    monkeypatch.delenv("B200BO_POTRF", raising=False)
    if potrf == "serial":
        monkeypatch.setenv("B200BO_POTRF", "serial")
    rs = np.random.RandomState(row)
    n, d, ls, jitter = 300, 3, 0.05, -1e-3
    X = rs.uniform(size=(n, d))
    X[row] = X[17]
    y = np.sin(X.sum(1))
    from sklearn.gaussian_process.kernels import Matern

    K = Matern(length_scale=ls, nu=2.5)(X)
    K[np.diag_indices(n)] += jitter
    info = lapack.dpotrf(K, lower=1)[1]
    assert info == row + 1  # the construction puts the first failing pivot where intended
    L = B.lib()
    h = C.c_void_p()
    assert L.b200bo_gp_create(C.byref(h), 0) == 0
    try:
        lsv = np.array([ls])
        spec = B.KernelSpec(B.KERNEL_MATERN, B.NU_25, 1, 0, 1.0, B.as_dp(lsv))
        Xc, yc = B.c_f64(X), B.c_f64(y)
        dinfo = C.c_int64()
        rc = L.b200bo_gp_fit(h, B.as_dp(Xc), B.as_dp(yc), n, d, C.byref(spec), jitter, 0, C.byref(dinfo))
        assert rc == B.ERR_NOT_PD
        assert dinfo.value == info
    finally:
        L.b200bo_gp_destroy(h)


# ---------------------------------------------------------------------------------------------------------------
# append path: 60 -> 128 on a clustered set, then tiled predict
# ---------------------------------------------------------------------------------------------------------------
APPEND_BAR = dict(fit=2e-8, predict=6e-7)  # pinned like PREDICT_BAR / FIT_BAR: measured 1.9e-9 and 5.9e-8


@pytest.mark.parametrize("precision", ("fp64", "fp32"))
def test_append_clustered_to_capacity_then_tiled_predict(bo, monkeypatch, precision):
    name = "a_m25_d3"
    c = MI.CASES[name]
    r = fixture(name)
    X, y = r["X"], r["y"]
    gp = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None,
                                         precision=precision)
    gp.fit(X[:60], y[:60])
    calls = []
    try_incremental = gp._try_incremental

    def spy(*a, **kw):
        ok = try_incremental(*a, **kw)
        calls.append(ok)
        return ok

    monkeypatch.setattr(gp, "_try_incremental", spy)
    for n in range(61, 129):
        gp.fit(X[:n], y[:n])
    assert calls == [True] * 68
    dev = _fit_errors(r, gp.L_, gp.alpha_)
    sk = _fit_errors(r, _sk_L(name), r["sk_alpha_"])
    _hold(dev, sk, ("L", "alpha"))
    _pin(monkeypatch, "m16n8k4")
    reps = 5  # 800 rows: several 128-candidate tiles
    xt = np.tile(r["xt"], (reps, 1))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = gp.predict(xt, return_std=True)
    acq = {k: -_acq(bo, gp, k, r)(xt) for k in ("ucb", "ei", "poi")}
    rr = {k: np.tile(v, reps) if isinstance(v, np.ndarray) and v.shape == r["mu"].shape else v for k, v in r.items()}
    e, es = _errors(rr, mu, sd, acq), _sk_errors(r)
    print(f"\nappend {precision}: {_fmt(dev)} | {_fmt(e)}\n  sklearn {_fmt(sk)} | {_fmt(es)}")
    assert max(dev.values()) <= APPEND_BAR["fit"]
    if precision == "fp32":
        e32 = _e32(r, sd, rr["var"])
        print(f"  fp32 e32 {e32:.1e}")
        assert e32 <= BAR32
        _hold(e, es, ("mu",))
    else:
        _hold(e, es, ("mu", "sd", "ucb", "ei", "poi"))
        assert max(e[k] for k in ("mu", "sd", "ucb", "ei", "poi")) <= APPEND_BAR["predict"]


# ---------------------------------------------------------------------------------------------------------------
# covariance primitives (sqrt_pos, exp_neg through cov_eval) over the whole range of the scaled squared distance
# ---------------------------------------------------------------------------------------------------------------
R2 = np.array([0.0, 1e-300, 1e-40, 1e-31, 1e-30, 3e-29, 1e-20, 1e-12, 1e-6, 1e-3, 0.1, 0.5, 1.0, 2.0, 10.0, 100.0,
               699.0, 700.0, 1.4e3, 1.5e3, 1e4, 1e6, 1e10, 1e20, 1e37, 1e38, 3.4e38, 3.5e38, 1e39, 1e100, 1e200,
               1e300])
ULPS = 4  # per unit of exp's argument + 1 (exp amplifies the relative error of its argument by the argument)


@pytest.mark.parametrize("kern", ("m05", "m15", "m25", "rbf"))
def test_covariance_primitives_over_the_range(bo, kern):
    """A one-point GP at the origin with unit length scale: phase A's max |k(x, X_j)| (the d_kmax output of
    b200bo_acq_prune_bound_dev) is the covariance at r^2 = x^2, against sklearn's formula at 50 digits.  Away from the
    clamp regions (r^2 < 1e-30 for the distance, exp arguments above 700) the error is within ULPS ulp per unit of
    exp's argument; inside them within the documented absolute bounds."""
    import mpmath as mp
    import torch

    from bayesianoptimization_b200 import _lib as B

    from sklearn.gaussian_process.kernels import RBF, Matern

    k = RBF(1.0) if kern == "rbf" else Matern(1.0, nu={"m05": 0.5, "m15": 1.5, "m25": 2.5}[kern])
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=1e-6, normalize_y=False, optimizer=None)
    gp.fit(np.zeros((1, 1)), np.zeros(1))
    x = np.sqrt(R2)
    r2 = x * x  # the device's r^2 = fma(x - 0, x - 0, 0)
    f = _acq(bo, gp, "ei", dict(y=np.zeros(1)))
    m = len(x)
    xd = torch.from_numpy(x[:, None].copy()).cuda()
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    kmax = torch.empty(m, dtype=torch.float64, device="cuda")
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), kmax.data_ptr(),
                                               s.cuda_stream))
    s.synchronize()
    got = kmax.cpu().numpy()
    mp.mp.dps = 50
    want = np.array([float(MI._cov(kern, mp.mpf(float(v)))) for v in r2])
    karg = r2 / 2 if kern == "rbf" else np.sqrt({"m05": 1.0, "m15": 3.0, "m25": 5.0}[kern] * r2)
    clamp_lo = (r2 < 1e-30) & (kern != "rbf")
    clamp_hi = karg > 700.0
    eps = np.finfo(float).eps
    err = np.abs(got - want)
    for v, g, w, e, a in zip(r2, got, want, err, karg):
        print(f"{kern} r2 {v:.3e}: device {g:.17e} exact {w:.17e} ({e / max(w * eps, 1e-300):.1f} ulp, arg {a:.1e})")
    ok = ~(clamp_lo | clamp_hi)
    assert np.all(err[ok] <= ULPS * (1.0 + karg[ok]) * eps * want[ok]), (R2[ok], err[ok] / (want[ok] * eps))
    assert np.all(err[clamp_lo] <= 1e-15)  # sqrt_pos: arguments below 1e-30 are taken as 1e-30
    assert np.all(got[clamp_hi] <= 1e-260) and np.all(got >= 0.0)  # exp_neg's clamp: the limit 0
    assert np.all(np.isfinite(got))
