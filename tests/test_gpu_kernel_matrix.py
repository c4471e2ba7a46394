"""Every covariance variant through every device kernel, against the live sklearn GaussianProcessRegressor.

The device kernels pick the covariance by family, as a template parameter or a runtime switch: Matern 1/2, 3/2, 5/2,
RBF (and Matern nu=inf, which routes to the RBF code), iso or ARD length scales, an optional ConstantKernel and
WhiteKernel, and the np.round input transform of int parameters.  The case tables (tests/kernel_matrix_cases.py) put
each of them through:

  A. predict + UCB/EI/PoI + argmin/top-10 on six kernel variants (m16n8k4 and m8n8k4 phase B, 8 warps, DFMA, the
     small-batch path, fp32 mode), with candidate coordinates in registers at even and odd d and without (d > 16),
     and N ragged against the 64- and 128-row blocks;
  B. one fused launch over a target and three constraint GPs of different covariances, and the Philox source;
  C. the fit state (K, L, alpha_) and the LML + gradient of the tile kernel (d <= 16) and of lml_grad_kernel (d > 16);
  D. fit() with restarts at d > 16;
  E. predict(return_cov=True) and the incremental (append) fit.

The reference is sklearn itself on the same kernel object (with bayes_opt's wrap_kernel for int columns), so WhiteKernel
and transform semantics come with it.  Every comparison asserts the north-star bar (1e-5 relative in fp64, DESIGN.md
section 2 in fp32) and a per-case bar pinned at about 10x the error measured on an H100; each case prints its measured
errors (pytest -s).

Metrics: mu as |dmu| / (|mu| + s_y); sigma through the variance, |d sigma^2| / (prior s_y^2) with prior = const + noise
(sigma^2 is a difference of O(prior) numbers, and at training inputs it is a cancellation residue of both computations,
so it is compared absolutely there); acquisitions with assert_allclose(rtol=1e-5, atol=1e-14), and pinned per case
on |d acq| / (|acq| + 1e-3).

Selection rule: the argmin and the top-10 equal numpy's on the reference values, except that two candidates may trade
places when their reference values are closer than the case's bar (relative to the values).
"""
import ctypes as C
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
from numpy.testing import assert_allclose
from scipy.stats import norm
from sklearn.gaussian_process import GaussianProcessRegressor

import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # north-star bar, fp64
ALPHA = 1e-6
KAPPA, XI = 2.576, 0.01
N_UNIFORM, N_EDGE = 2952, 16  # uniform rows + 16 training rows + 16 near-duplicates + 16 far-away rows = 3000

VARIANTS = {  # environment of each kernel variant (read per launch)
    "m16n8k4": {"B200BO_SMALL_PATH": "0"},
    "m8n8k4": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_MMA": "884"},
    "warps8": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_WARPS": "8"},
    "dfma": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_IMPL": "dfma"},
    "small": {"B200BO_SMALL_PATH": "1"},
    "fp32": {"B200BO_SMALL_PATH": "0"},
}
_ENV = ("B200BO_SMALL_PATH", "B200BO_PREDICT_MMA", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_IMPL")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(scope="module")
def O():
    from oracle import gp_oracle

    return gp_oracle


def _pin(monkeypatch, variant):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)


def _prior(case):
    return (case.get("const") or 1.0) + (case.get("white") or 0.0)


def _sk(kernel, X, y):
    return GaussianProcessRegressor(kernel=kernel, alpha=ALPHA, normalize_y=True, optimizer=None).fit(X, y)


def _predict_sk(sk, xt):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # "Predicted variances smaller than 0" at training inputs
        return sk.predict(xt, return_std=True)


def _predict_dev(gp, xt):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return gp.predict(xt, return_std=True)


def _candidates(case, X, d, rs):
    """Uniform rows in the box, 16 training rows, 16 rows 1e-7 away from training rows and 16 rows so far away that
    K* underflows through the exp_neg clamp (sigma -> prior, mu -> the mean of y)."""
    uni = KM.inputs(case, N_UNIFORM, d, rs)
    train = X[rs.choice(len(X), N_EDGE, replace=False)]
    near = X[rs.choice(len(X), N_EDGE, replace=False)] + 1e-7 * rs.choice([-1.0, 1.0], size=(N_EDGE, d))
    far = 1e4 * np.max(KM.length_scale(case, d)) * (1.0 + rs.uniform(size=(N_EDGE, d)))
    return np.vstack([uni, train, near, far])


def _ref_acq(mu, sd, y_max):
    from oracle import gp_oracle as O

    return {kind: -O.base_acq(kind, mu, sd, kappa=KAPPA, xi=XI, y_max=y_max) for kind in (O.ACQ_UCB, O.ACQ_EI, O.ACQ_POI)}


def _constraint_prob(mus, sds, lb, ub):
    """R/bayes_opt/constraint.py:200-221 as written: prod_j [norm(mu_j, sd_j).cdf(ub_j) - norm(mu_j, sd_j).cdf(lb_j)],
    an infinite bound contributing 0 or 1; scipy's frozen norm is NaN where sd <= 0."""
    p = np.ones(len(mus[0]))
    with np.errstate(invalid="ignore", divide="ignore"):
        for mu, sd, lo, hi in zip(mus, sds, lb, ub):
            dist = norm(loc=mu, scale=sd)
            p_lo = dist.cdf(lo) if lo != -np.inf else 0.0
            p_hi = dist.cdf(hi) if hi != np.inf else 1.0
            p = p * (p_hi - p_lo)
    return p


def _check_selection(idx, val, top, ys, ref, tol, k=10):
    """Device (argmin, value, top-k) against numpy on the reference values, with the near-tie rule of the module
    docstring."""
    assert val == ys[idx]
    want = [int(np.argmin(ref))] + list(np.argsort(ref, kind="stable")[:k])
    got = [int(idx)] + [int(t) for t in top]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if g != w:
            assert abs(ref[g] - ref[w]) <= tol, (g, w, ref[g], ref[w], tol)


def _acq_err(ys, ref):
    """Acquisition error pinned per case: |d acq| / (|acq| + 1e-3).  The floor keeps values near zero (UCB crossing
    zero, EI and PoI far from the incumbent) from turning round-off into large relative numbers."""
    return float(np.max(np.abs(ys - ref) / (np.abs(ref) + 1e-3)))


def _check_fp32(idx, val, ys, ref):
    """fp32 mode, on rows where every GP's sigma > 0.1 s_y: the acquisition within 2e-3 of each value or of the
    array's largest value (DESIGN.md section 2: 2e-3 on the acquisition, twice the 1e-3 on sigma^2), and the selected
    candidate (near-)optimal under the fp64 objective."""
    scale = float(np.max(np.abs(ref)))
    assert_allclose(ys, ref, rtol=2e-3, atol=2e-3 * scale)
    assert val == ys[idx]
    assert ref[idx] <= ref.min() + 2e-3 * scale


class _Cache:
    """sklearn results and fitted device GPs per case, shared by every variant of a case."""

    def __init__(self, bo):
        self.bo = bo
        self.refs, self.gps = {}, {}

    def predict_case(self, cid):
        if cid not in self.refs:
            c = KM.PREDICT[cid]
            n, d = c["n"], c["d"]
            X, y, rs = KM.problem(c, n, d, 100 + sorted(KM.PREDICT).index(cid))
            xt = _candidates(c, X, d, rs)
            k = KM.kernel(c, d)
            sk = _sk(k, X, y)
            mu, sd = _predict_sk(sk, xt)
            y_max = float(y.max())
            self.refs[cid] = SimpleNamespace(X=X, y=y, xt=xt, kernel=k, sk=sk, mu=mu, sd=sd, y_max=y_max,
                                             s_y=float(sk._y_train_std), prior=_prior(c), acq=_ref_acq(mu, sd, y_max))
        return self.refs[cid]

    def predict_gp(self, cid, precision):
        key = (cid, precision)
        if key not in self.gps:
            r = self.predict_case(cid)
            self.gps[key] = self.bo.B200GaussianProcessRegressor(
                kernel=r.kernel, alpha=ALPHA, normalize_y=True, optimizer=None, precision=precision).fit(r.X, r.y)
        return self.gps[key]

    def constrained_case(self, cid):
        key = ("B", cid)
        if key not in self.refs:
            c = KM.CONSTRAINED[cid]
            n, d = c["n"], c["d"]
            X, y, rs = KM.problem(KM.CONSTRAINED_TARGET, n, d, 200 + sorted(KM.CONSTRAINED).index(cid))
            s = X.sum(1) / np.sqrt(d)
            cv = np.column_stack([np.cos(2 * s), np.sin(3 * s) + 0.3 * X[:, 0], np.cos(s + X[:, 1])])
            xt = _candidates(KM.CONSTRAINED_TARGET, X, d, rs)
            kernels = [KM.kernel(KM.CONSTRAINED_TARGET, d)] + [KM.kernel(spec, d) for spec, _, _ in KM.CONSTRAINTS]
            targets = [y] + [cv[:, j] for j in range(cv.shape[1])]
            sks = [_sk(k, X, t) for k, t in zip(kernels, targets)]
            preds = [_predict_sk(sk, xt) for sk in sks]
            # rows where no GP's sigma is a cancellation residue (the fp32 mode is compared there)
            big = np.all([sd > 0.1 * sk._y_train_std for sk, (_, sd) in zip(sks, preds)], axis=0)
            lb = [lo for _, lo, _ in KM.CONSTRAINTS]
            ub = [hi for _, _, hi in KM.CONSTRAINTS]
            p = _constraint_prob([m for m, _ in preds[1:]], [s_ for _, s_ in preds[1:]], lb, ub)
            y_max = float(y.max())
            acq = _ref_acq(preds[0][0], preds[0][1], y_max)
            self.refs[key] = SimpleNamespace(X=X, y=y, cv=cv, xt=xt, kernels=kernels, lb=lb, ub=ub, y_max=y_max,
                                             s_y=float(np.std(y)), big=big, p=p, acq=acq)
        return self.refs[key]


@pytest.fixture(scope="module")
def cases(bo):
    return _Cache(bo)


def _acq_dev(bo, kind, gp, xt, y_max, constraint=None):
    f = bo.FusedAcquisition(kind, gp, constraint, kappa=KAPPA, xi=XI, y_max=y_max)
    return f, f(xt)


# ---------------------------------------------------------------------------------------------------------------
# A. predict + acquisition matrix
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_predict_and_acquisition_matrix(bo, O, cases, monkeypatch, cid, variant):
    c = KM.PREDICT[cid]
    r = cases.predict_case(cid)
    fp32 = variant == "fp32"
    gp = cases.predict_gp(cid, "fp32" if fp32 else "fp64")
    _pin(monkeypatch, variant)
    mu, sd = _predict_dev(gp, r.xt)
    e_mu = float(np.max(np.abs(mu - r.mu) / (np.abs(r.mu) + r.s_y)))
    e_var = float(np.max(np.abs(sd**2 - r.sd**2)) / (r.prior * r.s_y**2))
    rows = r.sd > 0.1 * r.s_y if fp32 else np.ones(len(r.xt), dtype=bool)
    errs, sel = {}, {}
    for kind in (O.ACQ_UCB, O.ACQ_EI, O.ACQ_POI):
        f, ys = _acq_dev(bo, kind, gp, r.xt[rows], r.y_max)
        ref = r.acq[kind][rows]
        errs[kind] = _acq_err(ys, ref)
        sel[kind] = (ys, ref, f.argmin_topk(r.xt[rows], 10))
    e_acq = max(errs.values())
    print(f"A {cid} {variant}: mu {e_mu:.1e} var {e_var:.1e} ucb {errs[O.ACQ_UCB]:.1e} ei {errs[O.ACQ_EI]:.1e} "
          f"poi {errs[O.ACQ_POI]:.1e}")
    assert_allclose(mu, r.mu, rtol=RTOL, atol=RTOL * r.s_y)  # the mean stays fp64 in every mode
    assert e_mu <= c["bar"]
    if fp32:
        # DESIGN.md section 2: |d sigma^2| <= 1e-3 sigma^2 + 1e-4 s_y^2
        assert np.all(np.abs(sd**2 - r.sd**2) <= 1e-3 * r.sd**2 + 1e-4 * r.s_y**2)
        assert e_var <= c["bar32"]
        for ys, ref, (idx, val, top) in sel.values():
            _check_fp32(idx, val, ys, ref)
        return
    assert e_var <= RTOL and e_var <= c["bar"]
    assert e_acq <= c["bar_acq"]
    for ys, ref, (idx, val, top) in sel.values():
        assert_allclose(ys, ref, rtol=RTOL, atol=1e-14)
        _check_selection(idx, val, top, ys, ref, c["bar"] * max(float(np.max(np.abs(ref))), 1e-14))


# ---------------------------------------------------------------------------------------------------------------
# B. heterogeneous constraint GPs in one launch
# ---------------------------------------------------------------------------------------------------------------
def _constraint_model(bo, r, precision):
    cm = bo.ConstraintModel(None, np.array(r.lb), np.array(r.ub))
    for m, k in zip(cm.model, r.kernels[1:]):
        m.set_params(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None, precision=precision)
    cm.fit(r.X, r.cv)
    return cm


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("cid", sorted(KM.CONSTRAINED))
def test_heterogeneous_constraints_one_launch(bo, O, cases, monkeypatch, cid, variant):
    c = KM.CONSTRAINED[cid]
    r = cases.constrained_case(cid)
    precision = "fp32" if variant == "fp32" else "fp64"
    gp = bo.B200GaussianProcessRegressor(kernel=r.kernels[0], alpha=ALPHA, normalize_y=True, optimizer=None,
                                         precision=precision).fit(r.X, r.y)
    cm = _constraint_model(bo, r, precision)
    _pin(monkeypatch, variant)
    fp32 = variant == "fp32"
    rows = r.big if fp32 else np.ones(len(r.xt), dtype=bool)
    errs = {}
    for kind in (O.ACQ_EI, O.ACQ_POI):
        f, ys = _acq_dev(bo, kind, gp, r.xt[rows], r.y_max, cm)
        ref = (r.acq[kind] * r.p)[rows]
        errs[kind] = _acq_err(ys, ref)
        idx, val, top = f.argmin_topk(r.xt[rows], 10)
        if fp32:
            _check_fp32(idx, val, ys, ref)
        else:
            assert_allclose(ys, ref, rtol=RTOL, atol=1e-14)
            _check_selection(idx, val, top, ys, ref, c["bar"] * max(float(np.max(np.abs(ref))), 1e-14))
    print(f"B {cid} {variant}: ei {errs[O.ACQ_EI]:.1e} poi {errs[O.ACQ_POI]:.1e}")
    if not fp32:
        assert max(errs.values()) <= c["bar"]


@pytest.mark.parametrize("cid", sorted(KM.CONSTRAINED))
def test_heterogeneous_constraints_philox_equals_host_rows(bo, O, cases, cid):
    """argmin_topk_philox (rows generated inside the kernel) == argmin_topk on the host regeneration of the same rows,
    with the four GPs of mixed covariances in the launch."""
    r = cases.constrained_case(cid)
    d = r.X.shape[1]
    gp = bo.B200GaussianProcessRegressor(kernel=r.kernels[0], alpha=ALPHA, normalize_y=True, optimizer=None).fit(r.X, r.y)
    cm = _constraint_model(bo, r, "fp64")
    f = bo.FusedAcquisition(O.ACQ_EI, gp, cm, xi=XI, y_max=r.y_max)
    m, k, seed, base = 30_000, 7, 99, 1_000_000
    bounds = np.column_stack([np.zeros(d), np.ones(d)])
    bounds[0] = (0.25, 0.75)
    idx, val, bx, top, tx = f.argmin_topk_philox(seed, bounds, m, k, index_base=base)
    rows = O.philox_uniform(seed, base + np.arange(m), d, bounds[:, 0], bounds[:, 1])
    hi, hv, htop = f.argmin_topk(rows, k)
    assert idx == base + hi and val == hv and list(top) == list(base + htop)
    assert np.array_equal(bx, rows[hi]) and np.array_equal(tx, rows[htop])


# ---------------------------------------------------------------------------------------------------------------
# C. fit state, LML and gradient
# ---------------------------------------------------------------------------------------------------------------
def _theta_offset(p):
    """A fixed offset from the case's theta, so that the gradient is not evaluated at a stationary point."""
    return 0.25 * np.sin(1.7 * np.arange(p) + 0.4)


@pytest.mark.parametrize("cid", sorted(KM.GRADIENT))
def test_fit_state_lml_and_gradient(bo, cid):
    from bayesianoptimization_b200 import _lib as B

    c = KM.GRADIENT[cid]
    n, d = c["n"], c["d"]
    X, y, _ = KM.problem(c, n, d, 300 + sorted(KM.GRADIENT).index(cid))
    k = KM.kernel(c, d)
    sk = _sk(k, X, y)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None).fit(X, y)
    K = np.empty((n, n))
    B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_K, B.as_dp(K), n * n))
    Kref = sk.kernel_(X)
    Kref[np.diag_indices(n)] += ALPHA
    assert_allclose(K, Kref, rtol=1e-12, atol=1e-15)
    assert_allclose(gp.L_, sk.L_, rtol=1e-8, atol=1e-12)
    assert_allclose(gp.alpha_, sk.alpha_, rtol=1e-6, atol=1e-9 * float(np.max(np.abs(sk.alpha_))))
    theta = k.theta + _theta_offset(k.theta.size)
    l1, g1 = gp.log_marginal_likelihood(theta, eval_gradient=True)
    l0, g0 = sk.log_marginal_likelihood(theta, eval_gradient=True)
    e_l = abs(l1 - l0) / abs(l0)
    e_g = float(np.max(np.abs(g1 - g0)) / max(float(np.max(np.abs(g0))), 1.0))
    print(f"C {cid} ({KM.grad_class(d)}, {k.theta.size} thetas): lml {e_l:.1e} grad {e_g:.1e}")
    assert g1.shape == g0.shape
    assert l1 == pytest.approx(l0, rel=1e-8)
    assert_allclose(g1, g0, rtol=1e-5, atol=1e-6)
    assert max(e_l, e_g) <= c["bar"]


# ---------------------------------------------------------------------------------------------------------------
# D. fit() with restarts at d > 16
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", sorted(KM.FIT))
def test_fit_with_restarts_above_tile_dimension(bo, cid):
    c = KM.FIT[cid]
    n, d = c["n"], c["d"]
    X, y, _ = KM.problem(c, n, d, 400 + sorted(KM.FIT).index(cid))
    k = KM.kernel(c, d)
    r1, r0 = np.random.RandomState(4), np.random.RandomState(4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True,
                                             n_restarts_optimizer=c["restarts"], random_state=r1).fit(X, y)
        sk = GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, n_restarts_optimizer=c["restarts"],
                                      random_state=r0).fit(X, y)
    s1, s0 = r1.get_state(), r0.get_state()
    assert np.array_equal(s1[1], s0[1]) and s1[2:] == s0[2:]
    l_sk = sk.log_marginal_likelihood_value_
    l_at = gp.log_marginal_likelihood(sk.kernel_.theta)
    l_dev = gp.log_marginal_likelihood_value_
    print(f"D {cid}: lml at sklearn theta* {abs(l_at - l_sk) / abs(l_sk):.1e}, own optimum - sklearn's "
          f"{(l_dev - l_sk) / abs(l_sk):+.1e} (relative)")
    assert l_at == pytest.approx(l_sk, rel=1e-9)
    assert l_dev >= l_sk - 1e-6 * abs(l_sk)
    if c["compare_theta"]:
        assert_allclose(gp.kernel_.theta, sk.kernel_.theta, rtol=0, atol=5e-3)


# ---------------------------------------------------------------------------------------------------------------
# E. predict(return_cov=True) and the incremental fit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", KM.RETURN_COV)
def test_return_cov_matrix(cases, cid):
    r = cases.predict_case(cid)
    gp = cases.predict_gp(cid, "fp64")
    m = KM.RETURN_COV_M
    # uniform rows plus the training rows and their near-duplicates (where the covariance is a cancellation residue)
    xt = np.vstack([r.xt[:m - 2 * N_EDGE], r.xt[N_UNIFORM:N_UNIFORM + 2 * N_EDGE]])
    mu0, c0 = r.sk.predict(xt, return_cov=True)
    mu, cv = gp.predict(xt, return_cov=True)
    assert cv.shape == (m, m)
    e_mu = float(np.max(np.abs(mu - mu0) / (np.abs(mu0) + r.s_y)))
    e_cov = float(np.max(np.abs(cv - c0)) / (r.prior * r.s_y**2))
    print(f"E {cid} return_cov: mu {e_mu:.1e} cov {e_cov:.1e}")
    assert e_mu <= RTOL and e_cov <= RTOL
    assert max(e_mu, e_cov) <= KM.PREDICT[cid]["bar"]


@pytest.mark.parametrize("cid", sorted(KM.APPEND))
def test_incremental_append_matrix(bo, monkeypatch, cid):
    """Fixed theta: fitting X[:n] after X[:120] appends one factor row per point (b200bo_gp_append: K row through
    append_krow_kernel, pivot const + noise + alpha - |l|^2) and must equal a from-scratch sklearn fit.  Every step must
    take the append path: no full device fit is made, and the launches are those of one appended row times the rows
    appended (a full fit at np = 128 launches about as many kernels as one or two appended rows, so a bound on the count
    alone could not tell the paths apart)."""
    c = KM.APPEND[cid]
    d = c["d"]
    X, y, rs = KM.problem(c, KM.APPEND_SIZES[-1], d, 500 + sorted(KM.APPEND).index(cid))
    xt = KM.inputs(c, 64, d, rs)
    k = KM.kernel(c, d)
    prior = _prior(c)
    gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=ALPHA, normalize_y=True, optimizer=None)
    gp.fit(X[:KM.APPEND_BASE], y[:KM.APPEND_BASE])
    calls = {"append": [], "full": 0}
    try_incremental, device_fit = gp._try_incremental, gp._device_fit

    def spy_incremental(*a, **kw):
        ok = try_incremental(*a, **kw)
        calls["append"].append(ok)
        return ok

    def spy_full(*a, **kw):
        calls["full"] += 1
        return device_fit(*a, **kw)

    monkeypatch.setattr(gp, "_try_incremental", spy_incremental)
    monkeypatch.setattr(gp, "_device_fit", spy_full)
    launches = bo._lib.lib().b200bo_launch_count
    worst, per_row, prev = 0.0, None, KM.APPEND_BASE
    for n in KM.APPEND_SIZES:
        calls["append"], calls["full"] = [], 0
        l0 = launches()
        gp.fit(X[:n], y[:n])
        used = launches() - l0
        assert calls["append"] == [True] and calls["full"] == 0, (n, calls)
        if per_row is None:
            assert n - prev == 1
            per_row = used
        assert used == (n - prev) * per_row, (n, used, per_row)
        prev = n
        sk = _sk(k, X[:n], y[:n])
        assert_allclose(gp.L_, sk.L_, rtol=1e-8, atol=1e-11)
        assert_allclose(gp.alpha_, sk.alpha_, rtol=1e-6, atol=1e-9 * float(np.max(np.abs(sk.alpha_))))
        mu, sd = _predict_dev(gp, xt)
        mu0, sd0 = _predict_sk(sk, xt)
        s_y = float(sk._y_train_std)
        e_mu = float(np.max(np.abs(mu - mu0) / (np.abs(mu0) + s_y)))
        e_var = float(np.max(np.abs(sd**2 - sd0**2)) / (prior * s_y**2))
        worst = max(worst, e_mu, e_var)
        assert e_mu <= RTOL and e_var <= RTOL
    assert calls["full"] == 0  # reading L_, alpha_ and predicting did not refit either
    print(f"E {cid} append: mu/var {worst:.1e} ({per_row} launches per appended row)")
    assert worst <= c["bar"]
