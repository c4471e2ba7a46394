"""Analytic input gradients on the device (DESIGN.md 4.10): b200bo_acq_value_grad and b200bo_paths_grad_rows against
the numpy restatement of tests/grad_oracle.py (pinned to extended-precision differences by tests/test_grad_cpu.py),
their own consistency (central differences of the device values, value bit-equality, row independence), the rules at
rounded dimensions / training inputs / clamped variances / NaN values, and the opt-in analytic refinement.

Gradient metric: max_j |d grad_j| / (max_j |grad_j| + |val| / min_j ls_j + 1e-6), per row, maximum over the rows (the
floor keeps rows where value and gradient underflow together, EI / PoI far below the incumbent, from turning round-off
into large relative numbers).  Every case prints its measured errors (pytest -s): uniform rows / rows at and 1e-3 from
training rows.
"""
from types import SimpleNamespace

import numpy as np
import pytest
from scipy.linalg import cho_solve

import grad_oracle as G
import kernel_matrix_cases as KM

pytestmark = pytest.mark.gpu

ALPHA = 1e-6
KAPPA, XI = 2.576, 0.01
# RTOL: north-star bar of the fp64 path (values).  Gradient bars: about 10x the largest error measured over the
# matrix on an H100 80GB HBM3 (700 W power limit), DESIGN.md 4.10: 3.7e-11 on uniform rows (p9); at and next to
# training rows 1.1e-9 for UCB / EI / PoI (p13) and 1.9e-4 for MES (p9: g = (y* - mu) / sigma divides by a sigma that
# is a cancellation residue there, which amplifies its relative error in the value and the gradient alike).
RTOL = 1e-5
BAR_UNIFORM, BAR_EDGE, BAR_EDGE_MES = 1e-9, 1e-8, 2e-3


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _oracle_gp(c, X, y, d):
    return G.GradGP(X, y, KM.NU[c["kern"]], KM.length_scale(c, d), const=c.get("const") or 1.0,
                    noise=c.get("white") or 0.0, alpha=ALPHA, rnd=c.get("rnd", 0))


def _device_gp(bo, c, X, y, d):
    return bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=ALPHA, normalize_y=True,
                                           optimizer=None).fit(X, y)


def _rows(c, X, d, rs):
    """16 uniform rows, 8 rows 1e-3 from a training row, 8 training rows."""
    uni = KM.inputs(c, 16, d, rs)
    near = X[rs.choice(len(X), 8, replace=False)] + 1e-3 * rs.choice([-1.0, 1.0], size=(8, d))
    return np.vstack([uni, near, X[rs.choice(len(X), 8, replace=False)]])


def _grad_err(grad, want, val, ls):
    scale = np.max(np.abs(want), axis=1) + np.abs(val) / np.min(ls) + 1e-6
    return np.max(np.abs(grad - want), axis=1) / scale


def _params(kind, y_max):
    if kind == G.UCB:
        return dict(kappa=KAPPA)
    if kind == G.MES:
        return dict(ystar=[y_max + 0.1, y_max + 0.4, y_max + 1.0])
    return dict(xi=XI, y_max=y_max)


def _closure(bo, kind, gp, y_max, constraint=None):
    kw = dict(max_values=_params(kind, y_max)["ystar"]) if kind == G.MES else {}
    return bo.FusedAcquisition(kind, gp, constraint, kappa=KAPPA, xi=XI, y_max=y_max, **kw)


@pytest.fixture(scope="module")
def cases(bo):
    cache = {}

    def get(cid):
        if cid not in cache:
            c = KM.PREDICT[cid]
            n, d = c["n"], c["d"]
            X, y, rs = KM.problem(c, n, d, 100 + sorted(KM.PREDICT).index(cid))
            cache[cid] = SimpleNamespace(c=c, d=d, X=X, y=y, xt=_rows(c, X, d, rs), y_max=float(np.median(y)),
                                         ogp=_oracle_gp(c, X, y, d), gp=_device_gp(bo, c, X, y, d))
        return cache[cid]

    return get


# ---------------------------------------------------------------------------------------------------------------
# gradient parity
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_gradient_parity_matrix(bo, cases, cid):
    r = cases(cid)
    worst = {}
    for kind in (G.UCB, G.EI, G.POI, G.MES):
        f = _closure(bo, kind, r.gp, r.y_max)
        val, grad = f.value_and_grad(r.xt)
        wv, wg = G.acq_value_grad(kind, r.ogp, r.xt, **_params(kind, r.y_max))
        ok = np.isfinite(wv)
        assert np.array_equal(np.isnan(val), ~ok)
        np.testing.assert_allclose(val[ok], wv[ok], rtol=RTOL, atol=1e-12)
        err = _grad_err(grad[ok], wg[ok], wv[ok], r.ogp.ls)
        worst[kind] = (float(np.max(err[:16])), float(np.max(err[16:])))
        if r.c.get("rnd"):
            assert np.all(grad[ok][:, r.d - r.c["rnd"]:] == 0.0)  # a rounded dimension: exactly 0
        assert np.all(np.isfinite(grad[ok]))  # also Matern 1/2 at a training row
    print(f"G {cid}: " + " ".join(f"{k}: {u:.1e}/{e:.1e}" for k, (u, e) in worst.items()))
    assert max(u for u, _ in worst.values()) <= BAR_UNIFORM
    assert max(e for k, (_, e) in worst.items() if k != G.MES) <= BAR_EDGE
    assert worst[G.MES][1] <= BAR_EDGE_MES


@pytest.mark.parametrize("cid", sorted(KM.CONSTRAINED))
def test_gradient_parity_two_constraints(bo, cid):
    c = KM.CONSTRAINED[cid]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(KM.CONSTRAINED_TARGET, n, d, 200 + sorted(KM.CONSTRAINED).index(cid))
    s = X.sum(1) / np.sqrt(d)
    cv = [np.cos(2 * s), np.sin(3 * s) + 0.3 * X[:, 0]]
    specs = KM.CONSTRAINTS[:2]
    xt = _rows(KM.CONSTRAINED_TARGET, X, d, rs)[:24]  # at a training row a constraint's sigma is a residue
    gp, ogp = _device_gp(bo, KM.CONSTRAINED_TARGET, X, y, d), _oracle_gp(KM.CONSTRAINED_TARGET, X, y, d)
    cgps = [_device_gp(bo, sp, X, t, d) for (sp, _, _), t in zip(specs, cv)]
    ocons = [(_oracle_gp(sp, X, t, d), lb, ub) for (sp, lb, ub), t in zip(specs, cv)]
    cm = SimpleNamespace(model=cgps, lb=[lb for _, lb, _ in specs], ub=[ub for _, _, ub in specs])
    y_max = float(np.median(y))
    val, grad = _closure(bo, G.EI, gp, y_max, cm).value_and_grad(xt)
    wv, wg = G.acq_value_grad(G.EI, ogp, xt, ocons, xi=XI, y_max=y_max)
    np.testing.assert_allclose(val, wv, rtol=RTOL, atol=1e-12)
    err = _grad_err(grad, wg, wv, ogp.ls)
    print(f"G2 {cid}: {np.max(err[:16]):.1e}/{np.max(err[16:]):.1e}")
    assert np.max(err[:16]) <= BAR_UNIFORM and np.max(err[16:]) <= BAR_EDGE


@pytest.mark.parametrize("cid", ["p7", "p12", "p11"])
def test_gradient_matches_differences_of_the_device_values(bo, cases, monkeypatch, cid):
    """Central differences of the device's own b200bo_acq_eval (small path, step 1e-5 ls): catches a formula that
    would match a wrong oracle.  Truncation is O(h^2); the values' round-off over h is what bounds the check."""
    monkeypatch.setenv("B200BO_SMALL_PATH", "1")
    r = cases(cid)
    xt = r.xt[:6]
    for kind in (G.UCB, G.EI):
        f = _closure(bo, kind, r.gp, r.y_max)
        val, grad = f.value_and_grad(xt)
        fd = np.empty_like(grad)
        for j in range(r.d):
            h = np.zeros(r.d)
            h[j] = 1e-5 * r.ogp.ls[j]
            fd[:, j] = (f(xt + h) - f(xt - h)) / (2 * h[j])
        assert np.max(_grad_err(grad, fd, val, r.ogp.ls)) <= 1e-4


# ---------------------------------------------------------------------------------------------------------------
# value bit-equality and row independence
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", ["p2", "p5"])
def test_value_is_bit_equal_and_rows_are_independent(bo, cases, monkeypatch, cid):
    monkeypatch.setenv("B200BO_SMALL_PATH", "1")
    r = cases(cid)
    rs = np.random.RandomState(9)
    big = KM.inputs(r.c, 300, r.d, rs)  # crosses pass (32) and launch-group (256) boundaries
    for kind in (G.EI, G.MES):
        f = _closure(bo, kind, r.gp, r.y_max)
        val, grad = f.value_and_grad(big)
        assert np.array_equal(val, f(big))
        row = big[7]
        v1, g1 = f.value_and_grad(row)
        assert v1[0] == val[7] and np.array_equal(g1[0], grad[7])
        for pos in (31, 32, 33, 299):
            batch = big.copy()
            batch[pos] = row
            v, g = f.value_and_grad(batch[:max(pos + 1, 34)] if pos < 299 else batch)
            assert v[pos] == val[7] and np.array_equal(g[pos], grad[7])


# ---------------------------------------------------------------------------------------------------------------
# rules
# ---------------------------------------------------------------------------------------------------------------
def test_clamped_variance_nan_values_and_infinite_bounds(bo):
    from sklearn.gaussian_process.kernels import RBF

    rs = np.random.RandomState(2)
    X = rs.uniform(size=(200, 2))
    y = np.sin(4 * X.sum(1))
    gp = bo.B200GaussianProcessRegressor(kernel=RBF(0.8), alpha=1e-10, normalize_y=True, optimizer=None).fit(X, y)
    xt = np.vstack([X[:40], rs.uniform(size=(8, 2))])
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, sd = gp.predict(xt, return_std=True)
    clamped = sd == 0.0  # where the variance is clamped (if anywhere on these rows): d sd := 0
    val, grad = bo.FusedAcquisition(bo._lib.ACQ_UCB, gp, kappa=KAPPA).value_and_grad(xt)
    assert np.all(np.isfinite(val)) and np.all(np.isfinite(grad))
    # a constraint GP with sigma = 0 makes the value NaN (frozen-norm rule): a NaN gradient row, nothing invented
    cm = SimpleNamespace(model=[gp], lb=[-0.5], ub=[0.5])
    val, grad = bo.FusedAcquisition(bo._lib.ACQ_UCB, gp, cm, kappa=KAPPA).value_and_grad(xt)
    assert np.all(np.isnan(val[clamped])) and np.all(np.isnan(grad[clamped]))
    assert np.all(np.isfinite(grad[~clamped]))
    # bounds (-inf, inf): p = 1 and d p = 0
    free = SimpleNamespace(model=[gp], lb=[-np.inf], ub=[np.inf])
    v0, g0 = bo.FusedAcquisition(bo._lib.ACQ_UCB, gp, kappa=KAPPA).value_and_grad(xt[~clamped])
    v1, g1 = bo.FusedAcquisition(bo._lib.ACQ_UCB, gp, free, kappa=KAPPA).value_and_grad(xt[~clamped])
    np.testing.assert_allclose(v1, v0, rtol=1e-15)
    np.testing.assert_allclose(g1, g0, rtol=1e-13, atol=1e-300)


def test_mes_gradient_is_finite_far_in_both_tails(bo, cases):
    r = cases("p12")
    xt = r.xt[:8]
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mu, sd = r.gp.predict(xt, return_std=True)
    for g in (38.0, -38.0, 45.0):
        ystar = [float(mu[0] + g * sd[0])]
        val, grad = bo.FusedAcquisition(bo._lib.ACQ_MES, r.gp, max_values=ystar).value_and_grad(xt)
        assert np.all(np.isfinite(val)) and np.all(np.isfinite(grad))


def test_multi_device_and_host_transform_are_refused(bo, cases):
    f = _closure(bo, G.EI, cases("p9").gp, 0.0)
    f.devices = [0, 1]
    with pytest.raises(NotImplementedError, match="one device"):
        f.value_and_grad(np.zeros((1, 8)))


# ---------------------------------------------------------------------------------------------------------------
# sample paths
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [1, 4, 16])
@pytest.mark.parametrize("cid", ["p10", "p11", "p13", "p5", "p4"])
def test_path_gradient_matches_the_restatement(bo, cases, cid, q):
    from bayesianoptimization_b200.paths import draw_path_inputs

    r = cases(cid)
    L = 200
    paths = r.gp.sample_paths(q, L, random_state=11)
    og = r.ogp
    omega, b, w, eps = draw_path_inputs(np.random.RandomState(11), q, L, r.d, og.nu, len(r.X), ALPHA + og.noise)
    feat = np.sqrt(2.0 * og.const / L) * np.cos(og.Xs @ omega.T + b)
    V = cho_solve((og.L, True), og.y_norm[:, None] - feat @ w - eps)
    xt = r.xt
    pidx = np.arange(len(xt)) % q
    val, grad = paths.grad_rows(xt, pidx)
    assert np.array_equal(val, paths.eval_rows(xt, pidx))
    worst = 0.0
    for p in range(q):
        rows = pidx == p
        wv, wg = G.path_value_grad(og, omega, b, w[:, p], V[:, p], xt[rows])
        np.testing.assert_allclose(val[rows], wv, rtol=RTOL, atol=RTOL * og.y_std)
        worst = max(worst, float(np.max(_grad_err(grad[rows], wg, wv, og.ls))))
    print(f"P {cid} q={q}: {worst:.1e}")
    assert worst <= 1e-6
    with pytest.raises(ValueError):
        paths.grad_rows(xt[:2], np.array([0, q]))
    from bayesianoptimization_b200.paths import PathBatchAcquisition

    acq = PathBatchAcquisition(paths)
    v, g = acq.value_and_grad(xt, pidx)
    assert np.array_equal(v, -val) and np.array_equal(g, -grad)


# ---------------------------------------------------------------------------------------------------------------
# refinement
# ---------------------------------------------------------------------------------------------------------------
def _space(ref, d, lo=0.0, hi=1.0):
    from bayes_opt.target_space import TargetSpace

    return TargetSpace(None, {f"x{j:02d}": (lo, hi) for j in range(d)})


def _fitted(bo, n, d, seed, kernel=None):
    from sklearn.gaussian_process.kernels import Matern

    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1) / np.sqrt(d)) + 0.5 * np.cos(2 * X[:, 0]) + 0.05 * rs.randn(n)
    gp = bo.B200GaussianProcessRegressor(kernel=kernel or Matern(nu=2.5, length_scale=0.3 * np.sqrt(d)), alpha=1e-4,
                                         normalize_y=True, optimizer=None).fit(X, y)
    return gp, X, y


@pytest.mark.parametrize("n,d", [(40, 2), (512, 8), (300, 17)])
def test_analytic_refinement_is_at_least_as_good_as_the_stencil(bo, ref, n, d):
    gp, X, y = _fitted(bo, n, d, 31 + d)
    cgp, _, _ = _fitted(bo, n, d, 77 + d)
    space = _space(ref, d)
    cm = SimpleNamespace(model=[cgp], lb=[-0.3], ub=[np.inf])
    made = {
        "ei": (bo.ExpectedImprovement(xi=XI), None), "ucb": (bo.UpperConfidenceBound(kappa=KAPPA), None),
        "poi_c": (bo.ProbabilityOfImprovement(xi=XI), cm), "mes": (bo.MaxValueEntropySearch(n_samples=4, n_features=256), None),
        "ts": (bo.ThompsonSampling(n_features=256), None),
    }
    for name, (acq, con) in made.items():
        acq.y_max = float(y.max())
        acq._path_rng, acq._suggest_space = np.random.RandomState(5), space  # the closure's draws (MES, TS)
        closure = acq._get_acq(gp, con)
        seeds = np.random.RandomState(3).uniform(size=(6, d))
        out = {}
        for mode in ("stencil", "analytic"):
            acq.b200_refine = mode
            x, f = acq._smart_minimize(closure, space, seeds, np.random.RandomState(0))
            assert np.all(x >= space.bounds[:, 0]) and np.all(x <= space.bounds[:, 1]), (name, mode)
            out[mode] = float(np.asarray(closure(x)).ravel()[0])
        scale = max(abs(out["stencil"]), 1e-3)
        print(f"R {name} d={d}: stencil {out['stencil']:.12g} analytic {out['analytic']:.12g}")
        assert out["analytic"] <= out["stencil"] + 1e-6 * scale, (name, out)


def test_batch_thompson_and_a_full_run_with_analytic_refinement(bo, ref):
    from bayes_opt import BayesianOptimization

    gp, X, y = _fitted(bo, 120, 3, 4)
    space = _space(ref, 3)
    for x_, y_ in zip(X, y):
        space.register(x_, y_)
    ts = bo.ThompsonSampling(n_features=256)
    ts.b200_refine = "analytic"
    pts = ts.suggest_batch(gp, space, 4, n_random=2000, n_smart=4, fit_gp=False, random_state=np.random.RandomState(1))
    assert pts.shape == (4, 3) and len({p.tobytes() for p in pts}) == 4
    assert np.all(pts >= 0) and np.all(pts <= 1)

    def run():
        opt = BayesianOptimization(f=lambda x, y: -(x - 0.3) ** 2 - (y + 0.2) ** 2 + np.sin(3 * x), verbose=0,
                                   pbounds={"x": (-1, 1), "y": (-1, 1)}, random_state=7)
        bo.enable(opt, refine="analytic")
        opt.maximize(init_points=5, n_iter=10)
        return np.array([[r["params"]["x"], r["params"]["y"]] for r in opt.res])

    a, b = run(), run()
    assert a.shape == (15, 2) and np.array_equal(a, b)  # deterministic


def test_default_refinement_never_asks_for_gradients(bo, ref, monkeypatch):
    from bayes_opt import BayesianOptimization

    calls = []
    orig = bo.FusedAcquisition.value_and_grad
    monkeypatch.setattr(bo.FusedAcquisition, "value_and_grad", lambda self, x: calls.append(1) or orig(self, x))
    opt = BayesianOptimization(f=lambda x, y: -(x - 0.3) ** 2 - (y + 0.2) ** 2, verbose=0,
                               pbounds={"x": (-1, 1), "y": (-1, 1)}, random_state=7)
    bo.enable(opt)
    opt.maximize(init_points=3, n_iter=3)
    assert not calls
    opt2 = BayesianOptimization(f=lambda x, y: -(x - 0.3) ** 2 - (y + 0.2) ** 2, verbose=0,
                                pbounds={"x": (-1, 1), "y": (-1, 1)}, random_state=7)
    bo.enable(opt2, refine="analytic")
    opt2.maximize(init_points=3, n_iter=3)
    assert calls
