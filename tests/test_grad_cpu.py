"""Analytic input gradients without a GPU (DESIGN.md 4.10).

* The closed forms restated in tests/grad_oracle.py - the oracle the device gradients are held to - agree with central
  differences of the closure value evaluated by mpmath at 50 digits, for every covariance code x iso/ARD x
  UCB/EI/PoI/MES x {0, 2} constraints, and for a sample path.  This pins the formulas independently of CUDA.
* ``_batched_lbfgsb(grad=True)`` equals ``scipy.optimize.minimize(jac=True, method="L-BFGS-B")`` bit for bit.
* The ``refine`` switch of ``enable`` / ``accelerate``: validation, propagation, defaults; the library exports the new
  entry points.
"""
import ctypes as C
import math

import mpmath as mp
import numpy as np
import pytest
from scipy.optimize import minimize

import grad_oracle as G

NUS = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}
KAPPA, XI = 2.576, 0.01


# ---------------------------------------------------------------------------------------------------------------
# the closure value at 50 digits
# ---------------------------------------------------------------------------------------------------------------
def _mp_k(r, nu):
    if nu == 0.5:
        return mp.exp(-r)
    if nu == 1.5:
        a = mp.sqrt(3) * r
        return (1 + a) * mp.exp(-a)
    if nu == 2.5:
        a = mp.sqrt(5) * r
        return (1 + a + a * a / 3) * mp.exp(-a)
    return mp.exp(-r * r / 2)


class _MpGP:
    """The GradGP's posterior re-evaluated in extended precision from the same inputs."""

    def __init__(self, gp):
        self.gp = gp
        n = gp.Xs.shape[0]
        self.Xs = [[mp.mpf(float(v)) for v in row] for row in gp.Xs]
        K = mp.matrix(n, n)
        for i in range(n):
            for j in range(n):
                r = mp.sqrt(sum((self.Xs[i][t] - self.Xs[j][t]) ** 2 for t in range(gp.d)))
                K[i, j] = mp.mpf(gp.const) * _mp_k(r, gp.nu)
            K[i, i] = mp.mpf(float(gp.K[i, i]))
        self.Kinv = K ** -1
        self.alpha = self.Kinv * mp.matrix([mp.mpf(float(v)) for v in gp.y_norm])

    def mean_sd(self, x):
        gp = self.gp
        xs = [x[j] / mp.mpf(float(gp.ls[j])) for j in range(gp.d)]
        ks = mp.matrix([mp.mpf(gp.const) * _mp_k(mp.sqrt(sum((xs[t] - row[t]) ** 2 for t in range(gp.d))), gp.nu)
                        for row in self.Xs])
        mean = mp.mpf(gp.y_std) * (ks.T * self.alpha)[0] + mp.mpf(gp.y_mean)
        var = mp.mpf(gp.prior) - (ks.T * self.Kinv * ks)[0]
        return mean, mp.mpf(gp.y_std) * mp.sqrt(var)


def _mp_value(kind, target, constraints, x, y_max, ystar):
    mean, sd = target.mean_sd(x)
    if kind == G.UCB:
        base = mean + KAPPA * sd
    elif kind == G.MES:
        base = 0
        for ys in ystar:
            g = (mp.mpf(float(ys)) - mean) / sd
            base += g * mp.npdf(g) / (2 * mp.ncdf(g)) - mp.log(mp.ncdf(g))
        base /= len(ystar)
    else:
        a = mean - y_max - XI
        z = a / sd
        base = mp.ncdf(z) if kind == G.POI else a * mp.ncdf(z) + sd * mp.npdf(z)
    val = -base
    for cgp, lb, ub in constraints:
        m, s = cgp.mean_sd(x)
        hi = 1 if ub == np.inf else mp.ncdf((ub - m) / s)
        lo = 0 if lb == -np.inf else mp.ncdf((lb - m) / s)
        val *= hi - lo
    return val


def _central(f, x, h=mp.mpf(10) ** -20):
    out = []
    for j in range(len(x)):
        xp, xm = list(x), list(x)
        xp[j] += h
        xm[j] -= h
        out.append(float((f(xp) - f(xm)) / (2 * h)))
    return np.array(out)


def _problem(nu, ard, seed, n=9, d=3):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    ls = np.array([0.2, 0.35, 0.6]) if ard else 0.3  # short: sigma stays a fair fraction of the prior
    y = np.sin(3 * X.sum(1)) + 0.1 * rs.randn(n)
    cy = [np.cos(2 * X.sum(1)), X[:, 0] - X[:, 1]]
    gp = G.GradGP(X, y, nu, ls, const=1.3, noise=1e-2, alpha=1e-6)
    cons = [(G.GradGP(X, cy[0], nu, ls, alpha=1e-2), -0.4, 0.9), (G.GradGP(X, cy[1], 2.5, 0.5, alpha=1e-2), -np.inf, 0.6)]
    return gp, cons, rs.uniform(0.7, 1.3, size=(3, d)), float(np.median(y))  # rows at the edge of the data, an
    # incumbent EI / PoI can resolve: every factor of the value is far from underflow, so fp64 carries 1e-8


@pytest.mark.parametrize("ncons", [0, 2])
@pytest.mark.parametrize("kind", [G.UCB, G.EI, G.POI, G.MES])
@pytest.mark.parametrize("ard", [False, True])
@pytest.mark.parametrize("kern", sorted(NUS))
def test_closed_form_gradient_matches_extended_precision_differences(kern, ard, kind, ncons):
    mp.mp.dps = 50
    gp, cons, xt, y_max = _problem(NUS[kern], ard, 7 + sorted(NUS).index(kern))
    cons = cons[:ncons]
    ystar = [y_max + 1.2, y_max + 1.7]
    val, grad = G.acq_value_grad(kind, gp, xt, cons, **(
        dict(kappa=KAPPA) if kind == G.UCB else dict(ystar=ystar) if kind == G.MES else dict(xi=XI, y_max=y_max)))
    mgp, mcons = _MpGP(gp), [(_MpGP(c), lb, ub) for c, lb, ub in cons]
    for i, x in enumerate(xt):
        xm = [mp.mpf(float(v)) for v in x]
        f = lambda p: _mp_value(kind, mgp, mcons, p, y_max, ystar)  # noqa: E731
        assert float(f(xm)) == pytest.approx(val[i], rel=1e-9, abs=1e-12)
        want = _central(f, xm)
        assert np.max(np.abs(grad[i] - want)) <= 1e-8 * (np.max(np.abs(want)) + abs(val[i])), (grad[i], want)


def test_oracle_value_matches_gp_oracle_predict():
    """The GradGP posterior is oracle/gp_oracle.py's predict on the same state."""
    from oracle import gp_oracle as O

    rs = np.random.RandomState(3)
    X, y = rs.uniform(size=(20, 4)), rs.randn(20)
    gp = G.GradGP(X, y, 2.5, 0.7, alpha=1e-6)
    st = O.fit_fixed(X, y, length_scale=0.7)
    xt = rs.uniform(size=(5, 4))
    mean, sd, _, _ = gp.predict_grad(xt)
    mu, s = O.predict(st, xt)
    np.testing.assert_allclose(mean, mu, rtol=1e-10)
    np.testing.assert_allclose(sd, s, rtol=1e-8)


def test_gradient_rules():
    rs = np.random.RandomState(5)
    X, y = rs.uniform(0, 3, size=(12, 3)), rs.randn(12)
    gp = G.GradGP(X, y, 0.5, 0.8, rnd=1)
    xt = np.vstack([rs.uniform(0, 3, size=(2, 3)), X[4]])
    val, grad = G.acq_value_grad(G.EI, gp, xt, xi=XI, y_max=float(y.max()))
    assert np.all(grad[:, 2] == 0.0)             # rounded dimension
    assert np.all(np.isfinite(grad))             # Matern 1/2 at a training row: h(0) := 0
    _, _, _, dsd = G.GradGP(X, y, 2.5, 0.8, alpha=0.0).predict_grad(X[:3])
    assert np.all(np.isfinite(dsd))              # sigma = 0 at a training row: d sd := 0 or finite


@pytest.mark.parametrize("kern", sorted(NUS))
def test_path_gradient_matches_extended_precision_differences(kern):
    mp.mp.dps = 50
    nu = NUS[kern]
    gp, _, xt, _ = _problem(nu, True, 21)
    rs = np.random.RandomState(1)
    L = 16
    omega, bias, w, v = rs.standard_normal((L, gp.d)), rs.uniform(0, 2 * np.pi, L), rs.standard_normal(L), rs.randn(9)
    val, grad = G.path_value_grad(gp, omega, bias, w, v, xt)

    def f(p):
        xs = [p[j] / mp.mpf(float(gp.ls[j])) for j in range(gp.d)]
        feat = sum(mp.mpf(float(w[l])) * mp.cos(sum(mp.mpf(float(omega[l, j])) * xs[j] for j in range(gp.d)) +
                                                 mp.mpf(float(bias[l]))) for l in range(L))
        upd = sum(mp.mpf(float(v[i])) * gp.const * _mp_k(mp.sqrt(sum((xs[t] - mp.mpf(float(gp.Xs[i, t]))) ** 2
                                                                     for t in range(gp.d))), nu) for i in range(9))
        return mp.mpf(gp.y_std) * (mp.sqrt(2 * mp.mpf(gp.const) / L) * feat + upd) + mp.mpf(gp.y_mean)

    for i, x in enumerate(xt):
        xm = [mp.mpf(float(t)) for t in x]
        assert float(f(xm)) == pytest.approx(val[i], rel=1e-12)
        want = _central(f, xm)
        assert np.max(np.abs(grad[i] - want)) <= 1e-11 * (np.max(np.abs(want)) + abs(val[i]))


# ---------------------------------------------------------------------------------------------------------------
# the batched driver with analytic gradients
# ---------------------------------------------------------------------------------------------------------------
class _Closure:
    """A test closure with exact gradients in the signature of the device closures."""

    def __init__(self, fun):
        self.fun = fun
        self.rows = 0

    def value_and_grad(self, x):
        x = np.atleast_2d(x)
        self.rows += len(x)
        out = [self.fun(r) for r in x]
        return np.array([f for f, _ in out]), np.array([g for _, g in out])


def _bowl(x):
    c = np.array([0.3, -0.2, 0.9, 1.4])
    s = np.array([1.0, 4.0, 0.5, 2.0])
    return float(np.sum(s * (x - c) ** 2)), 2 * s * (x - c)


def _rosen(x):
    f = np.sum(100.0 * (x[1:] - x[:-1] ** 2) ** 2 + (1 - x[:-1]) ** 2)
    g = np.zeros_like(x)
    g[:-1] = -400 * x[:-1] * (x[1:] - x[:-1] ** 2) - 2 * (1 - x[:-1])
    g[1:] += 200 * (x[1:] - x[:-1] ** 2)
    return float(f), g


@pytest.mark.parametrize("fun", [_bowl, _rosen])
def test_batched_lbfgsb_with_gradients_equals_scipy(fun):
    from bayesianoptimization_b200.fused import _batched_lbfgsb, lockstep_lbfgsb

    bounds = np.array([[-1.0, 1.2]] * 4)  # the bowl's minimiser (x_3 = 1.4) lies outside: that run ends on a bound
    rs = np.random.RandomState(0)
    seeds = list(rs.uniform(-1, 1.2, size=(5, 4))) + [np.array([-1.0, 1.2, 0.0, 1.2])]  # a seed on a bound
    acq = _Closure(fun)
    got = _batched_lbfgsb(acq, seeds, bounds, grad=True)
    assert acq.rows == sum(r.nfev for r in got)  # one row per evaluation
    for s, r in zip(seeds, got):
        w = minimize(fun, s, jac=True, bounds=bounds, method="L-BFGS-B")
        assert np.array_equal(r.x, w.x) and float(r.fun) == float(w.fun)
        assert (r.nit, r.nfev, r.status, r.success) == (w.nit, w.nfev, w.status, w.success)
        assert np.array_equal(r.jac, w.jac)
    # the public driver: lockstep, and the sequential route of a single seed
    for s, r in zip(seeds, lockstep_lbfgsb(_Closure(fun), seeds, bounds, grad=True)):
        assert np.array_equal(r.x, minimize(fun, s, jac=True, bounds=bounds, method="L-BFGS-B").x)
    one = lockstep_lbfgsb(_Closure(fun), seeds[:1], bounds, grad=True)[0]
    assert np.array_equal(one.x, minimize(fun, seeds[0], jac=True, bounds=bounds, method="L-BFGS-B").x)


def test_batched_lbfgsb_gradient_rows_carry_their_path():
    from bayesianoptimization_b200.fused import _batched_lbfgsb

    class Paths:
        def value_and_grad(self, x, path_idx):
            c = np.asarray(path_idx, dtype=float)[:, None] * 0.25
            return ((x - c) ** 2).sum(1), 2 * (x - c)

    bounds = np.array([[-1.0, 1.0]] * 2)
    runs = _batched_lbfgsb(Paths(), [np.zeros(2) + 0.7] * 3, bounds, run_paths=[0, 1, 2], grad=True)
    for p, r in enumerate(runs):
        np.testing.assert_allclose(r.x, 0.25 * p, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# the switch
# ---------------------------------------------------------------------------------------------------------------
def test_refine_switch(ref):
    import bayesianoptimization_b200 as bo
    from bayes_opt import BayesianOptimization
    from bayes_opt import acquisition as R
    from bayesianoptimization_b200.acquisition import DeviceHooks, accelerate

    assert DeviceHooks.b200_refine == "stencil"
    assert bo.ExpectedImprovement(xi=0.0).b200_refine == "stencil"
    acq = accelerate(R.UpperConfidenceBound(), refine="analytic")
    assert acq.b200_refine == "analytic" and acq.b200_candidate_source == "host_rng"
    assert accelerate(acq).b200_refine == "analytic"  # None leaves the setting
    with pytest.raises(ValueError, match="refine"):
        accelerate(R.UpperConfidenceBound(), refine="exact")
    liar = accelerate(R.ConstantLiar(R.ExpectedImprovement(xi=0.0)), refine="analytic")
    assert liar.base_acquisition.b200_refine == "analytic"
    hedge = accelerate(R.GPHedge([R.UpperConfidenceBound(), R.ExpectedImprovement(xi=0.0)]), refine="analytic")
    assert [a.b200_refine for a in hedge.base_acquisitions] == ["analytic"] * 2

    def make():
        return BayesianOptimization(f=None, pbounds={"x": (0, 1)}, acquisition_function=R.UpperConfidenceBound(),
                                    verbose=0, random_state=1)

    opt = make()
    with pytest.raises(ValueError, match="refine"):
        bo.enable(opt, refine="gradient")
    with pytest.raises(NotImplementedError, match="one device"):
        bo.enable(opt, devices=[0, 1], refine="analytic")
    assert not isinstance(opt._acquisition_function, DeviceHooks)  # a refused enable() changes nothing
    assert bo.enable(make())._acquisition_function.b200_refine == "stencil"
    opt = bo.enable(make(), refine="analytic")
    assert opt._acquisition_function.b200_refine == "analytic"
    assert "refine" not in str(opt._acquisition_function.get_acquisition_params())


def test_analytic_refinement_needs_a_gradient_closure(ref):
    """Anything without value_and_grad, a mixed space, or the default setting stays on the stencil."""
    import bayesianoptimization_b200 as bo
    from types import SimpleNamespace

    acq = bo.UpperConfidenceBound()
    cont = SimpleNamespace(continuous_dimensions=[True, True])
    mixed = SimpleNamespace(continuous_dimensions=[True, False])
    grad = SimpleNamespace(value_and_grad=lambda x: None, devices=[0])
    assert not acq._refine_grad(grad, cont)
    acq.b200_refine = "analytic"
    assert acq._refine_grad(grad, cont)
    assert not acq._refine_grad(grad, mixed)
    assert not acq._refine_grad(lambda x: x, cont)
    assert not acq._refine_grad(SimpleNamespace(value_and_grad=None, devices=[0]), cont)
    assert not acq._refine_grad(SimpleNamespace(value_and_grad=lambda x: None, devices=[0, 1]), cont)


def test_library_exports_gradient_entry_points():
    import __graft_entry__ as g

    g.build()
    from bayesianoptimization_b200 import _lib as B

    L = C.CDLL(B.LIB_PATH)
    for name in ("b200bo_acq_value_grad", "b200bo_paths_grad_rows"):
        assert hasattr(L, name) and name in B.EXPORTS
    assert B.lib().b200bo_acq_value_grad.argtypes is not None
    assert math.isfinite(B.lib().b200bo_version())
