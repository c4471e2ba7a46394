"""NEI with pending points without a GPU: the restatement tests/nei_batch_oracle.py against independent forms (the
full Cholesky factor of X u P, the closed-form posterior of the pending values, a brute-force Monte-Carlo of
E[(f(x) - max g(X u P))+] from the joint covariance), and the refusals of the acquisition layer."""
from __future__ import annotations

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve, cholesky
from sklearn.gaussian_process.kernels import ConstantKernel, Matern

import nei_batch_oracle as NB
import nei_oracle as NO

C0, LS = 1.3, 0.4


def _problem(n=12, p=3, d=2, s2=0.05, tau=1e-6, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    P = rs.uniform(size=(p, d))
    y_n = np.sin(3 * X.sum(1)) + np.sqrt(s2) * rs.randn(n)
    kc = ConstantKernel(C0) * Matern(length_scale=LS, nu=2.5)
    return kc, X, P, y_n, s2, tau


@pytest.mark.parametrize("s2", [0.05, 1e-6])  # WhiteKernel-like noise, and sigma_n^2 = tau
def test_restatement_equals_the_full_factor_form(s2):
    kc, X, P, y_n, _, tau = _problem(p=4)
    n, p, S = X.shape[0], P.shape[0], 5
    Z, E, Zp = NB.draws(np.random.RandomState(1), n, S, p)
    mask = np.ones(n, bool)
    Fa, A, best = NB.pending_fantasies(kc, X, P, y_n, s2, tau, Z, E, Zp, mask)
    Xa = np.vstack([X, P])
    L = cholesky(kc(Xa) + tau * np.eye(n + p), lower=True)
    W = NB.residual_solve(kc(X), y_n, s2, tau, Z, E)
    want = (L @ np.vstack([Z, Zp]))[n:] + kc(P, X) @ W
    np.testing.assert_allclose(Fa[n:], want, rtol=0, atol=1e-12)
    F, _, best0 = NO.fantasies(kc(X), y_n, s2, tau, Z, E, mask)
    np.testing.assert_array_equal(Fa[:n], F)
    assert np.array_equal(best, np.maximum(best0, Fa[n:].max(axis=0)))
    np.testing.assert_allclose(A, cho_solve(cho_factor(kc(Xa) + tau * np.eye(n + p), lower=True), Fa), atol=1e-9)
    if s2 == tau:  # F_js = mu(x_j) + l_P^T z_P + r z_js: the registered draws cancel
        mu = kc(P, X) @ cho_solve(cho_factor(kc(X) + tau * np.eye(n), lower=True), y_n)
        np.testing.assert_allclose(want[0], mu[0] + L[n, n] * Zp[0], atol=1e-10)


def test_no_pending_rows_change_nothing():
    kc, X, P, y_n, s2, tau = _problem()
    Z, E, Zp = NB.draws(np.random.RandomState(2), X.shape[0], 3, 0)
    Fa, A, best = NB.pending_fantasies(kc, X, P[:0], y_n, s2, tau, Z, E, Zp, np.ones(X.shape[0], bool))
    F, A0, best0 = NO.fantasies(kc(X), y_n, s2, tau, Z, E, np.ones(X.shape[0], bool))
    assert np.array_equal(Fa, F) and np.array_equal(best, best0)
    np.testing.assert_allclose(A, A0, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("s2", [0.05, 1e-6])
def test_pending_values_follow_the_posterior(s2):
    """Over 1e5 seeded draws the pending fantasies have the mean and covariance of g_tau(P) | y: mean
    k(P, X) K^-1 y, covariance K0(P, P) - k(P, X) K^-1 k(X, P), the tau nugget on its diagonal."""
    kc, X, P, y_n, _, tau = _problem(n=8, p=3)
    n, p, S = X.shape[0], P.shape[0], 100_000
    Z, E, Zp = NB.draws(np.random.RandomState(3), n, S, p)
    Fa, _, _ = NB.pending_fantasies(kc, X, P, y_n, s2, tau, Z, E, Zp, np.ones(n, bool))
    FP = Fa[n:]
    Kf = cho_factor(kc(X) + s2 * np.eye(n), lower=True)
    kpx = kc(P, X)
    mean = kpx @ cho_solve(Kf, y_n)
    cov = kc(P) + tau * np.eye(p) - kpx @ cho_solve(Kf, kpx.T)
    se = np.sqrt(np.diag(cov) / S)
    assert np.all(np.abs(FP.mean(axis=1) - mean) <= 4 * se)
    emp = np.cov(FP)
    se_cov = np.sqrt((np.outer(np.diag(cov), np.diag(cov)) + cov ** 2) / S)
    assert np.all(np.abs(emp - cov) <= 4 * se_cov)


@pytest.mark.parametrize("log", [False, True])
def test_nei_matches_a_brute_force_monte_carlo(log):
    """NEI on the grown noiseless GP against E[(f(x) - max g_tau(X u P))+] drawn directly from the joint posterior of
    (g_tau(X u P), f(x)) given y - no Matheron step."""
    kc, X, P, y_n, s2, tau = _problem(n=10, p=2, seed=4)
    n, p, S = X.shape[0], P.shape[0], 200_000
    mask = np.zeros(n, bool)
    mask[::2] = True
    xc = np.array([[0.3, 0.6], [0.8, 0.2]])
    Z, E, Zp = NB.draws(np.random.RandomState(5), n, S, p)
    Fa, A, best = NB.pending_fantasies(kc, X, P, y_n, s2, tau, Z, E, Zp, mask)
    got = NB.nei(kc, np.vstack([X, P]), A, best, tau, xc, 0.0, log=log)
    rs = np.random.RandomState(6)
    Xa = np.vstack([X, P])
    Kf = cho_factor(kc(X) + s2 * np.eye(n), lower=True)
    for i, x in enumerate(xc):
        T = np.vstack([Xa, x[None]])
        prior = kc(T) + np.diag(np.r_[np.full(n + p, tau), 0.0])
        cross = kc(T, X)
        m = cross @ cho_solve(Kf, y_n)
        C = prior - cross @ cho_solve(Kf, cross.T)
        w, V = np.linalg.eigh(C)
        G = m + (rs.standard_normal((S, len(m))) * np.sqrt(np.maximum(w, 0.0))) @ V.T
        inc = np.r_[mask, np.ones(p, bool)]
        imp = np.maximum(G[:, -1] - G[:, :n + p][:, inc].max(axis=1), 0.0)
        want, se = imp.mean(), imp.std() / np.sqrt(S)
        val = np.exp(got[i]) if log else got[i]
        # two independent Monte-Carlo estimates: their difference within 4 combined standard errors
        assert abs(val - want) <= 4 * np.sqrt(2.0) * se, (i, val, want, se)


def test_refusals():
    pytest.importorskip("bayes_opt")
    import bayesianoptimization_b200 as bo

    for base in (bo.ExpectedImprovement(xi=0.0), bo.UpperConfidenceBound(), bo.MaxValueEntropySearch(),
                 bo.ThompsonSampling()):
        with pytest.raises(TypeError, match="PendingNEI needs"):
            bo.PendingNEI(base)
    for cls in (bo.NoisyExpectedImprovement, bo.LogNoisyExpectedImprovement):
        acq = bo.PendingNEI(cls(n_samples=4))
        assert isinstance(acq, bo.AcquisitionFunction) and acq.dummies == []
        with pytest.raises(TypeError):
            bo.KrigingBeliever(cls())
        with pytest.raises(TypeError):
            bo.ConstantLiar(cls())
        with pytest.raises(TypeError):
            bo.GPHedge([cls()])


def test_empty_and_constrained_spaces_are_refused_before_any_device_work():
    pytest.importorskip("bayes_opt")
    from bayes_opt.constraint import ConstraintModel
    from bayes_opt.exception import ConstraintNotSupportedError, TargetSpaceEmptyError
    from bayes_opt.target_space import TargetSpace

    import bayesianoptimization_b200 as bo

    pb = {"a": (0.0, 1.0), "b": (0.0, 1.0)}
    acq = bo.PendingNEI(bo.LogNoisyExpectedImprovement(n_samples=2))
    with pytest.raises(TargetSpaceEmptyError):
        acq.suggest_batch(None, TargetSpace(None, pb), 2)
    space = TargetSpace(None, pb, constraint=ConstraintModel(lambda a, b: a - b, -np.inf, 0.0))
    space.register(np.array([0.2, 0.4]), 1.0, constraint_value=-0.2)
    with pytest.raises(ConstraintNotSupportedError):
        acq.suggest_batch(None, space, 2)
    with pytest.raises(ValueError):
        acq.suggest_batch(None, space, 0)
    with pytest.raises(TypeError, match="PendingNEI"):
        class Opt:
            _acquisition_function = bo.NoisyExpectedImprovement()
        bo.suggest_batch(Opt(), 2)


def test_multi_device_gp_is_refused_before_any_draw():
    import bayesianoptimization_b200 as bo

    gp = bo.B200GaussianProcessRegressor(devices=[0, 1])
    gp.X_train_ = np.zeros((3, 2))
    rs = np.random.RandomState(0)
    with pytest.raises(NotImplementedError, match="multi-device"):
        gp.noiseless_fantasies(2, random_state=rs, pending=np.zeros((1, 2)))
    assert np.array_equal(rs.get_state()[1], np.random.RandomState(0).get_state()[1])


@pytest.mark.parametrize("name", ["c_m25_d3", "b_m15_d17", "b_m25_c3"])
def test_double_double_fixtures_agree_with_the_restatement(name):
    """tests/golden/neibatch_*.npz (oracle/make_nei_batch.py): the inputs match the digests, and the fp64 restatement
    stored beside the truth meets it far inside the device's bars - the two pipelines share no code past the draws."""
    from oracle import make_nei_batch as NBB

    r = NBB.load(name)
    ys = float(r["y_std"])
    assert r["P"].shape == (NBB.P_MAX, r["X"].shape[1])
    for p in NBB.PS:
        F, best = r[f"p{p}_F"], r[f"p{p}_best"]
        assert F.shape == (p, NBB.S) and np.all(best >= r["p1_best"])
        assert np.max(np.abs(r[f"sk_p{p}_F"] - F) / (np.abs(F) + ys)) < 1e-9
        assert np.max(np.abs(r[f"sk_p{p}_best"] - best) / (np.abs(best) + ys)) < 1e-10
        assert np.max(np.abs(r[f"sk_p{p}_sd0"] - r[f"p{p}_sd0"]) / r[f"p{p}_sd0"]) < 1e-6
        nei = r[f"p{p}_nei"]
        assert np.max(np.abs(r[f"sk_p{p}_nei"] - nei)) < 1e-8 * np.max(nei)
