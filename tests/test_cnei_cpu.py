"""Constrained noisy expected improvement without a GPU: the numpy restatement (tests/cnei_oracle.py) against independent
sklearn regressors, its identities, the incumbent rule with its floor, the RNG order and the new exports."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest
from scipy.special import ndtr
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import ConstantKernel, Matern

import cnei_oracle as CO
import logei_oracle as LO
import nei_oracle as NO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = 1e-6


def _case(n=14, d=2, J=2, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    kern = [ConstantKernel(1.3) * Matern(length_scale=0.4, nu=2.5)] + \
           [ConstantKernel(0.8 + 0.3 * j) * Matern(length_scale=0.5 + 0.1 * j, nu=1.5) for j in range(J)]
    y = np.sin(3 * X.sum(1)) + 0.2 * rs.randn(n)
    cy = [np.cos(2 * X[:, 0] + j) + 0.2 * rs.randn(n) for j in range(J)]
    Xc = rs.uniform(size=(30, d))
    return X, Xc, kern, y, cy


def _all_fantasies(X, kern, ys, s2s, S, seed, mask=None):
    draws = CO.draws(np.random.RandomState(seed), X.shape[0], S, len(ys) - 1)
    out = []
    for k, y, s2, (Z, E) in zip(kern, ys, s2s, draws):
        F, A, best = NO.fantasies(k(X), y, s2, TAU, Z, E, np.ones(len(y), bool) if mask is None else mask)
        out.append((F, A, best))
    return out


def test_per_sample_terms_match_independent_regressors():
    """mu_js and sigma0_j of each sample from an sklearn regressor fitted to that sample's fantasy values with the
    kernel fixed and alpha = tau; the term from their predictions."""
    X, Xc, kern, y, cy = _case()
    S, xi = 3, 0.01
    lb, ub = [-np.inf, -0.5], [0.3, 0.6]
    fant = _all_fantasies(X, kern, [y, *cy], [0.05, 0.04, 0.03], S, seed=1)
    ok = CO.eligible(np.ones(len(y), bool), [f[0] for f in fant[1:]], lb, ub)
    best = CO.incumbents(fant[0][0], ok)
    terms = np.zeros((len(Xc), S))
    for s in range(S):
        preds = []
        for k, (F, _, _) in zip(kern, fant):
            gpr = GaussianProcessRegressor(kernel=k, alpha=TAU, optimizer=None, normalize_y=False).fit(X, F[:, s])
            preds.append(gpr.predict(Xc, return_std=True))
        mu, sd = preds[0]
        t = NO.ei(mu - best[s] - xi, sd)
        for j, (mj, sj) in enumerate(preds[1:]):
            t = t * (ndtr((ub[j] - mj) / sj) - (0.0 if lb[j] == -np.inf else ndtr((lb[j] - mj) / sj)))
        terms[:, s] = t
    Ks = [k(Xc, X) for k in kern]
    sds = [NO.noiseless_sd(k(X), TAU, K, k.k1.constant_value) for k, K in zip(kern, Ks)]
    v = CO.cnei(Ks[0], fant[0][1], best, sds[0], xi, Ks[1:], [f[1] for f in fant[1:]], sds[1:], lb, ub)
    np.testing.assert_allclose(v, terms.mean(axis=1), rtol=1e-10, atol=1e-14)
    lv = CO.cnei(Ks[0], fant[0][1], best, sds[0], xi, Ks[1:], [f[1] for f in fant[1:]], sds[1:], lb, ub, log=True)
    pos = v > 1e-250
    np.testing.assert_allclose(lv[pos], np.log(v[pos]), rtol=1e-9, atol=1e-12)


def test_noiseless_constraints_give_nei_times_pof():
    """sigma_n^2 = tau on every constraint GP: F_j = the observed values, P_js = p_j, the eligible rows = the mask."""
    X, Xc, kern, y, cy = _case()
    S, xi = 4, 0.0
    lb, ub = [-0.5, -np.inf], [0.6, 0.2]
    fant = _all_fantasies(X, kern, [y, *cy], [0.05, TAU, TAU], S, seed=2)
    for j in range(2):
        assert np.array_equal(fant[1 + j][0], np.repeat(cy[j][:, None], S, axis=1))
    mask = np.all([(lb[j] <= cy[j]) & (cy[j] <= ub[j]) for j in range(2)], axis=0)
    assert mask.any()
    ok = CO.eligible(np.ones(len(y), bool), [f[0] for f in fant[1:]], lb, ub)
    assert np.array_equal(ok, np.repeat(mask[:, None], S, axis=1))
    best = CO.incumbents(fant[0][0], ok)
    _, _, best_nei = NO.fantasies(kern[0](X), y, 0.05, TAU, *NO.draws(np.random.RandomState(2), len(y), S), mask)
    np.testing.assert_array_equal(best, best_nei)
    Ks = [k(Xc, X) for k in kern]
    sds = [NO.noiseless_sd(k(X), TAU, K, k.k1.constant_value) for k, K in zip(kern, Ks)]
    v = CO.cnei(Ks[0], fant[0][1], best, sds[0], xi, Ks[1:], [f[1] for f in fant[1:]], sds[1:], lb, ub)
    p = np.ones(len(Xc))
    lp = np.zeros(len(Xc))
    for j in range(2):
        mj = Ks[1 + j] @ np.linalg.solve(kern[1 + j](X) + TAU * np.eye(len(y)), cy[j])
        p = p * CO.factor(mj, sds[1 + j], lb[j], ub[j])
        lp = lp + LO.log_cfactor(lb[j], ub[j], mj, sds[1 + j])
    nei = NO.nei(Ks[0], fant[0][1], best, sds[0], xi)
    np.testing.assert_allclose(v, nei * p, rtol=1e-9, atol=1e-14)
    lv = CO.cnei(Ks[0], fant[0][1], best, sds[0], xi, Ks[1:], [f[1] for f in fant[1:]], sds[1:], lb, ub, log=True)
    np.testing.assert_allclose(lv, NO.nei(Ks[0], fant[0][1], best, sds[0], xi, log=True) + lp, rtol=1e-9, atol=1e-12)
    # the target noiseless too: EI x prod p
    fant0 = _all_fantasies(X, kern, [y, *cy], [TAU, TAU, TAU], S, seed=3)
    best0 = CO.incumbents(fant0[0][0], ok)
    assert np.all(best0 == y[mask].max())
    v0 = CO.cnei(Ks[0], fant0[0][1], best0, sds[0], xi, Ks[1:], [f[1] for f in fant0[1:]], sds[1:], lb, ub)
    mu = Ks[0] @ np.linalg.solve(kern[0](X) + TAU * np.eye(len(y)), y)
    np.testing.assert_allclose(v0, NO.ei(mu - y[mask].max() - xi, sds[0]) * p, rtol=1e-9, atol=1e-14)


def test_no_constraint_is_nei():
    X, Xc, kern, y, _ = _case(J=0)
    fant = _all_fantasies(X, kern, [y], [0.05], 5, seed=4)
    F, A, best = fant[0]
    assert np.array_equal(CO.incumbents(F, CO.eligible(np.ones(len(y), bool), [], [], [])), best)
    Ks = kern[0](Xc, X)
    sd = NO.noiseless_sd(kern[0](X), TAU, Ks, 1.3)
    for log in (False, True):
        np.testing.assert_array_equal(CO.cnei(Ks, A, best, sd, 0.01, [], [], [], [], [], log=log),
                                      NO.nei(Ks, A, best, sd, 0.01, log=log))


def test_incumbent_floor_and_bounds_part_of_the_mask():
    rs = np.random.RandomState(5)
    F = rs.standard_normal((6, 4))
    Fc = [rs.standard_normal((6, 4))]
    in_bounds = np.array([True, True, False, True, True, True])
    ok = CO.eligible(in_bounds, Fc, [-0.5], [0.5])
    assert not ok[2].any()  # outside the bounds: never eligible, whatever the constraint fantasy says
    np.testing.assert_array_equal(ok, in_bounds[:, None] & (np.abs(Fc[0]) <= 0.5))
    ok[:, 1] = False  # sample 1: no eligible row -> the smallest value over all rows
    best = CO.incumbents(F, ok)
    assert best[1] == F[:, 1].min()
    for s in (0, 2, 3):
        if ok[:, s].any():
            assert best[s] == F[ok[:, s], s].max()
        else:
            assert best[s] == F[:, s].min()


def test_rng_order_target_then_each_constraint():
    rs = np.random.RandomState(7)
    d = CO.draws(rs, 5, 3, 2)
    rs2 = np.random.RandomState(7)
    for Z, E in d:
        assert np.array_equal(Z, rs2.standard_normal((5, 3)))
        assert np.array_equal(E, rs2.standard_normal((5, 3)))
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)


def test_new_constants_and_export():
    from bayesianoptimization_b200 import _lib as B

    assert (B.ACQ_CNEI, B.ACQ_LOGCNEI) == (10, 11)
    assert "b200bo_gp_set_fantasy_incumbent" in B.EXPORTS
    with open(os.path.join(ROOT, "include", "b200bo.h")) as f:
        h = f.read()
    assert "#define B200BO_ACQ_CNEI 10" in h and "#define B200BO_ACQ_LOGCNEI 11" in h
    assert "int b200bo_gp_set_fantasy_incumbent(" in h
    if not os.path.exists(B.LIB_PATH):
        pytest.skip("library not built")
    assert hasattr(C.CDLL(B.LIB_PATH), "b200bo_gp_set_fantasy_incumbent")


def test_cnei_parameters_round_trip_and_refusals(ref):
    import bayesianoptimization_b200 as bo

    a = bo.ConstrainedNoisyExpectedImprovement(xi=0.02, n_samples=5, jitter=1e-5)
    p = a.get_acquisition_params()
    assert p == bo.NoisyExpectedImprovement(xi=0.02, n_samples=5, jitter=1e-5).get_acquisition_params()
    b = bo.LogConstrainedNoisyExpectedImprovement(xi=0.0)
    b.set_acquisition_params(p)
    assert (b.n_samples, b.jitter, b.xi) == (5, 1e-5, 0.02)
    with pytest.raises(ValueError):
        bo.ConstrainedNoisyExpectedImprovement(xi=0.0, n_samples=17)
    with pytest.raises(ValueError):
        bo.LogConstrainedNoisyExpectedImprovement(xi=0.0, jitter=-1.0)
    with pytest.raises(NotImplementedError):
        a.base_acq(np.zeros(1), np.ones(1))
    for wrap in (lambda x: bo.KrigingBeliever(x), lambda x: bo.ConstantLiar(x), lambda x: bo.GPHedge([x])):
        with pytest.raises(TypeError):
            wrap(bo.ConstrainedNoisyExpectedImprovement(xi=0.0))
    bo.PendingNEI(bo.LogConstrainedNoisyExpectedImprovement(xi=0.0))  # accepted as a base
    assert isinstance(a, bo.AcquisitionFunction) and isinstance(a, ref.acquisition.ExpectedImprovement)


def test_cnei_refuses_too_many_constraints_before_any_draw(ref):
    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200.acquisition import _SuggestStream

    class _Con:
        model = [bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5)) for _ in range(8)]

    a = bo.ConstrainedNoisyExpectedImprovement(xi=0.0)
    rs = np.random.RandomState(0)
    state = rs.get_state()[1].copy()
    a._path_rng, a._suggest_space = rs, object()
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5))
    with pytest.raises(NotImplementedError):
        a._get_acq(gp, _Con())
    assert np.array_equal(rs.get_state()[1], state)
    assert issubclass(type(a), _SuggestStream)


def test_product_eligibility_is_the_restatement(ref):
    """The class's mask (acquisition.cnei_eligible over acquisition._in_bounds) against tests/cnei_oracle.py, with rows
    outside the bounds and a constraint fantasy exactly on a bound."""
    from bayesianoptimization_b200.acquisition import _in_bounds, cnei_eligible

    rs = np.random.RandomState(9)
    params = rs.uniform(-1.0, 1.0, size=(8, 2))
    params[[1, 5], 1] = 1.5
    space = type("Space", (), {"params": params, "bounds": np.array([[-1.0, 1.0], [-1.0, 1.0]])})()
    inb = _in_bounds(space)
    np.testing.assert_array_equal(inb, np.all(np.abs(params) <= 1.0, axis=1))
    Fc = [rs.standard_normal((8, 3)), rs.standard_normal((8, 3))]
    Fc[0][2, 1] = 0.4  # on the upper bound: feasible
    lb, ub = np.array([-np.inf, -1.0]), np.array([0.4, 1.0])
    got = cnei_eligible(inb, Fc, lb, ub)
    np.testing.assert_array_equal(got, CO.eligible(inb, Fc, lb, ub))
    assert not got[[1, 5]].any() and got[2, 1] == (abs(Fc[1][2, 1]) <= 1.0)
