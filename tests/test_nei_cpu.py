"""Noisy expected improvement without a GPU: the numpy restatement (tests/nei_oracle.py) against the analytic posterior,
its reductions, the RNG order of noiseless_fantasies and the new exports of the built library."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import ConstantKernel, Matern

import nei_oracle as NO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(n=12, d=2, c=1.3, s2=0.05, tau=1e-6, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    k = ConstantKernel(c) * Matern(length_scale=0.4, nu=2.5)
    Kc = k(X)
    y = np.sin(3 * X.sum(1)) + np.sqrt(s2) * rs.randn(n)
    return X, k, Kc, y


def test_fantasies_match_the_analytic_posterior():
    """f_s = Matheron's rule: the columns are samples of the latent values given y under noise s2 - tau."""
    X, k, Kc, y = _case()
    s2, tau, S = 0.05, 1e-6, 20000
    Z, E = NO.draws(np.random.RandomState(1), len(y), S)
    F, _, _ = NO.fantasies(Kc, y, s2, tau, Z, E, np.ones(len(y), bool))
    K0 = Kc + tau * np.eye(len(y))
    K = Kc + s2 * np.eye(len(y))
    mean = K0 @ np.linalg.solve(K, y)
    cov = K0 - K0 @ np.linalg.solve(K, K0)
    emp_mean = F.mean(axis=1)
    emp_cov = np.cov(F)
    sd = np.sqrt(np.diag(cov))
    assert np.all(np.abs(emp_mean - mean) < 5 * sd / np.sqrt(S))
    # covariance entries: standard error of a sample covariance ~ sqrt((cov_ii cov_jj + cov_ij^2) / S)
    se = np.sqrt((np.outer(np.diag(cov), np.diag(cov)) + cov * cov) / S)
    assert np.all(np.abs(emp_cov - cov) < 6 * se)


def test_noise_equal_tau_gives_y_and_ei():
    X, k, Kc, y = _case()
    tau = 1e-6
    Z, E = NO.draws(np.random.RandomState(2), len(y), 4)
    mask = np.ones(len(y), bool)
    F, A, best = NO.fantasies(Kc, y, tau, tau, Z, E, mask)
    assert np.array_equal(F, np.repeat(y[:, None], 4, axis=1))
    assert np.all(best == y.max())
    Xc = np.random.RandomState(3).uniform(size=(50, 2))
    Ks = k(Xc, X)
    sd = NO.noiseless_sd(Kc, tau, Ks, 1.3)
    alpha = np.linalg.solve(Kc + tau * np.eye(len(y)), y)
    ei = NO.ei(Ks @ alpha - y.max() - 0.01, sd)
    np.testing.assert_allclose(NO.nei(Ks, A, best, sd, 0.01), ei, rtol=1e-9, atol=1e-12)


def test_log_nei_is_log_of_nei_and_finite_in_the_tail():
    X, k, Kc, y = _case()
    Z, E = NO.draws(np.random.RandomState(4), len(y), 8)
    F, A, best = NO.fantasies(Kc, y, 0.05, 1e-6, Z, E, np.ones(len(y), bool))
    rs = np.random.RandomState(5)
    Xc = np.vstack([rs.uniform(size=(40, 2)), X[:3] + 1e-7])
    Ks = k(Xc, X)
    sd = NO.noiseless_sd(Kc, 1e-6, Ks, 1.3)
    v = NO.nei(Ks, A, best, sd, 0.0)
    lv = NO.nei(Ks, A, best, sd, 0.0, log=True)
    ok = v > 1e-250
    np.testing.assert_allclose(lv[ok], np.log(v[ok]), rtol=1e-9, atol=1e-12)
    # far below every incumbent: NEI underflows to 0, LogNEI stays finite and ordered
    far = NO.nei(Ks, A, best + 60.0, sd, 0.0, log=True)
    assert np.all(np.isfinite(far))
    assert np.all(NO.nei(Ks, A, best + 60.0, sd, 0.0)[sd > 0.05] == 0.0)


def test_logmeanexp_rules():
    ls = np.array([[-np.inf, -np.inf], [np.nan, 0.0], [-1e6, -1e6 - 1.0]])
    out = NO.logmeanexp(ls)
    assert out[0] == -np.inf and np.isnan(out[1])
    np.testing.assert_allclose(out[2], -1e6 + np.log((1 + np.exp(-1.0)) / 2), rtol=1e-15)


def test_rng_order_is_z_then_e():
    rs = np.random.RandomState(7)
    Z, E = NO.draws(rs, 5, 3)
    rs2 = np.random.RandomState(7)
    assert np.array_equal(Z, rs2.standard_normal((5, 3)))
    assert np.array_equal(E, rs2.standard_normal((5, 3)))
    assert rs.randint(1 << 30) == rs2.randint(1 << 30)


def test_new_exports_in_the_library():
    from bayesianoptimization_b200 import _lib as B

    if not os.path.exists(B.LIB_PATH):
        pytest.skip("library not built")
    L = C.CDLL(B.LIB_PATH)
    assert hasattr(L, "b200bo_gp_set_fantasies")
    assert "b200bo_gp_set_fantasies" in B.EXPORTS
    assert (B.ACQ_NEI, B.ACQ_LOGNEI) == (8, 9)
    with open(os.path.join(ROOT, "include", "b200bo.h")) as f:
        h = f.read()
    assert "#define B200BO_ACQ_NEI 8" in h and "#define B200BO_ACQ_LOGNEI 9" in h


def test_nei_parameters_round_trip(ref):
    import bayesianoptimization_b200 as bo

    a = bo.NoisyExpectedImprovement(xi=0.02, n_samples=5, jitter=1e-5)
    p = a.get_acquisition_params()
    assert p["n_samples"] == 5 and p["jitter"] == 1e-5 and p["xi"] == 0.02
    b = bo.LogNoisyExpectedImprovement(xi=0.0)
    b.set_acquisition_params(p)
    assert (b.n_samples, b.jitter, b.xi) == (5, 1e-5, 0.02)
    with pytest.raises(ValueError):
        bo.NoisyExpectedImprovement(xi=0.0, n_samples=17)
    with pytest.raises(ValueError):
        bo.NoisyExpectedImprovement(xi=0.0, jitter=0.0)
    with pytest.raises(NotImplementedError):
        a.base_acq(np.zeros(1), np.ones(1))
    for wrap in (lambda x: bo.KrigingBeliever(x), lambda x: bo.ConstantLiar(x), lambda x: bo.GPHedge([x])):
        with pytest.raises(TypeError):
            wrap(bo.NoisyExpectedImprovement(xi=0.0))
    assert isinstance(a, bo.AcquisitionFunction) and isinstance(a, ref.acquisition.ExpectedImprovement)


def test_reference_wrappers_refuse_nei_through_enable(ref):
    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200.acquisition import accelerate

    wrappers = (ref.acquisition.ConstantLiar(bo.NoisyExpectedImprovement(xi=0.0)),
                ref.acquisition.GPHedge([ref.acquisition.ExpectedImprovement(xi=0.0),
                                         bo.LogNoisyExpectedImprovement(xi=0.0)]))
    for w in wrappers:
        with pytest.raises(TypeError):
            accelerate(w)
