"""The bound behind selection-only pruning (DESIGN.md 4.9), restated in numpy and checked against sklearn.

predict_bound_kernel (csrc/predict16.cuh) keys every candidate by v_lb, a lower bound on its closure value -acq built
from the posterior mean and the largest cross-covariance alone:
    var_ub = min(prior, prior - max_i k*_i^2 / K_ii + eps * prior) >= sigma^2
and EI / UCB (as max(mu, mu + kappa sigma)) / PoI (while a < 0) at sigma_ub, lowered by a relative and an absolute
margin (LogEI / LogPoI: the logs of EI / PoI, LogPoI 0 for a >= 0, lowered by 1e-9 |v| + 1e-9).  Candidates whose mean or bound is not finite, or whose a = mu - y_max - xi is within a few ulps of 0, are never
pruned (key 0).  Here: the bound lies below sklearn's exact closure value on small problems, training points and
near-duplicates included, for every acquisition kind and kappa of either sign.
"""
import numpy as np
import pytest
from scipy.stats import norm

import logei_oracle as LO
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

VAR_EPS, REL_MARGIN, ABS_MARGIN = 1e-8, 1e-9, 1e-300  # kPruneVarEps, kPruneRelMargin, kPruneAbsMargin
LOG_ABS_MARGIN = 1e-9  # kPruneLogAbsMargin


def bound_value(kind, mu, kmax, prior, kdiag, y_std, y_max, kappa, xi):
    """v_lb per candidate (data units): mu = posterior mean, kmax = max_i |k(x*, x_i)| (normalised units)."""
    var_ub = np.maximum(0.0, np.minimum(prior, prior - kmax * kmax / kdiag + VAR_EPS * prior))
    sd = np.sqrt(var_ub * y_std * y_std)
    a = mu - y_max - xi
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "ucb":
            base = np.maximum(mu, mu + kappa * sd)
            scale = np.abs(mu) + np.abs(kappa * sd)
        elif kind == "ei":
            z = a / sd
            base = a * norm.cdf(z) + sd * norm.pdf(z)
            scale = np.abs(base)
        elif kind in ("logei", "logpoi"):
            code = LO.LOGEI if kind == "logei" else LO.LOGPOI
            base = np.where((kind == "logpoi") & (a >= 0), 0.0, LO.log_acq_term(code, a, sd))
            scale = np.abs(base) + LOG_ABS_MARGIN / REL_MARGIN
        else:
            base = np.where(a < 0, norm.cdf(a / sd), 1.0)
            scale = np.abs(base)
    return -base - (REL_MARGIN * scale + ABS_MARGIN)


def never_prune(kind, mu, v_lb, y_max, xi):
    a = mu - y_max - xi
    near0 = (kind != "ucb") & (np.abs(a) <= 8 * np.finfo(float).eps * (np.abs(mu) + abs(y_max) + abs(xi)))
    return ~np.isfinite(mu) | ~np.isfinite(v_lb) | near0


def exact_value(kind, mu, sd, y_max, kappa, xi):
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "ucb":
            return -(mu + kappa * sd)
        a = mu - y_max - xi
        z = a / sd
        if kind == "ei":
            return -(a * norm.cdf(z) + sd * norm.pdf(z))
        if kind in ("logei", "logpoi"):
            return -LO.log_acq_term(LO.LOGEI if kind == "logei" else LO.LOGPOI, a, sd)
        return -norm.cdf(z)


KERNELS = {
    "m25": lambda d: Matern(length_scale=0.4, nu=2.5),
    "m05_ard_white": lambda d: ConstantKernel(1.7) * Matern(np.linspace(0.2, 1.0, d), nu=0.5) + WhiteKernel(1e-2),
    "rbf_const": lambda d: ConstantKernel(0.5) * RBF(0.3),
    "m15": lambda d: Matern(length_scale=0.6, nu=1.5),
}


@pytest.mark.parametrize("kname", sorted(KERNELS))
@pytest.mark.parametrize("kind,kappa", [("ei", 0.0), ("poi", 0.0), ("ucb", 2.576), ("ucb", -1.0), ("logei", 0.0),
                                        ("logpoi", 0.0)])
def test_bound_below_sklearn(kname, kind, kappa):
    rs = np.random.RandomState(3)
    n, d, alpha, xi = 120, 4, 1e-6, 0.01
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1)) + 0.05 * rs.randn(n)
    gp = GaussianProcessRegressor(kernel=KERNELS[kname](d), alpha=alpha, normalize_y=True, optimizer=None).fit(X, y)
    x = np.vstack([rs.uniform(size=(4000, d)), X[:20], X[:20] + 1e-7, X[:20] + 1e-3])
    mu, sd = gp.predict(x, return_std=True)
    exact = exact_value(kind, mu, sd, y.max(), kappa, xi)
    kmax = np.max(np.abs(gp.kernel_(x, X)), axis=1)
    kdiag = gp.kernel_(X[:1])[0, 0] + alpha
    prior = gp.kernel_.diag(x[:1])[0]
    lb = bound_value(kind, mu, kmax, prior, kdiag, gp._y_train_std, y.max(), kappa, xi)
    keep = never_prune(kind, mu, lb, y.max(), xi)
    assert np.all(lb[~keep] <= exact[~keep]), (lb - exact)[~keep].max()


def test_never_prune_predicate():
    mu = np.array([1.01, 1.01 + 1e-15, 1.5, np.nan, np.inf, 0.3])
    lb = np.array([-0.1, -0.1, -0.1, -0.1, -0.1, np.nan])
    keep = never_prune("ei", mu, lb, 1.0, 0.01)
    assert keep.tolist() == [True, True, False, True, True, True]
    assert never_prune("ucb", mu, lb, 1.0, 0.01).tolist() == [False, False, False, True, True, True]


def test_zero_sigma_at_a_zero_is_nan():
    """Why a ~ 0 is never pruned: sigma = 0 with a = 0 is the NaN that np.argmin reports first."""
    mu, sd = np.array([0.5]), np.array([0.0])
    assert np.isnan(exact_value("ei", mu, sd, 0.25, 0.0, 0.25))[0]
    assert np.isnan(exact_value("poi", mu, sd, 0.25, 0.0, 0.25))[0]
    assert never_prune("ei", mu, np.array([-1.0]), 0.25, 0.25)[0]
