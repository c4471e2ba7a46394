"""numpy restatement of a GP conditioned on pending points with Kriging-believer targets (DESIGN.md 4.11).

``conditioned_posterior`` refits nothing: it takes a fitted sklearn GaussianProcessRegressor (its kernel_, alpha,
X_train_, y_train_, alpha_ and y statistics), appends the pending rows P with the targets mu_norm(P) = k(P, X) alpha_,
and solves the augmented system by a fresh Cholesky factorisation.  ``closed_form`` is the same posterior from the
original GP's joint predictive covariance (the Schur complement): sigma_f^2 = sigma^2 - S(x,P) (S(P,P) + s_n^2 I)^-1
S(P,x) with s_n^2 = alpha * y_std^2, and mu_f = mu.  tests/test_kriging_believer_cpu.py pins the two against each
other; the device tests compare the device against ``closed_form``.
"""
import numpy as np
from scipy.linalg import cho_solve, cholesky, solve_triangular


def _ystats(gp):
    return float(np.ravel(gp._y_train_mean)[0]), float(np.ravel(gp._y_train_std)[0])


def believer_targets(gp, P):
    """mu_norm(P) = k(P, X) alpha_ (normalised units) of a fitted sklearn GP."""
    return gp.kernel_(np.atleast_2d(P), gp.X_train_) @ gp.alpha_


def conditioned_posterior(gp, P, Xq):
    """(mu, sd, alpha_aug) at the rows of Xq of ``gp`` conditioned on the rows of P; mu, sd in data units."""
    P = np.atleast_2d(np.asarray(P, dtype=np.float64))
    ym, ys = _ystats(gp)
    Xa = np.vstack([gp.X_train_, P])
    ya = np.concatenate([gp.y_train_, believer_targets(gp, P)])
    K = gp.kernel_(Xa)
    K[np.diag_indices_from(K)] += gp.alpha
    L = cholesky(K, lower=True)
    a = cho_solve((L, True), ya)
    Ks = gp.kernel_(Xq, Xa)
    mu = Ks @ a * ys + ym
    V = solve_triangular(L, Ks.T, lower=True)
    var = gp.kernel_.diag(Xq) - np.einsum("ij,ij->j", V, V)
    return mu, np.sqrt(np.maximum(var, 0.0)) * ys, a


def closed_form(gp, P, Xq):
    """(mu, sd) of the conditioned GP from the original GP's predict(return_cov=True) on [Xq; P]."""
    P = np.atleast_2d(np.asarray(P, dtype=np.float64))
    m = Xq.shape[0]
    _, ys = _ystats(gp)
    mu_all, cov = gp.predict(np.vstack([Xq, P]), return_cov=True)
    S_xx = np.diag(cov)[:m]
    S_xp, S_pp = cov[:m, m:], cov[m:, m:] + gp.alpha * ys * ys * np.eye(P.shape[0])
    Lp = cholesky(S_pp, lower=True)
    W = solve_triangular(Lp, S_xp.T, lower=True)
    var = S_xx - np.einsum("ij,ij->j", W, W)
    return mu_all[:m], np.sqrt(np.maximum(var, 0.0))
