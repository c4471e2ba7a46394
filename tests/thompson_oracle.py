"""numpy restatement of the posterior sample paths behind Thompson sampling.  TEST INFRASTRUCTURE ONLY.

The device computes (csrc/paths.cuh, bayesianoptimization_b200/paths.py), in the GP's normalised target units:

    phi_l(xs) = sqrt(2c/L) cos(omega_l . xs + b_l)                 xs = transform(x) / length_scale
    r         = y_norm - Phi(Xs) w - eps                             (n x q)
    v         = K^-1 r                                               K = c k(Xs, Xs) + (alpha + noise_level) I
    path(x)   = s_y (Phi(xs) w + c k(xs, Xs) v) + y_mean

(pathwise conditioning: Wilson, Borovitskiy, Terenin, Mostowsky, Deisenroth, "Efficiently sampling functions from
Gaussian process posteriors", ICML 2020, eq. (13) with random Fourier features for the prior term, Rahimi & Recht,
NIPS 2007).  Here the same formulas are evaluated with scipy's Cholesky solve and the kernels of
oracle/gp_oracle.py, which follows SK/gaussian_process/kernels.py.  The draws are restated too, so a test can
check the product's draw helper against them.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_solve, cholesky

from oracle.gp_oracle import KIND_MATERN, KIND_RBF, kernel_cross, kernel_train  # noqa: F401


def draws(rs, q, L, d, nu, n, noise_var):
    """The draws of q paths with L features from RandomState ``rs``, in this order: z (L,d) standard normal;
    for a Matern kernel of finite nu u = chisquare(2 nu, L) and omega = z sqrt(2 nu / u) - the spectral measure of
    the unit-length-scale Matern is a multivariate t with 2 nu degrees of freedom (Rasmussen & Williams 2006,
    eq. 4.15) - else omega = z (RBF: standard normal); b uniform(0, 2 pi, L); w (L,q) standard normal; eps (n,q)
    standard normal times sqrt(alpha + noise_level)."""
    z = rs.standard_normal((L, d))
    if nu == np.inf:
        omega = z
    else:
        u = rs.chisquare(2 * nu, L)
        omega = z * np.sqrt(2 * nu / u)[:, None]
    b = rs.uniform(0, 2 * np.pi, L)
    w = rs.standard_normal((L, q))
    eps = rs.standard_normal((n, q)) * np.sqrt(noise_var)
    return omega, b, w, eps


def features(Xs, omega, b, const):
    return np.sqrt(2.0 * const / omega.shape[0]) * np.cos(Xs @ omega.T + b)


def path_values(X, y, Xq, dr, **kw):
    """(M, q) values of the q paths defined by the draws ``dr`` at the rows of Xq.  X, Xq: inputs after the
    kernel's input transform (np.round for int parameters, the one-hot of categorical ones)."""
    return make_paths(X, y, dr, **kw)(Xq)


def make_paths(X, y, dr, *, kind=KIND_MATERN, nu=2.5, length_scale=1.0, const=1.0, alpha=1e-6, noise_level=0.0,
               normalize=True):
    """The paths as a function Xq -> (M, q) (v solved once)."""
    X = np.asarray(X, dtype=float)
    y = np.asarray(y, dtype=float)
    if normalize:
        m, s = float(np.mean(y)), float(np.std(y))
        s = 1.0 if s == 0.0 else s
    else:
        m, s = 0.0, 1.0
    yn = (y - m) / s
    omega, b, w, eps = dr
    ls = np.asarray(length_scale, dtype=float)
    K = kernel_train(X, kind=kind, nu=nu, length_scale=length_scale, const=const)
    K[np.diag_indices_from(K)] += alpha + noise_level
    r = yn[:, None] - features(X / ls, omega, b, const) @ w - eps
    v = cho_solve((cholesky(K, lower=True), True), r)

    def paths(Xq):
        Xq = np.atleast_2d(np.asarray(Xq, dtype=float))
        f = features(Xq / ls, omega, b, const) @ w + kernel_cross(Xq, X, kind=kind, nu=nu,
                                                                   length_scale=length_scale, const=const) @ v
        return s * f + m

    return paths
