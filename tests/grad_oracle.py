"""Numpy restatement of the analytic input gradients (DESIGN.md 4.10), shared by tests/test_grad_cpu.py (which pins
it against extended-precision central differences) and tests/test_gpu_grad.py (which holds the device to it).

In normalised units, xs = transform(x)/ls, k*_n = c k(|xs - Xs_n|), u = K^-1 k*:
    d k*_n / d x_j = -c h(r_n) (xs_j - Xs_nj) / ls_j,     h(r) = -(1/r) dk/dr   (0 at r = 0 for Matern 1/2)
    d mean / d x_j = s_y sum_n alpha_n d k*_n / d x_j,    d sd / d x_j = -s_y (sum_n u_n d k*_n / d x_j) / sqrt(var)
A rounded dimension has gradient 0; a variance clamped to 0 gives d sd = 0.
"""
import math

import numpy as np
from scipy.linalg import cho_solve, cholesky, solve_triangular
from scipy.spatial.distance import cdist
from scipy.special import erfcx, log_ndtr, ndtr

UCB, EI, POI, MES = 0, 1, 2, 4
_S2PI = math.sqrt(2.0 * math.pi)


def k_of_r(r, nu):
    if nu == 0.5:
        return np.exp(-r)
    if nu == 1.5:
        a = math.sqrt(3) * r
        return (1 + a) * np.exp(-a)
    if nu == 2.5:
        a = math.sqrt(5) * r
        return (1 + a + a * a / 3) * np.exp(-a)
    return np.exp(-0.5 * r * r)


def h_of_r(r, nu):
    if nu == 0.5:
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(r == 0, 0.0, np.exp(-r) / r)
    if nu == 1.5:
        return 3 * np.exp(-math.sqrt(3) * r)
    if nu == 2.5:
        a = math.sqrt(5) * r
        return 5.0 / 3.0 * (1 + a) * np.exp(-a)
    return np.exp(-0.5 * r * r)


def pdf(z):
    return np.exp(-z * z / 2.0) / _S2PI


def inv_mills(g):
    g = np.asarray(g, dtype=float)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        return np.where(g < 0, math.sqrt(2 / math.pi) / erfcx(-g / math.sqrt(2)), pdf(g) / ndtr(g))


class GradGP:
    """A GP at fixed hyper-parameters: covariance c k(r) + noise on the diagonal, jitter alpha, optional rounding of
    the last ``rnd`` input columns, normalised targets."""

    def __init__(self, X, y, nu, ls, const=1.0, noise=0.0, alpha=1e-6, normalize=True, rnd=0):
        X = np.asarray(X, dtype=float)
        n, d = X.shape
        self.nu, self.const, self.noise, self.d, self.rnd = nu, float(const), float(noise), d, rnd
        self.ls = np.broadcast_to(np.asarray(ls, dtype=float), (d,)).copy()
        self.Xs = self.transform(X) / self.ls
        y = np.asarray(y, dtype=float)
        self.y_mean, self.y_std = (float(y.mean()), float(y.std()) or 1.0) if normalize else (0.0, 1.0)
        self.y_norm = (y - self.y_mean) / self.y_std
        r = cdist(self.Xs, self.Xs)  # no (n, n, d) temporary: N = 8192, d = 32 would need 17 GB
        K = self.const * k_of_r(r, nu)
        K[np.diag_indices(n)] = self.const + self.noise + alpha
        self.K = K
        self.L = cholesky(K, lower=True)
        self.alpha_ = cho_solve((self.L, True), self.y_norm)
        self.prior = self.const + self.noise

    def transform(self, x):
        x = np.array(x, dtype=float, copy=True).reshape(-1, self.d)
        if self.rnd:
            x[:, self.d - self.rnd:] = np.round(x[:, self.d - self.rnd:])
        return x

    def predict_grad(self, x):
        """mean (m,), sd (m,), d mean (m,d), d sd (m,d) in data units."""
        xs = self.transform(x) / self.ls
        diff = xs[:, None, :] - self.Xs[None, :, :]                    # (m, n, d)
        r = np.sqrt((diff ** 2).sum(-1))
        ks = self.const * k_of_r(r, self.nu)                           # (m, n)
        dks = -(self.const * h_of_r(r, self.nu))[:, :, None] * diff / self.ls  # (m, n, d)
        if self.rnd:
            dks[:, :, self.d - self.rnd:] = 0.0
        V = solve_triangular(self.L, ks.T, lower=True)                 # (n, m)
        U = solve_triangular(self.L.T, V, lower=False)                 # K^-1 k*
        var = self.prior - (V * V).sum(0)
        clamped = var <= 0
        var = np.where(clamped, 0.0, var)
        mean = self.y_std * (ks @ self.alpha_) + self.y_mean
        sd = np.sqrt(var * self.y_std ** 2)
        dmean = self.y_std * np.einsum("n,mnj->mj", self.alpha_, dks)
        with np.errstate(divide="ignore", invalid="ignore"):
            dsd = -self.y_std * np.einsum("nm,mnj->mj", U, dks) / np.sqrt(var)[:, None]
        dsd[clamped] = 0.0
        return mean, sd, dmean, dsd


def base_value_grad(kind, mean, sd, dmean, dsd, kappa=2.576, xi=0.0, y_max=0.0, ystar=None):
    """(base (m,), d base (m,d)) of the un-negated base acquisition."""
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == UCB:
            return mean + kappa * sd, dmean + kappa * dsd
        a = mean - y_max - xi
        z = a / sd
        pos = sd > 0
        if kind == EI:
            return a * ndtr(z) + sd * pdf(z), ndtr(z)[:, None] * dmean + pdf(z)[:, None] * dsd
        if kind == POI:
            cm = np.where(pos, pdf(z) / sd, 0.0)
            cs = np.where(pos & (pdf(z) != 0), -z * pdf(z) / sd, 0.0)
            return ndtr(z), cm[:, None] * dmean + cs[:, None] * dsd
        if kind == MES:
            ystar = np.asarray(ystar, dtype=float)
            g = (ystar[None, :] - mean[:, None]) / sd[:, None]        # (m, K)
            lam = inv_mills(g)
            t = np.where(lam == 0, 0.0, 0.5 * g * lam) - log_ndtr(g)
            td = np.where(lam == 0, 0.0, -0.5 * lam - 0.5 * g * lam * (g + lam))
            base = np.where(pos, t.mean(1), 0.0)
            cm = np.where(pos, -td.sum(1) / (len(ystar) * sd), 0.0)
            cs = np.where(pos, -np.where(td == 0, 0.0, td * g).sum(1) / (len(ystar) * sd), 0.0)
            return base, cm[:, None] * dmean + cs[:, None] * dsd
    raise ValueError(kind)


def prob_value_grad(lb, ub, mean, sd, dmean, dsd):
    """(p (m,), d p (m,d)) of p = Phi((ub - mean)/sd) - Phi((lb - mean)/sd); an infinite bound contributes 0 to d p;
    sd == 0 gives NaN like scipy's frozen norm."""
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(sd > 0, (1.0 if ub == np.inf else ndtr((ub - mean) / sd)) -
                     (0.0 if lb == -np.inf else ndtr((lb - mean) / sd)), np.nan)
        dp = np.zeros_like(dmean)
        if lb != -np.inf:
            z = (lb - mean) / sd
            dp += (pdf(z) / sd)[:, None] * (dmean + z[:, None] * dsd)
        if ub != np.inf:
            z = (ub - mean) / sd
            dp -= (pdf(z) / sd)[:, None] * (dmean + z[:, None] * dsd)
    return p, dp


def acq_value_grad(kind, target, x, constraints=(), **params):
    """(val (m,), grad (m,d)) of the closure value -base * prod_j p_j; constraints: [(GradGP, lb, ub)].
    A NaN value gives a NaN gradient row."""
    x = np.asarray(x, dtype=float).reshape(-1, target.d)
    base, dbase = base_value_grad(kind, *target.predict_grad(x), **params)
    terms = [(base, dbase)] + [prob_value_grad(lb, ub, *gp.predict_grad(x)) for gp, lb, ub in constraints]
    val = -np.prod([t for t, _ in terms], axis=0) if len(terms) > 1 else -base
    grad = np.zeros_like(dbase)
    for g, (_, dt) in enumerate(terms):
        w = -np.prod([t for i, (t, _) in enumerate(terms) if i != g], axis=0) if len(terms) > 1 else -np.ones(len(x))
        grad += w[:, None] * dt
    grad[np.isnan(val)] = np.nan
    return val, grad


def path_value_grad(gp, omega, bias, w, v, x):
    """(val (m,), grad (m,d)) of one sample path (DESIGN.md 4.7) with feature weights w (L,) and update weights v (n,):
    path(x) = s_y (sqrt(2c/L) sum_l w_l cos(omega_l . xs + b_l) + sum_i v_i c k(|xs - Xs_i|)) + y_mean."""
    xs = gp.transform(x) / gp.ls
    fs = math.sqrt(2.0 * gp.const / len(w))
    ph = xs @ omega.T + bias                                          # (m, L)
    diff = xs[:, None, :] - gp.Xs[None, :, :]
    r = np.sqrt((diff ** 2).sum(-1))
    val = gp.y_std * (fs * (np.cos(ph) @ w) + gp.const * (k_of_r(r, gp.nu) @ v)) + gp.y_mean
    g = -fs * ((np.sin(ph) * w) @ omega) - gp.const * np.einsum("mn,mnj->mj", h_of_r(r, gp.nu) * v, diff)
    g = gp.y_std * g / gp.ls
    if gp.rnd:
        g[:, gp.d - gp.rnd:] = 0.0
    return val, g
