"""numpy restatement of noisy expected improvement (include/b200bo.h B200BO_ACQ_NEI / LOGNEI, DESIGN.md 4.13).

Everything in float64 with numpy / scipy factorisations, in the order of the definition; used by tests/test_nei_cpu.py
and tests/test_gpu_nei.py to hold the device to the same numbers."""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_factor, cho_solve, cholesky, solve_triangular
from scipy.special import ndtr

import logei_oracle as LO


def draws(rs, n, S):
    """The RandomState consumption of one suggest(): Z, then E."""
    Z = rs.standard_normal((n, S))
    E = rs.standard_normal((n, S))
    return Z, E


def fantasies(Kc, y_n, s2, tau, Z, E, mask, y_mean=0.0, y_std=1.0):
    """(F, A, best): F (n, S) normalised fantasies, A = K0^-1 F, best (S,) in data units.  Kc = c k(X, X)."""
    n = Kc.shape[0]
    K0 = Kc + tau * np.eye(n)
    K = Kc + s2 * np.eye(n)
    L0 = cholesky(K0, lower=True)
    sq, ds = np.sqrt(s2 - tau), s2 - tau
    Fp = L0 @ Z
    Y = y_n[:, None]
    if ds > 0.0:
        R = (Y - Fp) - sq * E
        F = (Y - sq * E) - ds * cho_solve(cho_factor(K, lower=True), R)
    else:
        F = np.repeat(Y, Z.shape[1], axis=1)
    A = cho_solve(cho_factor(K0, lower=True), F)
    best = (y_std * F[np.asarray(mask, dtype=bool)] + y_mean).max(axis=0)
    return F, A, best


def noiseless_sd(Kc, tau, Ks, c, y_std=1.0):
    """sigma0 (data units) of the noiseless GP at the candidates: Ks = c k(Xc, X) (m, n)."""
    L0 = cholesky(Kc + tau * np.eye(Kc.shape[0]), lower=True)
    V = solve_triangular(L0, Ks.T, lower=True)
    var = np.maximum(c - np.sum(V * V, axis=0), 0.0)
    return np.sqrt(var * y_std * y_std)


def ei(a, sd):
    """The device's EI formula at a = mean - best - xi, with its sigma = 0 limits (a, 0, NaN)."""
    with np.errstate(all="ignore"):
        z = a / sd
        return a * ndtr(z) + sd * np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)


def nei(Ks, A, best, sd, xi, y_mean=0.0, y_std=1.0, log=False):
    """NEI (or LogNEI) per candidate: Ks (m, n), A (n, S), best (S,), sd (m,) data units."""
    mu = y_std * (Ks @ A) + y_mean
    a = mu - best[None, :] - xi
    sd = np.asarray(sd, dtype=np.float64)[:, None]
    if not log:
        return ei(a, sd).mean(axis=1)
    return logmeanexp(_log_ei(a, sd))


def nei_value_grad(gp0, x, A, best, xi, log=False):
    """NEI (or LogNEI) and its input gradient (m, d) at the rows x.  gp0 is a grad_oracle.GradGP of the noiseless GP
    (K0 = c k(X, X) + tau I, the noisy GP's y statistics), A = K0^-1 F (n, S), best (S,) data units.  With
    d mu_s = s_y sum_n A_ns d k*_n / dx and d sd from GradGP.predict_grad, NEI's gradient is the mean over the fantasies
    of EI's, Phi(z_s) d mu_s + phi(z_s) d sd, and LogNEI's is NEI's over NEI."""
    import grad_oracle as GO

    xs = gp0.transform(x) / gp0.ls
    diff = xs[:, None, :] - gp0.Xs[None, :, :]
    r = np.sqrt((diff ** 2).sum(-1))
    ks = gp0.const * GO.k_of_r(r, gp0.nu)
    dks = -(gp0.const * GO.h_of_r(r, gp0.nu))[:, :, None] * diff / gp0.ls
    _, sd, _, dsd = gp0.predict_grad(x)
    mu = gp0.y_std * (ks @ A) + gp0.y_mean
    dmu = gp0.y_std * np.einsum("ns,mnj->msj", A, dks)
    a = mu - best[None, :] - xi
    with np.errstate(all="ignore"):
        z = a / sd[:, None]
        cdf, pdf = ndtr(z), np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)
    v = (a * cdf + sd[:, None] * pdf).mean(axis=1)
    g = (cdf[:, :, None] * dmu + pdf[:, :, None] * dsd[:, None, :]).mean(axis=1)
    if log:
        return np.log(v), g / v[:, None]
    return v, g


def _log_ei(a, sd):
    return LO.log_acq_term(LO.LOGEI, a, sd)


def logmeanexp(ls):
    """M + log sum exp(l - M) - log S per row; -inf when every l is -inf, NaN when any is NaN."""
    ls = np.asarray(ls, dtype=np.float64)
    S = ls.shape[1]
    M = ls.max(axis=1)
    out = np.full(ls.shape[0], -np.inf)
    ok = np.isfinite(M)
    with np.errstate(all="ignore"):
        out[ok] = M[ok] + np.log(np.exp(ls[ok] - M[ok, None]).sum(axis=1)) - np.log(S)
    out[np.isnan(ls).any(axis=1)] = np.nan
    out[M == np.inf] = np.inf
    return out
