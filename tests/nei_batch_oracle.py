"""numpy restatement of NEI with pending points (include/b200bo.h b200bo_gp_condition_fantasies, DESIGN.md 4.14).

Everything in float64 in the order of the definition: the noiseless factor grows by one row per pending point
(l = L0^-1 k, r = sqrt(c + tau - l^T l)), F_js = l^T [Z_s; z_1s .. z_(j-1)s] + r z_js + k(x_j, X_reg)^T W_s with
W = K^-1 R of the registered rows, A' = K0'^-1 F', and best_s' counts every pending row.  Used by
tests/test_nei_batch_cpu.py and tests/test_gpu_nei_batch.py."""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_factor, cho_solve, cholesky, solve_triangular

import nei_oracle as NO


def draws(rs, n, S, rows):
    """The RandomState consumption of noiseless_fantasies(pending=..., extra_rows=...): Z, E, then the z rows."""
    Z, E = NO.draws(rs, n, S)
    return Z, E, rs.standard_normal((rows, S))


def residual_solve(Kc, y_n, s2, tau, Z, E):
    """W = K^-1 R, R = y_n - L0 Z - sqrt(s2 - tau) E (n, S), the Matheron weights of the registered rows."""
    n = Kc.shape[0]
    L0 = cholesky(Kc + tau * np.eye(n), lower=True)
    R = (y_n[:, None] - L0 @ Z) - np.sqrt(s2 - tau) * E
    return cho_solve(cho_factor(Kc + s2 * np.eye(n), lower=True), R)


def pending_fantasies(kc, X, P, y_n, s2, tau, Z, E, Zp, mask, y_mean=0.0, y_std=1.0):
    """(F', A', best') over X u P: F' (n + p, S) normalised, A' = K0'^-1 F', best' (S,) data units.  kc is the scaled
    kernel c k (an sklearn kernel object); Zp holds at least p rows."""
    Kc = kc(X)
    n, p = X.shape[0], P.shape[0]
    F, _, best = NO.fantasies(Kc, y_n, s2, tau, Z, E, mask, y_mean, y_std)
    W = residual_solve(Kc, y_n, s2, tau, Z, E)
    c0 = float(kc.diag(X[:1])[0])
    L = cholesky(Kc + tau * np.eye(n), lower=True)
    Xa, Za, Fa = X, Z, F
    for j in range(p):
        x = P[j:j + 1]
        k = kc(Xa, x)[:, 0]
        l = solve_triangular(L, k, lower=True)
        r = np.sqrt(c0 + tau - l @ l)
        f = l @ Za + r * Zp[j] + kc(x, X)[0] @ W
        L = np.block([[L, np.zeros((L.shape[0], 1))], [l[None, :], np.array([[r]])]])
        Xa, Za, Fa = np.vstack([Xa, x]), np.vstack([Za, Zp[j:j + 1]]), np.vstack([Fa, f[None, :]])
        best = np.maximum(best, y_std * f + y_mean)
    A = cho_solve((L, True), Fa)
    return Fa, A, best


def grown_sd(kc, Xa, tau, Xc, y_std=1.0):
    """sigma0 (data units) of the noiseless GP over the grown set Xa at the candidates Xc."""
    return NO.noiseless_sd(kc(Xa), tau, kc(Xc, Xa), float(kc.diag(Xc[:1])[0]), y_std)


def nei(kc, Xa, A, best, tau, Xc, xi, y_mean=0.0, y_std=1.0, log=False):
    """NEI (or LogNEI) at the candidates Xc on the grown noiseless GP with (A', best')."""
    return NO.nei(kc(Xc, Xa), A, best, grown_sd(kc, Xa, tau, Xc, y_std), xi, y_mean, y_std, log=log)
