"""numpy/scipy statement of max-value entropy search (MES).  TEST INFRASTRUCTURE ONLY.

Wang & Jegelka, "Max-value Entropy Search for Efficient Bayesian Optimization", ICML 2017, eq. (6), in data units:

    g_k(x)  = (y*_k - mu(x)) / sigma(x)
    alpha(x) = (1/K) sum_{k=0..K-1}, in k order, [ g_k psi(g_k) / (2 Psi(g_k)) - log Psi(g_k) ]
    closure  = -alpha(x) [* prod_j p_j(x)]

psi, Psi: standard normal pdf and cdf; alpha = 0 where sigma = 0.  log Psi is scipy.special.log_ndtr and
psi / Psi = exp(norm.logpdf(g) - log_ndtr(g)), both finite for every finite g.
"""
from __future__ import annotations

import numpy as np
from scipy.special import log_ndtr
from scipy.stats import norm


def mes_term(g):
    """g psi(g) / (2 Psi(g)) - log Psi(g), elementwise."""
    g = np.asarray(g, dtype=np.float64)
    ln = log_ndtr(g)
    return g * np.exp(norm.logpdf(g) - ln) / 2.0 - ln


def mp_mes_term(g, dps=50):
    """(g psi(g) / (2 Psi(g)) - log Psi(g), its derivative in g) at `dps` digits (mpmath) for an fp64 or mpmath g:
    with lambda = psi / Psi, d lambda / dg = -lambda (g + lambda), the derivative is -lambda/2 - g lambda (g + lambda)/2."""
    import mpmath as mp

    with mp.workdps(dps):
        g = mp.mpf(g)
        P = mp.ncdf(g)
        lam = mp.npdf(g) / P
        return g * lam / 2 - mp.log(P), -lam / 2 - g * lam * (g + lam) / 2


def mes_alpha(mu, sd, ystar):
    mu = np.asarray(mu, dtype=np.float64)
    sd = np.asarray(sd, dtype=np.float64)
    out = np.zeros(np.broadcast(mu, sd).shape)
    pos = sd > 0
    mu_p, sd_p = np.broadcast_to(mu, out.shape)[pos], np.broadcast_to(sd, out.shape)[pos]
    acc = np.zeros(mu_p.shape)
    for y in np.asarray(ystar, dtype=np.float64).reshape(-1):
        acc = acc + mes_term((y - mu_p) / sd_p)
    out[pos] = acc / len(np.asarray(ystar).reshape(-1))
    return out


def mes_closure(mu, sd, ystar, prod=None):
    a = mes_alpha(mu, sd, ystar)
    return -1 * a if prod is None else -1 * a * prod
