"""numpy restatement of constrained NEI with pending points (include/b200bo.h b200bo_gp_set_constrained_incumbent,
DESIGN.md 4.16).

Float64 numpy / scipy in the order of the definition, built from tests/nei_batch_oracle.py (the fantasies of each GP over
X u P) and tests/cnei_oracle.py (eligibility, the incumbent rule with its floor, the CNEI value); used by
tests/test_cnei_batch_cpu.py and tests/test_gpu_cnei_batch.py."""
from __future__ import annotations

import numpy as np

import cnei_oracle as CO
import nei_batch_oracle as NB


def draws(rs, n, S, J, rows):
    """The RandomState consumption of one closure: per GP (the target, then constraint 0..J-1) Z, E, then its z rows."""
    return [NB.draws(rs, n, S, rows) for _ in range(J + 1)]


def rows_in_bounds(rows, bounds):
    """(m,) mask of the rows inside the parameter bounds ((d, 2))."""
    b = np.asarray(bounds, dtype=np.float64)
    return np.all((b[:, 0] <= rows) & (rows <= b[:, 1]), axis=1)


def grown(gp, X, P, Z, E, Zp):
    """(F', A') of one GP over X u P: F' (n + p, S) normalised, A' = K0'^-1 F'.  gp: a dict with kc (the scaled kernel
    c k), y_n (normalised targets), s2 (noise variance), tau, y_mean, y_std."""
    F, A, _ = NB.pending_fantasies(gp["kc"], X, P, gp["y_n"], gp["s2"], gp["tau"], Z, E, Zp, np.ones(X.shape[0], bool),
                                   gp["y_mean"], gp["y_std"])
    return F, A


def data_units(F, gp):
    return gp["y_std"] * F + gp["y_mean"]


def incumbents(F_target, Fc, in_bounds, lb, ub):
    """(best', eligible) over X u P from the data-unit fantasies: row i is eligible in sample s when it lies within the
    bounds and every constraint fantasy lies in [lb_j, ub_j]; best_s' the largest eligible target fantasy, or the
    smallest over all rows when none is."""
    ok = CO.eligible(in_bounds, Fc, lb, ub)
    return CO.incumbents(F_target, ok), ok


def cnei(gps, Xa, As, best, Xc, xi, lb, ub, log=False):
    """CNEI (or LogCNEI) at the candidates Xc on the grown noiseless GPs (gps[0] the target) with A'_g and best'."""
    Ks = [g["kc"](Xc, Xa) for g in gps]
    sds = [NB.grown_sd(g["kc"], Xa, g["tau"], Xc, g["y_std"]) for g in gps]
    return CO.cnei(Ks[0], As[0], best, sds[0], xi, Ks[1:], As[1:], sds[1:], lb, ub, gps[0]["y_mean"], gps[0]["y_std"],
                   [g["y_mean"] for g in gps[1:]], [g["y_std"] for g in gps[1:]], log=log)


def pipeline(gps, X, P, rs, S, extra_rows, in_bounds, lb, ub):
    """One closure of the class over the pending rows P: the draws in order, every GP grown, best'.
    Returns (per GP (F' data units, A'), best', eligible, the draws)."""
    d = draws(rs, X.shape[0], S, len(gps) - 1, P.shape[0] + extra_rows)
    out = []
    for g, (Z, E, Zp) in zip(gps, d):
        F, A = grown(g, X, P, Z, E, Zp)
        out.append((data_units(F, g), A))
    best, ok = incumbents(out[0][0], [o[0] for o in out[1:]], in_bounds, lb, ub)
    return out, best, ok, d
