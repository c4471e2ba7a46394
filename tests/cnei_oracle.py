"""numpy restatement of constrained noisy expected improvement (include/b200bo.h B200BO_ACQ_CNEI / LOGCNEI,
DESIGN.md 4.15).

Float64 numpy / scipy, in the order of the definition; used by tests/test_cnei_cpu.py and tests/test_gpu_cnei.py.  The
target and every constraint GP get fantasies by nei_oracle.fantasies; the constraint factors per sample follow the
device's factor rules (EI's for CNEI, log_cfactor's for LogCNEI)."""
from __future__ import annotations

import numpy as np
from scipy.special import ndtr

import logei_oracle as LO
import nei_oracle as NO


def draws(rs, n, S, J):
    """The RandomState consumption of one suggest(): the target's Z, E, then Z_j, E_j per constraint j."""
    return [NO.draws(rs, n, S) for _ in range(J + 1)]


def eligible(in_bounds, Fc, lb, ub):
    """(n, S) incumbent mask: within the bounds and lb_j <= F_j <= ub_j for every j (Fc: list of (n, S), data units)."""
    ok = np.asarray(in_bounds, dtype=bool)[:, None]
    for j, F in enumerate(Fc):
        ok = ok & (lb[j] <= F) & (F <= ub[j])
    return ok


def incumbents(F, ok):
    """best_s: the largest F[:, s] over the eligible rows, or the smallest over all rows when none is (the floor)."""
    hi = np.where(ok, F, -np.inf).max(axis=0)
    return np.where(ok.any(axis=0), hi, F.min(axis=0))


def factor(mean, sd, lb, ub):
    """P = Phi((ub - mean)/sd) - Phi((lb - mean)/sd) with the device's rules (cnei_factor): an infinite bound
    contributes 0 / 1, a finite bound with sd <= 0 gives NaN (scipy's frozen norm), and where the mean lies below a
    finite lb the pair is reflected, Phi((mean - lb)/sd) - Phi((mean - ub)/sd), so that the upper tail does not
    cancel."""
    with np.errstate(all="ignore"):
        def cdf(b):
            return np.where(sd > 0.0, ndtr((b - mean) / sd), np.nan)
        p_lo = 0.0 if lb == -np.inf else cdf(lb)
        p_hi = 1.0 if ub == np.inf else cdf(ub)
        if lb == -np.inf:
            return p_hi - p_lo
        refl = ndtr((mean - lb) / sd) - (0.0 if ub == np.inf else ndtr((mean - ub) / sd))
        return np.where((lb > mean) & (sd > 0.0), refl, p_hi - p_lo)


def cnei(Ks, A, best, sd, xi, Kc_list, Ac_list, sdc_list, lb, ub, y_mean=0.0, y_std=1.0, cy_mean=None, cy_std=None,
         log=False):
    """CNEI (or LogCNEI) per candidate.  Target: Ks (m, n), A (n, S), best (S,), sd (m,), as nei_oracle.nei.
    Constraint j: Kc_list[j] (m, n) = c_j k_j(Xc, X), Ac_list[j] = K0_j^-1 F_j (normalised), sdc_list[j] (m,) its
    noiseless sd (data units), its y statistics cy_mean[j], cy_std[j]."""
    J = len(Kc_list)
    cy_mean = [0.0] * J if cy_mean is None else cy_mean
    cy_std = [1.0] * J if cy_std is None else cy_std
    mu = y_std * (Ks @ A) + y_mean
    a = mu - best[None, :] - xi
    sd = np.asarray(sd, dtype=np.float64)[:, None]
    t = LO.log_acq_term(LO.LOGEI, a, sd) if log else NO.ei(a, sd)
    for j in range(J):
        mj = cy_std[j] * (Kc_list[j] @ Ac_list[j]) + cy_mean[j]
        sj = np.broadcast_to(np.asarray(sdc_list[j], dtype=np.float64)[:, None], mj.shape)
        if log:
            t = t + LO.log_cfactor(lb[j], ub[j], mj, sj)
        else:
            t = t * factor(mj, sj, lb[j], ub[j])
    return NO.logmeanexp(t) if log else t.mean(axis=1)
