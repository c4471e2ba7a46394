"""Oracle of the LogEI / LogPoI epilogue (DESIGN.md 4.12): a numpy restatement of the device formulas
(csrc/common.cuh log_h, log_h_ratios, log1mexp; csrc/predict_kernels.cuh log_acq_term(_grad), log_cfactor(_grad)),
operation for operation, and a 60-digit mpmath evaluation of the same quantities from their definitions.

The restatement is what the device tests compare with (on the device's own mu and sigma); tests/test_logei_cpu.py pins
it to the mpmath evaluation."""
import numpy as np
from scipy.special import erfcx, ndtr

LOGEI, LOGPOI = 6, 7
LOG_H_TAIL = -(2.0**26)
HALF_LOG_2PI = 0.91893853320467274178
HALF_LOG_PI_2 = 0.22579135264472743236
SQRT_PI_2 = 1.25331413731550025121
INV_SQRT2 = 0.70710678118654752440


def _f(x):
    return np.asarray(x, dtype=np.float64)


def norm_pdf(x):
    x = _f(x)
    with np.errstate(all="ignore"):
        return np.exp(-(x * x) / 2.0) / 2.50662827463100050242


def log_ndtr(g):
    """common.cuh log_ndtr: erfcx below 0, log1p(-ndtr(-g)) at and above."""
    g = _f(g)
    with np.errstate(all="ignore"):
        return np.where(g < 0.0, np.log(0.5 * erfcx(-g * INV_SQRT2)) - 0.5 * (g * g), np.log1p(-ndtr(-g)))


def inv_mills(g):
    g = _f(g)
    with np.errstate(all="ignore"):
        return np.where(g < 0.0, 0.79788456080286535588 / erfcx(-g * INV_SQRT2), norm_pdf(g) / ndtr(g))


def log1mexp(x):
    x = _f(x)
    with np.errstate(all="ignore"):
        return np.where(x > -0.69314718055994530942, np.log(-np.expm1(x)), np.log1p(-np.exp(x)))


def _tail_arg(z):
    return np.log(erfcx(-z * INV_SQRT2) * -z) + HALF_LOG_PI_2


def log_h(z):
    z = _f(z)
    with np.errstate(all="ignore"):
        log_phi = -0.5 * (z * z) - HALF_LOG_2PI
        direct = np.log(norm_pdf(z) + z * ndtr(z))
        mid = log_phi + log1mexp(_tail_arg(z))
        far = log_phi - 2.0 * np.log(-z)
        return np.where(z > -1.0, direct, np.where(z > LOG_H_TAIL, mid, far))


def log_h_ratios(z):
    """(r, q) = (Phi/h, phi/h)."""
    z = _f(z)
    with np.errstate(all="ignore"):
        pz, cz = norm_pdf(z), ndtr(z)
        h = pz + z * cz
        e = erfcx(-z * INV_SQRT2)
        w = -np.expm1(np.log(e * -z) + HALF_LOG_PI_2)
        r = np.where(z > -1.0, cz / h, np.where(z > LOG_H_TAIL, SQRT_PI_2 * e / w, -z))
        q = np.where(z > -1.0, pz / h, np.where(z > LOG_H_TAIL, 1.0 / w, z * z))
    return r, q


def _ei_limit(a):
    with np.errstate(all="ignore"):
        return np.where(a > 0.0, np.log(np.where(a > 0.0, a, 1.0)), np.where(a < 0.0, -np.inf, np.nan))


def log_acq_term(kind, a, sd):
    a, sd = np.broadcast_arrays(_f(a), _f(sd))
    with np.errstate(all="ignore"):
        z = a / sd
        if kind == LOGPOI:
            return log_ndtr(z)
        return np.where((sd == 0.0) | np.isinf(z), _ei_limit(a), log_h(z) + np.log(sd))


def log_acq_term_grad(kind, a, sd):
    """(value, cm, cs): d value = cm d mean + cs d sd."""
    a, sd = np.broadcast_arrays(_f(a), _f(sd))
    with np.errstate(all="ignore"):
        z = a / sd
        ok = (sd > 0.0) & ~np.isinf(z)
        if kind == LOGPOI:
            lam = inv_mills(z)
            cm = np.where(ok, lam / sd, 0.0)
            cs = np.where(ok & (lam != 0.0), -z * lam / sd, 0.0)
            return log_ndtr(z), cm, cs
        r, q = log_h_ratios(z)
        lim = (sd == 0.0) | np.isinf(z)
        cm = np.where(lim, np.where(a > 0.0, 1.0 / a, 0.0), r / sd)
        cs = np.where(lim, 0.0, q / sd)
        return log_acq_term(kind, a, sd), cm, cs


def cfactor_std(l, u):
    """log(Phi(u) - Phi(l)) on standardised bounds (l = -inf / u = +inf: one-sided), as log_cfactor forms it."""
    l, u = np.broadcast_arrays(_f(l), _f(u))
    with np.errstate(all="ignore"):
        if np.all(np.isneginf(l)):
            return log_ndtr(u)
        if np.all(np.isposinf(u)):
            return log_ndtr(-l)
        refl = l >= 0.0
        a, b = np.where(refl, -u, l), np.where(refl, -l, u)
        lpb = log_ndtr(b)
        return np.where((l < 0.0) & (u > 0.0), np.log(ndtr(u) - ndtr(l)), lpb + log1mexp(log_ndtr(a) - lpb))


def cfactor_partials(l, u):
    """(F_l, F_u): the partials of cfactor_std in l and u, in log_cfactor_grad's form."""
    l, u = np.broadcast_arrays(_f(l), _f(u))
    z = np.zeros(l.shape)
    with np.errstate(all="ignore"):
        if np.all(np.isneginf(l)):
            return z, inv_mills(u)
        if np.all(np.isposinf(u)):
            return -inv_mills(-l), z
        p = ndtr(u) - ndtr(l)
        s_fu, s_fl = norm_pdf(u) / p, -norm_pdf(l) / p
        refl = l >= 0.0
        a, b = np.where(refl, -u, l), np.where(refl, -l, u)
        d = log_ndtr(a) - log_ndtr(b)
        om = -np.expm1(d)
        gb = inv_mills(b) / om
        la = inv_mills(a)
        ga = np.where(la == 0.0, 0.0, -la * np.exp(d) / om)
        fl = np.where(refl, -gb, ga)
        fu = np.where(refl, -ga, gb)
        strad = (l < 0.0) & (u > 0.0)
        return np.where(strad, s_fl, fl), np.where(strad, s_fu, fu)


def log_cfactor(lb, ub, mean, sd):
    mean, sd = np.broadcast_arrays(_f(mean), _f(sd))
    if lb == -np.inf and ub == np.inf:
        return np.zeros(mean.shape)
    with np.errstate(all="ignore"):
        u, l = (ub - mean) / sd, (lb - mean) / sd
        if lb == -np.inf:
            l = np.full(mean.shape, -np.inf)
        if ub == np.inf:
            u = np.full(mean.shape, np.inf)
        v = cfactor_std(l, u)
        return np.where((sd > 0.0) & ~np.isnan(mean), v, np.nan)


def log_cfactor_grad(lb, ub, mean, sd):
    """(cm, cs) of one constraint factor; 0 where sd <= 0."""
    mean, sd = np.broadcast_arrays(_f(mean), _f(sd))
    z = np.zeros(mean.shape)
    if lb == -np.inf and ub == np.inf:
        return z, z
    with np.errstate(all="ignore"):
        u, l = (ub - mean) / sd, (lb - mean) / sd
        if lb == -np.inf:
            l = np.full(mean.shape, -np.inf)
        if ub == np.inf:
            u = np.full(mean.shape, np.inf)
        fl, fu = cfactor_partials(l, u)
        cm = -(fl + fu) / sd
        cs = -(np.where(fl == 0.0, 0.0, l * fl) + np.where(fu == 0.0, 0.0, u * fu)) / sd
        ok = sd > 0.0
        return np.where(ok, cm, 0.0), np.where(ok, cs, 0.0)


def closure(kind, mean, sd, y_max, xi, cons=()):
    """The closure value -(alpha + sum_j log p_j), summed in j order; cons: (mean_j, sd_j, lb_j, ub_j) per constraint."""
    s = log_acq_term(kind, _f(mean) - y_max - xi, sd)
    for m_, s_, lo, hi in cons:
        s = s + log_cfactor(lo, hi, m_, s_)
    return -s


# ---- 60-digit evaluation from the definitions --------------------------------------------------------------------
def _mp():
    import mpmath as mp

    mp.mp.dps = 60
    return mp


def mp_Phi(mp, x):
    return mp.erfc(-x / mp.sqrt(2)) / 2


# Each mp_* takes an fp64 or an mpmath argument and returns fp64 values, or with exact=True the mpmath values themselves
# (oracle/make_acq_big.py evaluates them on its unrounded double-double mu and sigma).
def _out(exact, *v):
    v = v if exact else tuple(float(x) for x in v)
    return v[0] if len(v) == 1 else v


def mp_log_h(z, exact=False):
    """log h, h = phi(z) + z Phi(z); for z < -1 from the Mills form so that the cancellation stays inside 60 digits."""
    mp = _mp()
    z = mp.mpf(z)
    if z > -1:
        return _out(exact, mp.log(mp.npdf(z) + z * mp_Phi(mp, z)))
    mp.mp.dps = 60 + int(2 * mp.log10(-z)) + 10
    h = mp.npdf(z) + z * mp_Phi(mp, z)
    return _out(exact, mp.log(h))


def mp_log_h_ratios(z, exact=False):
    mp = _mp()
    z = mp.mpf(z)
    if z < -1:
        mp.mp.dps = 60 + int(2 * mp.log10(-z)) + 10
    P, p = mp_Phi(mp, z), mp.npdf(z)
    h = p + z * P
    return _out(exact, P / h, p / h)


def mp_log_ndtr(g, exact=False):
    mp = _mp()
    x = mp.mpf(g)
    return _out(exact, mp.log(mp_Phi(mp, x)) if x < 0 else mp.log1p(-mp.erfc(x / mp.sqrt(2)) / 2))  # 1 - Phi exactly


def mp_cfactor(l, u, exact=False):
    """(log p, dlogp/dl, dlogp/du) for p = Phi(u) - Phi(l), standardised bounds (+-inf allowed)."""
    mp = _mp()
    lm = -mp.inf if l == -np.inf else mp.mpf(l)
    um = mp.inf if u == np.inf else mp.mpf(u)
    # Phi(u) - Phi(l) = Phi(-l) - Phi(-u): take the form without cancellation
    if lm >= 0:
        p = mp.erfc(lm / mp.sqrt(2)) / 2 - mp.erfc(um / mp.sqrt(2)) / 2
    else:
        p = mp_Phi(mp, um) - mp_Phi(mp, lm)
    dl = mp.mpf(0) if lm == -mp.inf else -mp.npdf(lm) / p
    du = mp.mpf(0) if um == mp.inf else mp.npdf(um) / p
    return _out(exact, mp.log(p), dl, du)
