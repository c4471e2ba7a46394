"""The error bound of the Gram bound pass of pruning (predict_bound_gram_kernel, csrc/predict16.cuh; DESIGN.md 4.9),
restated in numpy and checked on adversarial inputs.

The pass forms r~^2 = [x, |x|^2, 1] . [-2y, 1, |y|^2] on the fp64 tensor pipe.  Its bound, with S = |x|^2 + Ymax from
the rounded norms and g_n = n u / (1 - n u):
    |r~^2 - r^2_direct| <= 6 g_{d+2} S          (kGramCg = 6)
where r^2_direct is phase A's sum of squared differences, the value the exact path builds its covariance from.  Every
product-add of the Gram sum is taken as IEEE-rounded, in any order: here the sum is emulated exactly (fractions, one
correct rounding per step) in random orders, both as fused and as separate product / add roundings.  Then
    dk = constv (Lip dr2 + 64 u),   dmu = A1 (dk + 3 g_np constv) (1 + 2^-20)
must hold mu, summed from the direct covariances, within [mu~ - dmu, mu~ + dmu] of the Gram sum.
"""
from fractions import Fraction

import numpy as np
import pytest

U = 2.0 ** -53
CG, CCOV = 6.0, 64.0  # kGramCg, kGramCcov
LIP = {"m15": 1.5, "m25": 5.0 / 6.0, "rbf": 0.5}


def gamma(n):
    return n * U / (1 - n * U)


def rn(q):
    """Fraction -> the nearest double (ties to even)."""
    return float(q)


def fma(a, b, c):
    return rn(Fraction(a) * Fraction(b) + Fraction(c))


def direct_r2(x, y):
    """phase A: d_j = x_j - y_j rounded, then an fma chain."""
    acc = 0.0
    for xj, yj in zip(x, y):
        dj = float(xj - yj)
        acc = fma(dj, dj, acc)
    return acc


def norm2(v):
    acc = 0.0
    for vj in v:
        acc = fma(vj, vj, acc)
    return acc


def gram_r2(x, y, rs, fused):
    """[x, |x|^2, 1] . [-2y, 1, |y|^2], every product-add rounded, in a random order."""
    a = list(x) + [norm2(x), 1.0]
    b = [-2.0 * v for v in y] + [1.0, norm2(y)]
    acc = 0.0
    for k in rs.permutation(len(a)):
        if fused:
            acc = fma(a[k], b[k], acc)
        else:
            acc = rn(Fraction(rn(Fraction(a[k]) * Fraction(b[k]))) + Fraction(acc))
    return acc


def exact_r2(x, y):
    return sum((Fraction(a) - Fraction(b)) ** 2 for a, b in zip(x, y))


def dr2_bound(d, x2, ymax):
    return CG * gamma(d + 2) * (x2 + ymax)


def cov(kind, r2):
    if kind == "rbf":
        return np.exp(-0.5 * r2)
    r = np.sqrt(np.maximum(r2, 0.0))
    if kind == "m15":
        k = np.sqrt(3.0) * r
        return (1 + k) * np.exp(-k)
    k = np.sqrt(5.0) * r
    return (1 + k + k * k / 3) * np.exp(-k)


def inputs(d, case, rs):
    """(candidates, training rows) already divided by the length scales."""
    if case == "uniform":
        y = rs.uniform(size=(24, d)) / 0.3
        x = rs.uniform(size=(24, d)) / 0.3
    elif case == "near_duplicates":
        y = rs.uniform(size=(24, d)) / 0.7
        x = y + 1e-9 * rs.standard_normal(size=y.shape)
        x[:4] = y[:4]
    elif case == "scaled":  # coordinates at 1e3 / ls, near-duplicates among them
        y = rs.uniform(-1, 1, size=(24, d)) * 1e3 / 0.05
        x = y + rs.standard_normal(size=y.shape) * np.where(np.arange(24)[:, None] < 12, 1e-6, 10.0)
    else:  # ARD: length scales over six decades
        ls = np.logspace(-3, 3, d)
        y = rs.uniform(-5, 5, size=(24, d)) / ls
        x = y + 1e-7 * rs.standard_normal(size=y.shape) / ls
    return x, y


@pytest.mark.parametrize("d", (2, 16, 17, 32, 64))
@pytest.mark.parametrize("case", ("uniform", "near_duplicates", "scaled", "ard"))
def test_gram_r2_within_bound(d, case):
    rs = np.random.RandomState(d * 7 + len(case))
    x, y = inputs(d, case, rs)
    ymax = max(norm2(v) for v in y)
    worst = 0.0
    for i in range(x.shape[0]):
        x2 = norm2(x[i])
        for j in range(0, y.shape[0], 3):
            ex = exact_r2(x[i], y[j])
            dr = direct_r2(x[i], y[j])
            bound = dr2_bound(d, x2, ymax)
            for fused in (True, False):
                g = gram_r2(x[i], y[j], rs, fused)
                err = abs(Fraction(g) - Fraction(dr))
                assert err <= Fraction(bound), (i, j, float(err), bound)
                # the part against the exact value alone stays within the Gram term of the bound (3 g S)
                assert abs(Fraction(g) - ex) <= Fraction(bound) / 2
                worst = max(worst, float(err) / (CG * gamma(d + 2) * (x2 + ymax)))
    print(f"d={d} {case}: largest |r~^2 - r^2_direct| / bound = {worst:.3e}")


@pytest.mark.parametrize("kind", sorted(LIP))
@pytest.mark.parametrize("d", (2, 16, 64))
def test_mu_interval_holds_direct_mu(kind, d):
    """mu summed from the direct covariances lies within dmu of the Gram sum, for heavy cancelling alpha."""
    rs = np.random.RandomState(d + len(kind))
    n, constv = 200, 1.7
    y = rs.uniform(size=(n, d)) / 0.4
    xs = np.vstack([rs.uniform(size=(30, d)) / 0.4, y[:10] + 1e-9])
    alpha = rs.standard_normal(n) * 10.0 ** rs.uniform(-2, 6, n)
    a1 = np.sum(np.abs(alpha))
    ymax = max(norm2(v) for v in y)
    for x in xs:
        x2 = norm2(x)
        r2d = np.array([direct_r2(x, v) for v in y])
        r2g = np.array([gram_r2(x, v, rs, True) for v in y])
        kd = constv * cov(kind, r2d)
        kg = cov(kind, r2g)
        mu = 0.0
        for i in range(n):  # phase A's order
            mu = fma(alpha[i], kd[i], mu)
        acc = 0.0
        for i in rs.permutation(n):  # the Gram pass's order differs: any order
            acc = fma(alpha[i], kg[i], acc)
        mu_g = constv * acc
        dk = constv * (LIP[kind] * dr2_bound(d, x2, ymax) + CCOV * U)
        dmu = a1 * (dk + 3 * gamma(n) * constv) * (1 + 2.0 ** -20)
        assert abs(mu - mu_g) <= dmu, (mu, mu_g, dmu)
        # max |k| from below
        kmax_lb = max(0.0, constv * float(np.max(kg)) - dk)
        assert kmax_lb <= float(np.max(np.abs(kd)))


def test_lipschitz_constants():
    """sup |dk/d(r^2)| of the unit covariances, numerically, against the constants of the bound."""
    s = np.concatenate([np.logspace(-14, 3, 20000), [0.0]])
    h = 1e-7
    for kind, lip in LIP.items():
        deriv = np.abs(cov(kind, s + h) - cov(kind, s)) / h
        assert np.max(deriv) <= lip * (1 + 1e-5), kind
        assert np.max(deriv) >= lip * (1 - 1e-3), kind
