"""The branch-free covariance primitives of csrc/common.cuh, restated with exact rational arithmetic.

Phase A evaluates k * k / 3 (Matern 2.5) and the rint / exponent steps of exp_neg once per (candidate, training row)
pair.  The device computes them without a division, FRND or F2I (div3_rn; the 1.5 * 2^52 shift), and these must give
the same double as the IEEE operations they replace, bit for bit.  Each FMA is evaluated exactly with
fractions.Fraction and rounded once by float() (correctly rounded, half to even), which is what DFMA does.
"""
import math
import struct
from fractions import Fraction

import numpy as np

THIRD = 1.0 / 3.0  # RN(1/3), the constant div3_rn multiplies by
LOG2E = 1.4426950408889634074  # kExpR[0]
SHIFT = 6755399441055744.0  # 1.5 * 2^52


def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def div3_rn(x):
    """csrc/common.cuh div3_rn: q = RN(x RN(1/3)), r = fma(-q, 3, x), fma(r, RN(1/3), q)."""
    q = x * THIRD
    r = fma(-q, 3.0, x)
    return fma(r, THIRD, q)


def lo_word(v):
    return struct.unpack("<ii", struct.pack("<d", v))[0]


def hi_word(v):
    return struct.unpack("<ii", struct.pack("<d", v))[1]


def from_words(hi, lo):
    return struct.unpack("<d", struct.pack("<ii", lo, hi))[0]


def _div3_arguments():
    """The range the callers pass (k^2, k from sqrt_pos: [1e-30, 5e38]): log-uniform values, exact multiples of 3 and
    their neighbours, arguments whose quotient lies next to a midpoint between two doubles, and squares of k."""
    rs = np.random.RandomState(1234)
    xs = list(10.0 ** rs.uniform(np.log10(1e-30), np.log10(5e38), 20000))
    for y in 10.0 ** rs.uniform(-30, 38, 4000):  # x = 3 y exactly when representable, and the doubles around it
        x = 3.0 * float(y)
        xs += [x, np.nextafter(x, 0.0), np.nextafter(x, np.inf)]
    for y in 10.0 ** rs.uniform(-30, 38, 4000):  # x / 3 near the midpoint of y and its successor
        mid = Fraction(float(y)) + (Fraction(float(np.nextafter(y, np.inf))) - Fraction(float(y))) / 2
        x = float(3 * mid)
        xs += [x, np.nextafter(x, 0.0), np.nextafter(x, np.inf)]
    for k in 10.0 ** rs.uniform(-15, 19.3, 6000):  # k * k as Matern 2.5 forms it
        xs.append(float(k) * float(k))
    xs += [float(i) for i in range(1, 3000)]  # small integers: many exact quotients and ties of the residual
    return [float(x) for x in xs if 1e-30 <= x <= 5e38]


def test_div3_rn_is_the_ieee_quotient():
    xs = _div3_arguments()
    assert len(xs) > 40000
    bad = [x for x in xs if div3_rn(x) != x / 3.0]
    assert not bad, bad[:5]


def _rint_arguments():
    """Products p = RN(-k log2e) over exp_neg's domain k in [0, 700]: random k, the half-integers and their
    neighbours (round half to even decides them), and the products of k near those ties."""
    rs = np.random.RandomState(4321)
    ps = [-(float(k) * LOG2E) for k in rs.uniform(0.0, 700.0, 20000)]
    ps += [-(float(k) * LOG2E) for k in 10.0 ** rs.uniform(-20, math.log10(700.0), 5000)]
    for m in range(0, 1010):
        h = -(m + 0.5)
        ps += [h, float(np.nextafter(h, 0.0)), float(np.nextafter(h, -np.inf)), -float(m)]
        k = (m + 0.5) / LOG2E
        for kk in (k, np.nextafter(k, 0.0), np.nextafter(k, np.inf)):
            ps.append(-(float(kk) * LOG2E))
    ps += [-(700.0 * LOG2E), 0.0, -0.0, -1e-300, -0.49999999999999994]
    return [p for p in ps if -1010.0 <= p <= 0.0]


def test_shifted_rint_and_exponent():
    """n = (p + 1.5 2^52) - 1.5 2^52 equals rint(p) (Python's round(): half to even), the low word of the shifted sum
    is n as an integer, and adding n << 20 to the high word of a p in [sqrt(1/2), sqrt(2)] is the multiply by 2^n."""
    rs = np.random.RandomState(99)
    ps = _rint_arguments()
    assert len(ps) > 30000
    for p in ps:
        t = p + SHIFT
        n = t - SHIFT
        assert n == round(p), p
        assert lo_word(t) == round(p), p
        poly = float(rs.uniform(math.sqrt(0.5), math.sqrt(2.0)))
        e = ((lo_word(t) << 20) + (1 << 31)) % (1 << 32) - (1 << 31)  # the int32 the device adds
        assert from_words(hi_word(poly) + e, lo_word(poly)) == math.ldexp(poly, round(p)), p
    for poly in (math.sqrt(0.5), float(np.nextafter(math.sqrt(0.5), 0.0)), 1.0, math.sqrt(2.0),
                 float(np.nextafter(math.sqrt(2.0), np.inf))):
        for n in (0, -1, -1009, -1010):
            assert from_words(hi_word(poly) + n * (1 << 20), lo_word(poly)) == math.ldexp(poly, n)
