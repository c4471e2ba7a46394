"""Double-double reference of the GP fit, posterior and log-marginal likelihood at production sizes.

The 50-digit references (oracle/make_illcond.py, oracle/make_illcond_ext.py) cost about N^3 mpmath operations and stop
at N = 200.  Double-double arithmetic carries a number as an unevaluated sum hi + lo of two fp64 values, about 106
bits (unit roundoff about 1.2e-32), at a few tens of fp64 operations per operation, so the same pipeline runs at
N = 1000 .. 4096 in seconds to minutes on the CPU (numba, parallel over rows or candidates).  At cond(K) = 1e12 its
forward error on sigma^2 stays below 1e-16 of the prior, far under any fp64 computation's error.

Every reduction runs in a fixed order (one sequential loop per output element; the parallel loops only split the
output elements), so the results are bit-reproducible whatever the thread count.  Products are Dekker's two_prod
(Veltkamp splitting, no FMA), so they do not depend on the compiler contracting a * b + c either.

The covariances are those of make_illcond._cov: sklearn's Matern 1/2, 3/2, 5/2 and RBF of the scaled squared distance
r^2 = sum ((x - x') / l)^2, times a ConstantKernel value, plus a WhiteKernel value and alpha on the diagonal.  Length
scales and constants are powers of two, so the scaled inputs are exact in fp64; their differences are exact as
double-doubles (two_sum) and so are the squares up to the 106-bit rounding of each product.

Arrays of double-doubles are pairs (hi, lo) of fp64 arrays of the same shape.
"""
from __future__ import annotations

import mpmath as mp
import numpy as np
from numba import njit, prange

CODES = {"m05": 0, "m15": 1, "m25": 2, "rbf": 3}

_SPLIT = 134217729.0  # 2^27 + 1 (Veltkamp)
# ln 2, sqrt 3, sqrt 5 and 5/3 as double-doubles (hi = the fp64 rounding, lo = the fp64 rounding of the rest)
mp.mp.dps = 50


def _pair(v):
    hi = float(v)
    return hi, float(v - mp.mpf(hi))


LN2_H, LN2_L = _pair(mp.log(2))
SQRT3_H, SQRT3_L = _pair(mp.sqrt(3))
SQRT5_H, SQRT5_L = _pair(mp.sqrt(5))
EXP_HALVINGS = 10  # exp(r) = exp(r / 2^10)^(2^10) after the reduction by k ln 2
EXP_TERMS = 12  # Taylor terms of expm1 at |r| <= ln2 / 2^11: the 12th is below 1e-50
# pi/2 as the sum of three doubles (each the fp64 rounding of the rest): k (pi/2 - P1 - P2 - P3) stays below 1e-40
# for any |k| < 2^40, far past every feature argument of the path fixtures (|omega . xs + b| < 1e8).
_PIO2 = mp.pi / 2
PIO2_1 = float(_PIO2)
PIO2_2 = float(_PIO2 - PIO2_1)
PIO2_3 = float(_PIO2 - PIO2_1 - PIO2_2)
TWO_OVER_PI = float(2 / mp.pi)
# Taylor coefficients (-1)^k / (2k)! of cos and (-1)^k / (2k+1)! of sin (k = 0 .. 14) as double-doubles: at |r| <= pi/4
# the first omitted terms are below 3e-36.
TRIG_TERMS = 15
COS_C = np.array([_pair(mp.mpf(-1) ** k / mp.factorial(2 * k)) for k in range(TRIG_TERMS)])
SIN_C = np.array([_pair(mp.mpf(-1) ** k / mp.factorial(2 * k + 1)) for k in range(TRIG_TERMS)])


# ---------------------------------------------------------------------------------------------------------------
# scalar arithmetic
# ---------------------------------------------------------------------------------------------------------------
@njit(cache=False)
def two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


@njit(cache=False)
def quick_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


@njit(cache=False)
def _split(a):
    t = _SPLIT * a
    hi = t - (t - a)
    return hi, a - hi


@njit(cache=False)
def two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


@njit(cache=False)
def dd_add(ah, al, bh, bl):
    s, e = two_sum(ah, bh)
    t, f = two_sum(al, bl)
    e += t
    s, e = quick_two_sum(s, e)
    e += f
    return quick_two_sum(s, e)


@njit(cache=False)
def dd_sub(ah, al, bh, bl):
    return dd_add(ah, al, -bh, -bl)


@njit(cache=False)
def dd_mul(ah, al, bh, bl):
    p, e = two_prod(ah, bh)
    e += ah * bl + al * bh
    return quick_two_sum(p, e)


@njit(cache=False)
def dd_mul_d(ah, al, b):
    p, e = two_prod(ah, b)
    e += al * b
    return quick_two_sum(p, e)


@njit(cache=False)
def dd_div(ah, al, bh, bl):
    q1 = ah / bh
    ph, pl = dd_mul_d(bh, bl, q1)
    rh, rl = dd_sub(ah, al, ph, pl)
    q2 = rh / bh
    ph, pl = dd_mul_d(bh, bl, q2)
    rh, rl = dd_sub(rh, rl, ph, pl)
    q3 = rh / bh
    q1, q2 = quick_two_sum(q1, q2)
    return dd_add(q1, q2, q3, 0.0)


@njit(cache=False)
def dd_sqrt(ah, al):
    """One Newton step from the fp64 root (Karp-Markstein); 0 at a non-positive argument."""
    if ah <= 0.0:
        return 0.0, 0.0
    x = 1.0 / np.sqrt(ah)
    ax = ah * x
    ph, pl = two_prod(ax, ax)
    dh, _ = dd_sub(ah, al, ph, pl)
    return two_sum(ax, dh * (x * 0.5))


@njit(cache=False)
def dd_exp(ah, al):
    """exp: a = k ln2 + 2^10 r, expm1(r) by its Taylor series (Horner), doubled back ten times through
    expm1(2x) = expm1(x) (2 + expm1(x)), then scaled by 2^k.  0 below -745.2 (the fp64 underflow)."""
    if ah < -745.2:
        return 0.0, 0.0
    k = np.floor(ah / LN2_H + 0.5)
    ph, pl = dd_mul_d(LN2_H, LN2_L, k)
    rh, rl = dd_sub(ah, al, ph, pl)
    sc = 1.0 / (1 << EXP_HALVINGS)
    rh *= sc
    rl *= sc
    sh, sl = 1.0, 0.0
    for n in range(EXP_TERMS, 1, -1):  # s = 1 + r/n s
        th, tl = dd_mul(rh, rl, sh, sl)
        th, tl = dd_div(th, tl, float(n), 0.0)
        sh, sl = dd_add(th, tl, 1.0, 0.0)
    sh, sl = dd_mul(rh, rl, sh, sl)  # expm1(r)
    for _ in range(EXP_HALVINGS):
        th, tl = dd_add(sh, sl, 2.0, 0.0)
        sh, sl = dd_mul(sh, sl, th, tl)
    sh, sl = dd_add(sh, sl, 1.0, 0.0)
    ki = int(k)
    return np.ldexp(sh, ki), np.ldexp(sl, ki)


@njit(cache=False)
def dd_cos_sin(ah, al):
    """(cos a, sin a) as double-doubles: a = k pi/2 + r with pi/2 in three doubles (the products k P_i exact), then the
    Taylor series of cos and sin on |r| <= pi/4 (Horner in r^2) and the quadrant k mod 4."""
    k = np.floor(ah * TWO_OVER_PI + 0.5)
    ph, pl = two_prod(k, PIO2_1)
    rh, rl = dd_sub(ah, al, ph, pl)
    ph, pl = two_prod(k, PIO2_2)
    rh, rl = dd_sub(rh, rl, ph, pl)
    ph, pl = two_prod(k, PIO2_3)
    rh, rl = dd_sub(rh, rl, ph, pl)
    zh, zl = dd_mul(rh, rl, rh, rl)
    ch, cl = COS_C[TRIG_TERMS - 1, 0], COS_C[TRIG_TERMS - 1, 1]
    sh, sl = SIN_C[TRIG_TERMS - 1, 0], SIN_C[TRIG_TERMS - 1, 1]
    for i in range(TRIG_TERMS - 2, -1, -1):
        ch, cl = dd_mul(ch, cl, zh, zl)
        ch, cl = dd_add(ch, cl, COS_C[i, 0], COS_C[i, 1])
        sh, sl = dd_mul(sh, sl, zh, zl)
        sh, sl = dd_add(sh, sl, SIN_C[i, 0], SIN_C[i, 1])
    sh, sl = dd_mul(sh, sl, rh, rl)
    quad = int(k) % 4
    if quad == 0:
        return ch, cl, sh, sl
    if quad == 1:
        return -sh, -sl, ch, cl
    if quad == 2:
        return -ch, -cl, -sh, -sl
    return sh, sl, -ch, -cl


@njit(cache=False)
def cov_dd(code, r2h, r2l):
    """The unit covariance of the scaled squared distance (make_illcond._cov)."""
    if code == 3:
        return dd_exp(-0.5 * r2h, -0.5 * r2l)
    dh, dl = dd_sqrt(r2h, r2l)
    if code == 0:
        return dd_exp(-dh, -dl)
    if code == 1:
        kh, kl = dd_mul(dh, dl, SQRT3_H, SQRT3_L)
        eh, el = dd_exp(-kh, -kl)
        ph, pl = dd_add(kh, kl, 1.0, 0.0)
        return dd_mul(ph, pl, eh, el)
    kh, kl = dd_mul(dh, dl, SQRT5_H, SQRT5_L)
    eh, el = dd_exp(-kh, -kl)
    qh, ql = dd_mul(kh, kl, kh, kl)
    qh, ql = dd_div(qh, ql, 3.0, 0.0)
    ph, pl = dd_add(kh, kl, 1.0, 0.0)
    ph, pl = dd_add(ph, pl, qh, ql)
    return dd_mul(ph, pl, eh, el)


@njit(cache=False)
def grad_factor_dd(code, r2h, r2l, kh, kl):
    """g with dk / dlog(l_t) = g (dx_t / l_t)^2 (make_illcond._grad_factor); kh + kl = the covariance at r2."""
    if code == 3:
        return kh, kl
    dh, dl = dd_sqrt(r2h, r2l)
    if code == 0:
        if r2h == 0.0:
            return 0.0, 0.0
        return dd_div(kh, kl, dh, dl)
    if code == 1:
        th, tl = dd_mul(dh, dl, SQRT3_H, SQRT3_L)
        eh, el = dd_exp(-th, -tl)
        return dd_mul_d(eh, el, 3.0)
    th, tl = dd_mul(dh, dl, SQRT5_H, SQRT5_L)
    eh, el = dd_exp(-th, -tl)
    ph, pl = dd_add(th, tl, 1.0, 0.0)
    ph, pl = dd_mul(ph, pl, eh, el)
    ph, pl = dd_mul_d(ph, pl, 5.0)
    return dd_div(ph, pl, 3.0, 0.0)


@njit(cache=False)
def _r2(a, b):
    """sum_t (a_t - b_t)^2 of two scaled fp64 rows, in order t = 0 .. d-1."""
    sh, sl = 0.0, 0.0
    for t in range(a.shape[0]):
        dh, dl = two_sum(a[t], -b[t])
        qh, ql = dd_mul(dh, dl, dh, dl)
        sh, sl = dd_add(sh, sl, qh, ql)
    return sh, sl


@njit(cache=False)
def _dot(ah, al, bh, bl, lo, hi):
    """sum_{k = lo}^{hi - 1} a_k b_k in order."""
    sh, sl = 0.0, 0.0
    for k in range(lo, hi):
        ph, pl = dd_mul(ah[k], al[k], bh[k], bl[k])
        sh, sl = dd_add(sh, sl, ph, pl)
    return sh, sl


# ---------------------------------------------------------------------------------------------------------------
# matrices
# ---------------------------------------------------------------------------------------------------------------
@njit(parallel=True, cache=False)
def cross_cov(A, B, code, c):
    """c k(A, B) for scaled rows A (m, d) and B (n, d); c a power of two (exact)."""
    m, n = A.shape[0], B.shape[0]
    Kh = np.empty((m, n))
    Kl = np.empty((m, n))
    for i in prange(m):
        for j in range(n):
            rh, rl = _r2(A[i], B[j])
            kh, kl = cov_dd(code, rh, rl)
            Kh[i, j] = c * kh
            Kl[i, j] = c * kl
    return Kh, Kl


@njit(parallel=True, cache=False)
def chol_rows(Kh, Kl, koff, Lh, Ll, i0, i1, block):
    """Rows i0 .. i1-1 of the lower Cholesky factor in place, rows below i0 given; row i of K is K[i - koff] (only
    its first i + 1 entries are read).  Column panels of `block`: the rows inside a panel's diagonal block one after
    the other, the rows below it in parallel; every entry is one sequential dot product.  Returns 0, or the 1-based
    row of the first non-positive pivot."""
    for j0 in range(0, i1, block):
        j1 = min(j0 + block, i1)
        for i in range(max(j0, i0), j1):
            for j in range(j0, i + 1):
                sh, sl = _dot(Lh[i], Ll[i], Lh[j], Ll[j], 0, j)
                sh, sl = dd_sub(Kh[i - koff, j], Kl[i - koff, j], sh, sl)
                if j == i:
                    if sh <= 0.0:
                        return i + 1
                    Lh[i, i], Ll[i, i] = dd_sqrt(sh, sl)
                else:
                    Lh[i, j], Ll[i, j] = dd_div(sh, sl, Lh[j, j], Ll[j, j])
        for i in prange(max(j1, i0), i1):
            for j in range(j0, j1):
                sh, sl = _dot(Lh[i], Ll[i], Lh[j], Ll[j], 0, j)
                sh, sl = dd_sub(Kh[i - koff, j], Kl[i - koff, j], sh, sl)
                Lh[i, j], Ll[i, j] = dd_div(sh, sl, Lh[j, j], Ll[j, j])
    return 0


@njit(parallel=True, cache=False)
def forward_rows(Lh, Ll, Bh, Bl, n):
    """V[t] = L[:n, :n]^-1 B[t, :n] for every row t of B, by forward substitution (rows in parallel)."""
    m = Bh.shape[0]
    Vh = np.zeros((m, n))
    Vl = np.zeros((m, n))
    for t in prange(m):
        for i in range(n):
            sh, sl = _dot(Lh[i], Ll[i], Vh[t], Vl[t], 0, i)
            sh, sl = dd_sub(Bh[t, i], Bl[t, i], sh, sl)
            Vh[t, i], Vl[t, i] = dd_div(sh, sl, Lh[i, i], Ll[i, i])
    return Vh, Vl


@njit(cache=False)
def backward(Lh, Ll, zh, zl, n):
    """x = L[:n, :n]^-T z."""
    xh = np.zeros(n)
    xl = np.zeros(n)
    for i in range(n - 1, -1, -1):
        sh, sl = 0.0, 0.0
        for k in range(i + 1, n):
            ph, pl = dd_mul(Lh[k, i], Ll[k, i], xh[k], xl[k])
            sh, sl = dd_add(sh, sl, ph, pl)
        sh, sl = dd_sub(zh[i], zl[i], sh, sl)
        xh[i], xl[i] = dd_div(sh, sl, Lh[i, i], Ll[i, i])
    return xh, xl


@njit(parallel=True, cache=False)
def backward_rows(Lh, Ll, Zh, Zl, n):
    """X[t] = L[:n, :n]^-T Z[t, :n] for every row t of Z: backward() row by row (rows in parallel), bit-equal to it.
    Reads L's columns through a transposed copy."""
    Th = np.ascontiguousarray(Lh[:n, :n].T)
    Tl = np.ascontiguousarray(Ll[:n, :n].T)
    m = Zh.shape[0]
    Xh = np.zeros((m, n))
    Xl = np.zeros((m, n))
    for t in prange(m):
        for i in range(n - 1, -1, -1):
            sh, sl = 0.0, 0.0
            for k in range(i + 1, n):
                ph, pl = dd_mul(Th[i, k], Tl[i, k], Xh[t, k], Xl[t, k])
                sh, sl = dd_add(sh, sl, ph, pl)
            sh, sl = dd_sub(Zh[t, i], Zl[t, i], sh, sl)
            Xh[t, i], Xl[t, i] = dd_div(sh, sl, Th[i, i], Tl[i, i])
    return Xh, Xl


@njit(parallel=True, cache=False)
def lower_rows(Lh, Ll, Bh, Bl, n):
    """V[t] = L[:n, :n] B[t, :n] for every row t of B: one ordered dot product per entry (factor rows in parallel)."""
    m = Bh.shape[0]
    Vh = np.zeros((m, n))
    Vl = np.zeros((m, n))
    for i in prange(n):
        for t in range(m):
            Vh[t, i], Vl[t, i] = _dot(Lh[i], Ll[i], Bh[t], Bl[t], 0, i + 1)
    return Vh, Vl


@njit(parallel=True, cache=False)
def cross_cov_grad(A, B, code, c, inv_ls, Wh, Wl):
    """G[t, q, j] = sum_i W[t, q, i] d(c k(a_t, b_i)) / d x_j for scaled rows A (m, d) and B (n, d), the derivative in
    unscaled input coordinates: d k / d x_j = -c g(r^2) (a_tj - b_ij) / l_j with g of grad_factor_dd (0 at r = 0 for
    Matern 1/2) and inv_ls = 1 / l (powers of two: exact).  Sums over i in order; rows t in parallel."""
    m, d = A.shape
    n = B.shape[0]
    nq = Wh.shape[1]
    Gh = np.zeros((m, nq, d))
    Gl = np.zeros((m, nq, d))
    for t in prange(m):
        for i in range(n):
            rh, rl = _r2(A[t], B[i])
            kh, kl = cov_dd(code, rh, rl)
            gh, gl = grad_factor_dd(code, rh, rl, kh, kl)
            for j in range(d):
                dh, dl = two_sum(A[t, j], -B[i, j])
                dh, dl = dd_mul(dh, dl, gh, gl)
                dh, dl = -c * inv_ls[j] * dh, -c * inv_ls[j] * dl
                for q in range(nq):
                    ph, pl = dd_mul(Wh[t, q, i], Wl[t, q, i], dh, dl)
                    Gh[t, q, j], Gl[t, q, j] = dd_add(Gh[t, q, j], Gl[t, q, j], ph, pl)
    return Gh, Gl


@njit(parallel=True, cache=False)
def inverse_t(Lh, Ll, n):
    """Wt = (L^-1)^T: row j of Wt is column j of L^-1, zero before j (columns in parallel)."""
    Wh = np.zeros((n, n))
    Wl = np.zeros((n, n))
    for j in prange(n):
        Wh[j, j], Wl[j, j] = dd_div(1.0, 0.0, Lh[j, j], Ll[j, j])
        for i in range(j + 1, n):
            sh, sl = _dot(Lh[i], Ll[i], Wh[j], Wl[j], j, i)
            Wh[j, i], Wl[j, i] = dd_div(-sh, -sl, Lh[i, i], Ll[i, i])
    return Wh, Wl


@njit(parallel=True, cache=False)
def _grad_rows(Wh, Wl, ah, al, Xs, code, c, ard):
    """Per row i: sum_{j <= i} w_ij dK_ij / dtheta with w_ij = (alpha_i alpha_j - Kinv_ij) (2 off the diagonal),
    Kinv_ij = sum_{k >= i} Wt[i, k] Wt[j, k].  Columns of the result: const, the length scale(s), the diagonal."""
    n, d = Xs.shape
    nls = d if ard else 1
    G = np.zeros((n, 2 + nls, 2))
    for i in prange(n):
        gch, gcl = 0.0, 0.0
        glh = np.zeros(nls)
        gll = np.zeros(nls)
        for j in range(i + 1):
            kih, kil = _dot(Wh[i], Wl[i], Wh[j], Wl[j], i, n)
            wh, wl = dd_mul(ah[i], al[i], ah[j], al[j])
            wh, wl = dd_sub(wh, wl, kih, kil)
            if j != i:
                wh *= 2.0
                wl *= 2.0
            rh, rl = _r2(Xs[i], Xs[j])
            kh, kl = cov_dd(code, rh, rl)
            th, tl = dd_mul(wh, wl, kh, kl)
            gch, gcl = dd_add(gch, gcl, c * th, c * tl)
            fh, fl = grad_factor_dd(code, rh, rl, kh, kl)
            fh, fl = dd_mul(fh, fl, wh, wl)
            fh *= c
            fl *= c
            if ard:
                for t in range(d):
                    dh, dl = two_sum(Xs[i, t], -Xs[j, t])
                    dh, dl = dd_mul(dh, dl, dh, dl)
                    ph, pl = dd_mul(fh, fl, dh, dl)
                    glh[t], gll[t] = dd_add(glh[t], gll[t], ph, pl)
            else:
                ph, pl = dd_mul(fh, fl, rh, rl)
                glh[0], gll[0] = dd_add(glh[0], gll[0], ph, pl)
            if j == i:
                G[i, 1 + nls, 0], G[i, 1 + nls, 1] = wh, wl
        G[i, 0, 0], G[i, 0, 1] = gch, gcl
        for t in range(nls):
            G[i, 1 + t, 0], G[i, 1 + t, 1] = glh[t], gll[t]
    return G


@njit(cache=False)
def _sum_rows(G):
    """Column sums of G (n, m, 2) in row order."""
    n, m = G.shape[0], G.shape[1]
    out = np.zeros((m, 2))
    for i in range(n):
        for q in range(m):
            out[q, 0], out[q, 1] = dd_add(out[q, 0], out[q, 1], G[i, q, 0], G[i, q, 1])
    return out


@njit(parallel=True, cache=False)
def _residual_rows(K, a, yh, yl):
    n = K.shape[0]
    r = np.zeros(n)
    for i in prange(n):
        sh, sl = 0.0, 0.0
        for j in range(n):
            ph, pl = two_prod(K[i, j], a[j])
            sh, sl = dd_add(sh, sl, ph, pl)
        rh, rl = dd_sub(yh[i], yl[i], sh, sl)
        r[i] = abs(rh + rl)
    return r


@njit(parallel=True, cache=False)
def _sumsq_prefix(Vh, Vl, ends):
    """S[t, q] = sum_{i < ends[q]} V[t, i]^2 (ends increasing), in index order."""
    m = Vh.shape[0]
    S = np.zeros((m, len(ends), 2))
    for t in prange(m):
        sh, sl = 0.0, 0.0
        i = 0
        for q in range(len(ends)):
            while i < ends[q]:
                ph, pl = dd_mul(Vh[t, i], Vl[t, i], Vh[t, i], Vl[t, i])
                sh, sl = dd_add(sh, sl, ph, pl)
                i += 1
            S[t, q, 0], S[t, q, 1] = sh, sl
    return S


@njit(parallel=True, cache=False)
def _matvec(Ah, Al, xh, xl):
    m, n = Ah.shape
    oh = np.zeros(m)
    ol = np.zeros(m)
    for t in prange(m):
        oh[t], ol[t] = _dot(Ah[t], Al[t], xh, xl, 0, n)
    return oh, ol


# ---------------------------------------------------------------------------------------------------------------
# the GP pipeline
# ---------------------------------------------------------------------------------------------------------------
def to_mp(h, l):
    return mp.mpf(float(h)) + mp.mpf(float(l))


def from_mp(v):
    return _pair(v)


def ls_vec(case):
    ls = case["ls"]
    return np.asarray(ls, dtype=float) if np.iterable(ls) else np.full(case["d"], float(ls))


def scaled(case, X):
    """X / l, exact (l a power of two)."""
    ls = ls_vec(case)
    assert np.all(np.frexp(ls)[0] == 0.5), "length scales must be powers of two"
    return np.ascontiguousarray(np.asarray(X, dtype=float) / ls)


class Fit:
    """The double-double fit of a case (a make_illcond.CASES dict) on (X, y), with room for `extra` rows appended to
    the factor later (extend()).  Attributes: K (the upper-left n x n block, pair of arrays), L (pair, (n + extra)^2),
    alpha_ (pair), y_mean / y_std (mpmath), yn (pair)."""

    BLOCK = 32

    def __init__(self, case, X, y, extra=0):
        mp.mp.dps = 50
        self.case = case
        self.code = CODES[case["kern"]]
        self.c = float(case.get("const") or 1.0)
        assert np.frexp(self.c)[0] == 0.5, "ConstantKernel values must be powers of two"
        self.white = float(case.get("white") or 0.0)
        self.Xs = scaled(case, X)
        n = self.n = len(X)
        self.rows = n
        self.K = cross_cov(self.Xs, self.Xs, self.code, self.c)
        dh, dl = self.diag = from_mp(mp.mpf(self.c) + mp.mpf(self.white) + mp.mpf(case["alpha"]))
        np.fill_diagonal(self.K[0], dh)
        np.fill_diagonal(self.K[1], dl)
        self.prior = mp.mpf(self.c) + mp.mpf(self.white)
        N = n + extra
        self.L = (np.zeros((N, N)), np.zeros((N, N)))
        info = chol_rows(self.K[0], self.K[1], 0, self.L[0], self.L[1], 0, n, self.BLOCK)
        if info:
            raise ValueError(f"K is not positive definite at row {info}")
        ym = [mp.mpf(float(v)) for v in y]
        self.y_mean = mp.fsum(ym) / n
        std = mp.sqrt(mp.fsum([(v - self.y_mean) ** 2 for v in ym]) / n)
        self.y_std = std if std != 0 else mp.mpf(1)
        yn = [from_mp((v - self.y_mean) / self.y_std) for v in ym]
        self.yn = (np.array([a for a, _ in yn]), np.array([b for _, b in yn]))
        z = forward_rows(self.L[0], self.L[1], self.yn[0][None, :].copy(), self.yn[1][None, :].copy(), n)
        self.alpha_ = backward(self.L[0], self.L[1], z[0][0], z[1][0], n)

    def cross(self, Xt_scaled, rows=None):
        B = self.Xs if rows is None else rows
        return cross_cov(np.ascontiguousarray(Xt_scaled), np.ascontiguousarray(B), self.code, self.c)

    def mean(self, Ks):
        """mu (mpmath list) from the cross covariances to the n training rows."""
        h, l = _matvec(np.ascontiguousarray(Ks[0][:, :self.n]), np.ascontiguousarray(Ks[1][:, :self.n]),
                       *self.alpha_)
        return [to_mp(a, b) * self.y_std + self.y_mean for a, b in zip(h, l)]

    def extend(self, Ps):
        """Append the scaled rows Ps to the factor (Kriging-believer conditioning): the Cholesky of the Schur
        complement, row by row.  Returns the new pivots (pairs) and the cross covariances of Ps to the n rows."""
        r0 = self.rows
        allrows = np.vstack([self.Xs] + ([self.Pall] if r0 > self.n else []) + [Ps])
        Kn = self.cross(Ps, allrows)
        for q in range(len(Ps)):
            Kn[0][q, r0 + q], Kn[1][q, r0 + q] = self.diag
        info = chol_rows(Kn[0], Kn[1], r0, self.L[0], self.L[1], r0, r0 + len(Ps), self.BLOCK)
        if info:
            raise ValueError(f"the extended K is not positive definite at row {info}")
        self.Pall = allrows[self.n:]
        self.rows = r0 + len(Ps)
        idx = np.arange(r0, self.rows)
        return (self.L[0][idx, idx].copy(), self.L[1][idx, idx].copy()), Kn

    def variance(self, Ks, ends):
        """sigma^2 (mpmath lists, data units) at each prefix length in `ends` of the (extended) factor; Ks the cross
        covariances to every row of the factor."""
        m = max(ends)
        V = forward_rows(self.L[0], self.L[1], Ks[0], Ks[1], m)
        S = _sumsq_prefix(V[0], V[1], np.asarray(ends, dtype=np.int64))
        s2 = self.y_std ** 2
        return [[(self.prior - to_mp(S[t, q, 0], S[t, q, 1])) * s2 for t in range(len(S))]
                for q in range(len(ends))]

    def lml(self):
        n = self.n
        yy = to_mp(*_dot(self.yn[0], self.yn[1], self.alpha_[0], self.alpha_[1], 0, n))
        logdet = mp.fsum(mp.log(to_mp(self.L[0][i, i], self.L[1][i, i])) for i in range(n))
        return -yy / 2 - logdet - n * mp.log(2 * mp.pi) / 2

    def lml_grad(self):
        """d lml / d theta in sklearn's order (log of const, length scale(s), white; each when present)."""
        n = self.n
        Wt = inverse_t(self.L[0], self.L[1], n)
        ard = bool(np.iterable(self.case["ls"]))
        G = _sum_rows(_grad_rows(Wt[0], Wt[1], self.alpha_[0], self.alpha_[1], self.Xs, self.code, self.c, ard))
        g = [to_mp(*G[q]) / 2 for q in range(len(G))]
        out = ([g[0]] if self.case.get("const") is not None else []) + g[1:-1]
        if self.case.get("white") is not None:
            out.append(g[-1] * mp.mpf(self.white))
        return np.array([float(v) for v in out])

    def residual(self, K, a):
        """max |y_n - K a| / max |y_n| for a given fp64 K and a, evaluated in double-double."""
        r = _residual_rows(np.ascontiguousarray(K, dtype=float), np.ascontiguousarray(a, dtype=float), *self.yn)
        return float(np.max(r)) / float(np.max(np.abs(self.yn[0])))


def solve_rows(fit, Bh, Bl):
    """K^-1 B[t] for every row t of B, through the factor of `fit`."""
    n = fit.n
    V = forward_rows(fit.L[0], fit.L[1], Bh, Bl, n)
    return backward_rows(fit.L[0], fit.L[1], V[0], V[1], n)


def posterior_grad(fit, xs, Kg, W):
    """The input gradients of the posterior at the scaled rows xs, whose cross covariances to the n training rows are
    Kg (pair of (m, n) arrays): U = K^-1 k* per row (pair), and G = cross_cov_grad with the weights [W; u_t] of each
    row t, so that G[t, q, j] = sum_i W[q, i] dk*_ti / dx_j for the rows q of W (the same for every t) and
    G[t, -1, j] = u_t . dk*_t / dx_j.  With W = alpha_: d mu / dx_j = s_y G[t, 0, j] and
    d sigma^2 / dx_j = -2 s_y^2 G[t, -1, j]."""
    n, m = fit.n, len(xs)
    U = solve_rows(fit, *Kg)
    q = len(W[0])
    Wh = np.ascontiguousarray(np.concatenate([np.broadcast_to(W[0], (m, q, n)), U[0][:, None, :]], axis=1))
    Wl = np.ascontiguousarray(np.concatenate([np.broadcast_to(W[1], (m, q, n)), U[1][:, None, :]], axis=1))
    G = cross_cov_grad(np.ascontiguousarray(xs), fit.Xs, fit.code, fit.c, 1.0 / ls_vec(fit.case), Wh, Wl)
    return U, G


@njit(parallel=True, cache=False)
def feature_sums(Xs, omega, b, W, grad):
    """F[t, p] = sum_l W[l, p] cos(omega_l . xs_t + b_l) at the scaled rows Xs (m, d), and with `grad`
    S[t, p, j] = sum_l W[l, p] sin(omega_l . xs_t + b_l) omega_lj (else an empty S).  The phase is sum_j omega_lj xs_tj
    in order j, then + b_l; the sums over l run in order; rows t in parallel."""
    m, d = Xs.shape
    L, q = W.shape
    Fh = np.zeros((m, q))
    Fl = np.zeros((m, q))
    ms = m if grad else 0
    Sh = np.zeros((ms, q, d))
    Sl = np.zeros((ms, q, d))
    for t in prange(m):
        for l in range(L):
            ph, pl = 0.0, 0.0
            for j in range(d):
                xh, xl = two_prod(omega[l, j], Xs[t, j])
                ph, pl = dd_add(ph, pl, xh, xl)
            ph, pl = dd_add(ph, pl, b[l], 0.0)
            ch, cl, sh, sl = dd_cos_sin(ph, pl)
            for p in range(q):
                xh, xl = dd_mul_d(ch, cl, W[l, p])
                Fh[t, p], Fl[t, p] = dd_add(Fh[t, p], Fl[t, p], xh, xl)
                if grad:
                    uh, ul = dd_mul_d(sh, sl, W[l, p])
                    for j in range(d):
                        vh, vl = dd_mul_d(uh, ul, omega[l, j])
                        Sh[t, p, j], Sl[t, p, j] = dd_add(Sh[t, p, j], Sl[t, p, j], vh, vl)
    return Fh, Fl, Sh, Sl


@njit(parallel=True, cache=False)
def _rows_dot(Ah, Al, Bh, Bl):
    """O[t, p] = sum_i A[t, i] B[p, i] in order i (rows t in parallel)."""
    m, n = Ah.shape
    q = Bh.shape[0]
    Oh = np.zeros((m, q))
    Ol = np.zeros((m, q))
    for t in prange(m):
        for p in range(q):
            Oh[t, p], Ol[t, p] = _dot(Ah[t], Al[t], Bh[p], Bl[p], 0, n)
    return Oh, Ol


@njit(cache=False)
def _abs_sums(Vh, Vl):
    """sum_i |V[p, i]| per row p, in order i."""
    q, n = Vh.shape
    out = np.zeros((q, 2))
    for p in range(q):
        for i in range(n):
            h, l = (Vh[p, i], Vl[p, i]) if Vh[p, i] >= 0.0 else (-Vh[p, i], -Vl[p, i])
            out[p, 0], out[p, 1] = dd_add(out[p, 0], out[p, 1], h, l)
    return out


class Paths:
    """Posterior sample paths of a Fit (DESIGN.md 4.7, bayesianoptimization_b200/paths.py) on the draws
    (omega (L, d), b (L,), w (L, q), eps (n, q)) of paths.draw_path_inputs, in double-double:

        Phi(xs) = sqrt(2c/L) cos(omega xs + b)             (no WhiteKernel term: a path is the latent function)
        V       = K^-1 (y_n - Phi(Xs) w - eps)             (K's diagonal c + white + alpha, as the Fit's)
        path(x) = s_y (Phi(xs) w + c k(xs, Xs) V) + y_mean

    The cross covariances c k(xs, Xs) carry no WhiteKernel term either.  V is (q, n), a pair."""

    def __init__(self, fit, omega, b, w, eps):
        mp.mp.dps = 50
        self.fit = fit
        self.omega = np.ascontiguousarray(omega, dtype=float)
        self.b = np.ascontiguousarray(b, dtype=float)
        self.w = np.ascontiguousarray(w, dtype=float)
        self.eps = np.asarray(eps, dtype=float)
        self.fs = mp.sqrt(2 * mp.mpf(fit.c) / self.omega.shape[0])
        fs = _pair(self.fs)
        Fh, Fl, _, _ = feature_sums(fit.Xs, self.omega, self.b, self.w, False)
        q, n = self.w.shape[1], fit.n
        Rh, Rl = np.empty((q, n)), np.empty((q, n))
        for p in range(q):
            for i in range(n):
                th, tl = dd_mul(Fh[i, p], Fl[i, p], fs[0], fs[1])
                th, tl = dd_sub(fit.yn[0][i], fit.yn[1][i], th, tl)
                Rh[p, i], Rl[p, i] = dd_sub(th, tl, self.eps[i, p], 0.0)
        self.V = solve_rows(fit, Rh, Rl)

    def normalised(self, xs, Ks=None):
        """Phi(xs) w + c k(xs, Xs) V (mpmath, (m, q) nested lists) at the scaled rows xs; Ks their cross covariances to
        the training rows when the caller has them."""
        xs = np.ascontiguousarray(xs)
        Ks = self.fit.cross(xs) if Ks is None else Ks
        Fh, Fl, _, _ = feature_sums(xs, self.omega, self.b, self.w, False)
        Uh, Ul = _rows_dot(Ks[0], Ks[1], self.V[0], self.V[1])
        return [[to_mp(Fh[t, p], Fl[t, p]) * self.fs + to_mp(Uh[t, p], Ul[t, p]) for p in range(Fh.shape[1])]
                for t in range(len(Fh))]

    def values(self, xs, Ks=None):
        """Path values (mpmath, (m, q) nested lists, data units) at the scaled rows xs."""
        f = self.fit
        return [[f.y_std * v + f.y_mean for v in row] for row in self.normalised(xs, Ks)]

    def grads(self, xs):
        """d path / dx (mpmath, (m, q, d) nested lists, unscaled input coordinates) at the scaled rows xs: the feature
        term through sin, the update term through cross_cov_grad."""
        f = self.fit
        xs = np.ascontiguousarray(xs)
        (m, d), (q, n) = xs.shape, self.V[0].shape
        _, _, Sh, Sl = feature_sums(xs, self.omega, self.b, self.w, True)
        Wh = np.ascontiguousarray(np.broadcast_to(self.V[0], (m, q, n)))
        Wl = np.ascontiguousarray(np.broadcast_to(self.V[1], (m, q, n)))
        inv_ls = 1.0 / ls_vec(f.case)
        Gh, Gl = cross_cov_grad(xs, f.Xs, f.code, f.c, inv_ls, Wh, Wl)
        return [[[f.y_std * (to_mp(Gh[t, p, j], Gl[t, p, j]) - self.fs * to_mp(Sh[t, p, j], Sl[t, p, j]) * inv_ls[j])
                  for j in range(d)] for p in range(q)] for t in range(m)]

    def v_abs_sums(self):
        """sum_i |V[p, i]| per path (mpmath)."""
        return [to_mp(a, b) for a, b in _abs_sums(self.V[0], self.V[1])]

    def bounds(self):
        """B_p = |y_mean| + s_y (sqrt(2c/L) sum_l |w_lp| + c sum_i |V_pi|) >= |path_p(x)| everywhere (mpmath)."""
        f = self.fit
        sv = self.v_abs_sums()
        return [abs(f.y_mean) + f.y_std * (self.fs * mp.fsum(abs(mp.mpf(float(a))) for a in self.w[:, p])
                                           + f.c * sv[p]) for p in range(len(sv))]

    def train_identity(self, i, p):
        """y_mean + s_y (y_n,i - eps_ip - (white + alpha) V_pi): the value of path p at training row i in exact
        arithmetic (K V = r with K's diagonal c + white + alpha, and c k(X_i, X_i) = c)."""
        f = self.fit
        s2 = to_mp(*f.diag) - f.c
        r = to_mp(f.yn[0][i], f.yn[1][i]) - mp.mpf(self.eps[i, p]) - s2 * to_mp(self.V[0][p, i], self.V[1][p, i])
        return f.y_mean + f.y_std * r


def acquisitions(mu, var, y_max, kappa, xi):
    """UCB, EI and PoI at 50 digits from mu and sigma^2 (mpmath lists); mpmath's Phi and phi."""
    mp.mp.dps = 50
    out = dict(sd=[], acq_ucb=[], acq_ei=[], acq_poi=[])
    for m, v in zip(mu, var):
        sd = mp.sqrt(v) if v > 0 else mp.mpf(0)
        ucb = m + kappa * sd
        a = m - mp.mpf(y_max) - mp.mpf(xi)
        if sd == 0:
            e, p = max(a, mp.mpf(0)), mp.mpf(1 if a > 0 else 0)
        else:
            z = a / sd
            e, p = a * mp.ncdf(z) + sd * mp.npdf(z), mp.ncdf(z)
        for k, x in zip(out, (sd, ucb, e, p)):
            out[k].append(float(x))
    return {k: np.array(v) for k, v in out.items()}


def posterior(case, X, y, xt, kappa, xi, with_grad=True):
    """The results of make_illcond.exact (mu, var, sd, acq_*, alpha_, prior, y_std, lml, lml_grad) in double-double,
    rounded to fp64, and the Fit."""
    fit = Fit(case, X, y)
    Ks = fit.cross(scaled(case, xt))
    mu = fit.mean(Ks)
    var = fit.variance(Ks, [fit.n])[0]
    res = dict(mu=np.array([float(v) for v in mu]), var=np.array([float(v) for v in var]))
    res.update(acquisitions(mu, var, float(np.max(y)), kappa, xi))
    res["alpha_"] = fit.alpha_[0] + fit.alpha_[1]
    res["prior"] = float(fit.prior)
    res["y_std"] = float(fit.y_std)
    res["lml"] = float(fit.lml())
    if with_grad:
        res["lml_grad"] = fit.lml_grad()
    return res, fit


def l_dense(fit, n=None):
    """The factor rounded to fp64."""
    n = fit.n if n is None else n
    return fit.L[0][:n, :n] + fit.L[1][:n, :n]
