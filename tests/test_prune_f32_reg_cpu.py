"""The margin of the register-fragment fp32 Gram bound pass of pruning (predict_bound_gram_reg_kernel, the default at
d <= 16; csrc/predict16.cuh, DESIGN.md 4.9), restated in numpy and checked on adversarial inputs.

The pass evaluates the covariance as predict_bound_gram_kernel<COV, true> does (cov_f32, with the same R and Q) and
differs in three places, restated here:
  * the |k| maximum: the pass keeps the least clamped fp32 argument s~ per candidate (rows >= n excluded) and evaluates
    k~ (1 - u (R + Q z~)) once, at that s~.  cov_f32 is a function of s~ alone, so this is the per-row lower bound of
    that row, and so no larger than max_i k_i;
  * W: per row, the operand image holds (|a| R, |a| Q) in fp32 (a = alpha_i in fp32), and W += k~ fma(z~, |a| Q, |a| R);
  * the fp32 mu partial spans the thread's two rows of two consecutive n8 tiles (4 rows, as before, in the kernel's
    order), then goes into the fp64 sum.
The bound the pass applies is unchanged:
    dmu = constv (A1 (Lip dr2 + 64 u53 + 1e-30 + 3 g_np) + u W (1 + (np + 16) 2^-23)) (1 + 2^-20),
    kmax_lb = constv k~ (1 - u (R + Q z~)) |_{least s~} (1 - 2^-22) - constv (Lip dr2 + 64 u53 + 1e-30).
Every fp32 operation is emulated with IEEE rounding (fused multiply-adds through fp64, where the product is exact), and
rsqrtf / exp2f are moved by up to 2 ulp in either direction, as in test_prune_f32_cpu.py.
"""
import numpy as np
import pytest

from test_prune_f32_cpu import ABS, COV, MU_SUM_R, U, U32, F, cov_exact, cov_f32, fmaf, inputs
from test_prune_gram_cpu import CG, LIP

CHUNK = 64  # PA_CHUNK: rows per ring slot


def mu_groups(np_):
    """Row indices of every fp32 mu partial, in summation order: warp row slab rs (32 rows of a chunk), thread column
    t4, tile pair q; rows t * 8 + 2 t4 + j for t = 2q, 2q + 1 and j = 0, 1."""
    out = []
    for c0 in range(0, np_, CHUNK):
        for rs in range(2):
            for t4 in range(4):
                for q in range(2):
                    out.append([c0 + rs * 32 + t * 8 + 2 * t4 + j for t in (2 * q, 2 * q + 1) for j in (0, 1)])
    return np.array(out)


def clamp_arg(kind, r2):
    return np.minimum(np.maximum(np.asarray(r2, dtype=np.float64).astype(F), F(2.0 ** -100)), F(COV[kind][0]))


def emulate_reg_pass(kind, X, x, alpha, constv, sign, rs):
    """mu interval and kmax_lb of one candidate tile as predict_bound_gram_reg_kernel forms them."""
    n, d = X.shape
    _, R, Q = COV[kind]
    lip = LIP[kind]
    np_ = n + (-n) % 128
    x2, y2 = np.sum(x * x, 1), np.sum(X * X, 1)
    r2g = (x2[:, None] + y2[None, :]) - 2.0 * (x @ X.T)  # the Gram form, in some order
    e = np.full(r2g.shape, sign) if sign else rs.randint(-2, 3, size=r2g.shape)
    kt, z = cov_f32(kind, r2g, e, e)
    s = clamp_arg(kind, r2g)
    # rows n .. np - 1: zero operand rows (r~^2 = 0, s~ = 2^-100), alpha_ and weights 0, out of the least s~
    pad = np_ - n
    kt = np.pad(kt, ((0, 0), (0, pad)), constant_values=F(1.0))
    z = np.pad(z, ((0, 0), (0, pad)), constant_values=F(0.0))
    af = np.pad(alpha.astype(F), (0, pad))
    aR, aQ = (np.abs(af) * F(R)).astype(F), (np.abs(af) * F(Q)).astype(F)
    # mu: fp32 over the four rows of each group, then fp64
    mu = np.zeros(x.shape[0])
    for grp in mu_groups(np_):
        mp = np.zeros(x.shape[0], dtype=F)
        for r in grp:
            mp = fmaf(af[r], kt[:, r], mp)
        mu += mp.astype(np.float64)
    mu *= constv
    W = np.zeros(x.shape[0], dtype=F)
    for r in range(np_):
        W = fmaf(kt[:, r], fmaf(z[:, r], aQ[r], aR[r]), W)
    # kmax: k~ (1 - u (R + Q z~)) at the least s~, evaluated as the row's own (the same MUFU error)
    imin = np.argmin(s, 1)
    rows = np.arange(x.shape[0])
    k0, z0 = cov_f32(kind, r2g[rows, imin], e[rows, imin], e[rows, imin])
    kl = fmaf((k0 * F(-U32)).astype(F), fmaf(z0, F(Q), F(R)), k0).astype(np.float64)
    a1 = np.sum(np.abs(alpha))
    gk, gn = (d + 2) * U / (1 - (d + 2) * U), np_ * U / (1 - np_ * U)
    dr2 = CG * gk * (x2 + np.max(y2))
    dk1 = lip * dr2 + 64 * U + ABS
    wr = W.astype(np.float64) * U32 * (1 + (np_ + 16) * 2.0 ** -23)
    dmu = constv * (1 + 2.0 ** -20) * (a1 * (dk1 + 3 * gn) + wr)
    out = 1 + 8 * U  # the kernel rounds every step outward; a few ulps here stand for that
    lo, hi = mu - dmu * out, mu + dmu * out
    kmax_lb = np.maximum(0.0, constv * kl * (1 - 2.0 ** -22) / out - constv * dk1 * out)
    return lo, hi, kmax_lb, dmu


def test_weights_cover_the_w_terms():
    """Per row, k~ fma(z~, fp32(|a| Q), fp32(|a| R)) is within 3 u of |a| k~ (R + Q z~): the two roundings of the
    weights and the fma's, as the two of the ring kernel's |a| k~ and fma(z~, Q, R), so (np + 16) 2^-23 still covers W."""
    rs = np.random.RandomState(5)
    a = (rs.randn(20000) * 10.0 ** rs.uniform(-6, 6, 20000)).astype(F)
    z = rs.uniform(0, 90, 20000).astype(F)
    k = rs.uniform(0, 1, 20000).astype(F)
    for kind, (_, R, Q) in COV.items():
        aR, aQ = (np.abs(a) * F(R)).astype(F), (np.abs(a) * F(Q)).astype(F)
        t = (k.astype(np.float64) * fmaf(z, aQ, aR).astype(np.float64))
        exact = np.abs(a.astype(np.float64)) * k.astype(np.float64) * (R + Q * z.astype(np.float64))
        assert np.all(np.abs(t - exact) <= 3 * U32 * exact + 1e-300), kind


@pytest.mark.parametrize("kind", sorted(COV))
def test_least_argument_gives_a_lower_bound(kind):
    """At every s~, k~ (1 - u (R + Q z~)) <= the exact k at any r^2 that rounds and clamps to s~ (the argument of the
    row the pass keeps), for every combination of worst-case MUFU errors."""
    _, R, Q = COV[kind]
    rs = np.random.RandomState(11)
    r2 = np.concatenate([np.logspace(-9, 4, 6001), rs.uniform(0, 2 * COV[kind][0], 20000)])
    k = cov_exact(kind, r2)
    for er in (-2, 0, 2):
        for ee in (-2, 0, 2):
            kt, z = cov_f32(kind, r2, er, ee)
            kl = fmaf((kt * F(-U32)).astype(F), fmaf(z, F(Q), F(R)), kt).astype(np.longdouble)
            assert np.all(kl <= k + ABS), (kind, er, ee)


def test_mu_partial_spans_four_rows():
    """Each fp32 mu partial holds four distinct rows, and the partials cover every row once: the 6 u of R that the
    ring kernel's comment counts for its four-row partial (MU_SUM_R) covers this one too."""
    g = mu_groups(4096)
    assert g.shape[1] == 4 and MU_SUM_R >= 1 + 4 + 1
    assert np.array_equal(np.sort(g.ravel()), np.arange(4096))


@pytest.mark.parametrize("d", (2, 16))
@pytest.mark.parametrize("case", ("uniform", "near_dup", "ard"))
@pytest.mark.parametrize("kind", sorted(COV))
def test_mu_interval_and_kmax_hold(kind, case, d):
    rs = np.random.RandomState(d * 37 + len(case))
    X, x = inputs(d, case, rs, n=250)
    ls = 0.5 * np.sqrt(d)
    X, x = X / ls, x / ls
    alpha = rs.randn(X.shape[0]) * 10.0 ** rs.uniform(-2, 3, X.shape[0])
    constv = 1.7
    r2 = np.sum((x[:, None, :].astype(np.longdouble) - X[None, :, :]) ** 2, 2)
    k = cov_exact(kind, r2)
    mu = constv * np.sum(k * alpha[None, :].astype(np.longdouble), 1)
    kmax = constv * np.max(k, 1)
    for sign in (2, -2, 0):
        lo, hi, kmax_lb, dmu = emulate_reg_pass(kind, X, x, alpha, constv, sign, rs)
        assert np.all(lo <= mu) and np.all(mu <= hi), (kind, case, d, sign)
        assert np.all(kmax_lb <= kmax), (kind, case, d, sign)
        used = np.max(np.abs(0.5 * (lo + hi) - mu) / dmu)
        print(f"{kind} {case} d={d} mufu {sign:+d}: max |mu~ - mu| / dmu {float(used):.3f}")
