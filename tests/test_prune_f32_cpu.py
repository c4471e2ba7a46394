"""The margin of the fp32 Gram bound pass of pruning (predict_bound_gram_kernel<COV, true>, cov_f32, csrc/predict16.cuh;
DESIGN.md 4.9), restated in numpy and checked on adversarial inputs.

The pass rounds the Gram distance r~^2 to fp32, evaluates the covariance with rsqrtf, exp2f and fp32 arithmetic, sums
alpha_ k~ over four rows in fp32 before the fp64 sum, and widens mu and max |k| by
    per row:  u k~ (R + Q z~) + Lip dr2 + 64 u53 + 1e-30          (u = 2^-24, z~ the exp argument's magnitude)
    dmu = constv (A1 (Lip dr2 + 64 u53 + 1e-30 + 3 g_np) + u W (1 + (np + 16) 2^-23)) (1 + 2^-20),
    W = sum_i |alpha_i| k~_i (R + Q z~_i),
    kmax_lb = constv max_i k~_i (1 - u (R + Q z~_i)) (1 - 2^-22) - constv (Lip dr2 + 64 u53 + 1e-30).
Here every fp32 operation is emulated with IEEE rounding (numpy float32; the fused multiply-adds through fp64, where
the product is exact), and rsqrtf / exp2f return the correctly rounded value moved by up to 2 ulp (their documented
maximum error) in either direction.  The reference is the formula in extended precision at the direct distance.
"""
import numpy as np
import pytest

from test_prune_gram_cpu import CG, LIP

F = np.float32
U32 = 2.0 ** -24
U = 2.0 ** -53
# CovF32<COV>: clamp, R, Q (csrc/predict16.cuh)
COV = {"m15": (2300.0, 24.0, 8.0), "m25": (1400.0, 32.0, 8.0), "rbf": (166.0, 12.0, 4.0)}
ABS = 1e-30
MU_SUM_R = 6.0


def ulps(v, n):
    """v (float32) moved by n ulps (n < 0: towards -inf)."""
    v = np.asarray(v, dtype=F)
    for _ in range(abs(n)):
        v = np.nextafter(v, F(np.inf) if n > 0 else F(-np.inf)).astype(F)
    return v


def fmaf(a, b, c):
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(F)


def cov_f32(kind, r2, e_rsq=0, e_ex2=0):
    """cov_f32<COV> with rsqrtf / exp2f off by e_rsq / e_ex2 ulps (scalars or arrays of the same shape)."""
    r2max = COV[kind][0]
    s = np.minimum(np.maximum(np.asarray(r2, dtype=np.float64).astype(F), F(2.0 ** -100)), F(r2max))
    if kind == "rbf":
        z = (F(0.5) * s).astype(F)
        ea = (s * F(-0.72134751081466674805)).astype(F)
        return _ex2(ea, e_ex2), z
    y = _perturb((1.0 / np.sqrt(s.astype(np.float64))).astype(F), e_rsq)
    r = (s * y).astype(F)
    if kind == "m25":
        z = (r * F(2.23606801033020019531)).astype(F)
        e = _ex2((r * F(-3.22596406936645507812)).astype(F), e_ex2)
        return (fmaf(fmaf(z, F(0.33333334326744079590), F(1.0)), z, F(1.0)) * e).astype(F), z
    z = (r * F(1.73205077648162841797)).astype(F)
    e = _ex2((r * F(-2.49882102012634277344)).astype(F), e_ex2)
    return ((F(1.0) + z).astype(F) * e).astype(F), z


def _perturb(v, e):
    e = np.broadcast_to(np.asarray(e), v.shape)
    out = v.copy()
    for n in np.unique(e):
        sel = e == n
        out[sel] = ulps(v[sel], int(n))
    return out


def _ex2(ea, e):
    return _perturb(np.exp2(ea.astype(np.float64)).astype(F), e)


def cov_exact(kind, r2):
    r2 = np.asarray(r2, dtype=np.longdouble)
    if kind == "rbf":
        return np.exp(-r2 / 2)
    r = np.sqrt(r2)
    if kind == "m25":
        z = r * np.sqrt(np.longdouble(5))
        return (1 + z + z * z / 3) * np.exp(-z)
    z = r * np.sqrt(np.longdouble(3))
    return (1 + z) * np.exp(-z)


def r2_sweep(kind):
    r2max = COV[kind][0]
    edge = np.float64(F(r2max))
    v = [0.0, 1e-300, 1e-40, 2.0 ** -100, 1e-30, 1e-20, 1e-12, 1e-9, 1e-6]
    v += list(np.logspace(-6, 4, 4001))
    v += [edge * (1 + t) for t in np.linspace(-1e-5, 1e-5, 41)]
    v += [2 * edge, 1e6, 1e30, 1e300]
    rs = np.random.RandomState(7)
    v += list(rs.uniform(0, 2 * edge, 20000))
    return np.array(v)


@pytest.mark.parametrize("kind", sorted(COV))
def test_row_error_within_margin(kind):
    """|k~ - k(r^2)| <= u k~ (R - 6 + Q z~) + 1e-30 at every r^2, for every combination of worst-case MUFU errors."""
    _, R, Q = COV[kind]
    r2 = r2_sweep(kind)
    k = cov_exact(kind, r2)
    worst = 0.0
    for er in (-2, 0, 2):
        for ee in (-2, 0, 2):
            kt, z = cov_f32(kind, r2, er, ee)
            bound = U32 * kt.astype(np.float64) * ((R - MU_SUM_R) + Q * z.astype(np.float64)) + ABS
            err = np.abs(kt.astype(np.longdouble) - k)
            assert np.all(err <= bound), (kind, er, ee, r2[np.argmax(err / bound)])
            worst = max(worst, float(np.max(err / bound)))
    print(f"{kind}: largest error / margin {worst:.3f}")


def inputs(d, case, rs, n=256, m=96):
    if case == "uniform":
        X, x = rs.uniform(size=(n, d)), rs.uniform(size=(m, d))
    elif case == "near_dup":
        X = rs.uniform(size=(n, d))
        x = np.vstack([X[: m // 2] + 1e-9 * rs.randn(m // 2, d), X[: m // 2]])
    else:  # ARD over six decades: the coordinates / length scales span 1e-3 .. 1e3
        sc = 10.0 ** rs.uniform(-3, 3, size=d)
        X, x = rs.uniform(size=(n, d)) * sc, rs.uniform(size=(m, d)) * sc
        x[: m // 4] = X[: m // 4] * (1 + 1e-7)
    return X, x


def emulate_pass(kind, X, x, alpha, constv, sign, rs):
    """mu interval and kmax_lb of one candidate tile as the kernel forms them (MUFU errors: +2, -2 or random)."""
    n, d = X.shape
    _, R, Q = COV[kind]
    lip = LIP[kind]
    x2, y2 = np.sum(x * x, 1), np.sum(X * X, 1)
    r2g = (x2[:, None] + y2[None, :]) - 2.0 * (x @ X.T)  # the Gram form, in some order
    e = np.full(r2g.shape, sign) if sign else rs.randint(-2, 3, size=r2g.shape)
    kt, z = cov_f32(kind, r2g, e, e[::-1, ::-1] if not sign else e)
    af = alpha.astype(F)
    w = fmaf(z, F(Q), F(R))
    # mu: fp32 over four rows, then fp64
    mp = np.zeros((x.shape[0], (n + 3) // 4), dtype=F)
    for j in range(4):
        mp = fmaf(np.pad(af, (0, (-n) % 4))[j::4][None, :], np.pad(kt, ((0, 0), (0, (-n) % 4)))[:, j::4], mp)
    mu = constv * np.sum(mp.astype(np.float64), 1)
    W = np.zeros(x.shape[0], dtype=F)
    for i in range(n):
        W = fmaf((np.abs(af[i]) * kt[:, i]).astype(F), w[:, i], W)
    kl = np.max(fmaf((kt * F(-U32)).astype(F), w, kt), 1).astype(np.float64)
    a1 = np.sum(np.abs(alpha))
    np_ = n + (-n) % 128
    gk, gn = (d + 2) * U / (1 - (d + 2) * U), np_ * U / (1 - np_ * U)
    dr2 = CG * gk * (x2 + np.max(y2))
    dk1 = lip * dr2 + 64 * U + ABS
    wr = W.astype(np.float64) * U32 * (1 + (np_ + 16) * 2.0 ** -23)
    dmu = constv * (1 + 2.0 ** -20) * (a1 * (dk1 + 3 * gn) + wr)
    out = 1 + 8 * U  # the kernel rounds every step outward; a few ulps here stand for that
    lo, hi = mu - dmu * out, mu + dmu * out
    kmax_lb = np.maximum(0.0, constv * kl * (1 - 2.0 ** -22) / out - constv * dk1 * out)
    return lo, hi, kmax_lb, dmu


@pytest.mark.parametrize("d", (2, 16, 17, 32))
@pytest.mark.parametrize("case", ("uniform", "near_dup", "ard"))
@pytest.mark.parametrize("kind", sorted(COV))
def test_mu_interval_and_kmax_hold(kind, case, d):
    rs = np.random.RandomState(d * 31 + len(case))
    X, x = inputs(d, case, rs)
    ls = 0.5 * np.sqrt(d)
    X, x = X / ls, x / ls
    alpha = rs.randn(X.shape[0]) * 10.0 ** rs.uniform(-2, 3, X.shape[0])
    constv = 1.7
    r2 = np.sum((x[:, None, :].astype(np.longdouble) - X[None, :, :]) ** 2, 2)
    k = cov_exact(kind, r2)
    mu = constv * np.sum(k * alpha[None, :].astype(np.longdouble), 1)
    kmax = constv * np.max(k, 1)
    for sign in (2, -2, 0):
        lo, hi, kmax_lb, dmu = emulate_pass(kind, X, x, alpha, constv, sign, rs)
        assert np.all(lo <= mu) and np.all(mu <= hi), (kind, case, d, sign)
        assert np.all(kmax_lb <= kmax), (kind, case, d, sign)
        used = np.max(np.abs(0.5 * (lo + hi) - mu) / dmu)
        print(f"{kind} {case} d={d} mufu {sign:+d}: max |mu~ - mu| / dmu {float(used):.3f}")


def test_constants_cover_first_order_error():
    """R and Q leave headroom over the first-order counts of the kernel comment (R: 23, 14.5, 5 plus 6 for the mu
    partial; Q: 7.5, 7.5, 3)."""
    need = {"m25": (23 + 6, 7.5), "m15": (14.5 + 6, 7.5), "rbf": (5 + 6, 3.0)}
    for kind, (r, q) in need.items():
        assert COV[kind][1] >= r and COV[kind][2] >= q
    # the covariance at the clamp is inside the absolute part, and the exp argument stays normal there
    for kind, (r2max, _, _) in COV.items():
        assert float(cov_exact(kind, r2max)) < 1.2e-33
        zmax = r2max / 2 if kind == "rbf" else np.sqrt((5 if kind == "m25" else 3) * r2max)
        assert zmax / np.log(2) < 126
