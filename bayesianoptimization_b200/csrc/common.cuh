// common.cuh - shared device helpers for the b200bo kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "../../include/b200bo.h"

namespace b200bo {

constexpr int kPad = 128;  // training-set size is padded to a multiple of this

// ---- acquisition kinds (B200BO_ACQ_*, include/b200bo.h) -------------------------------------
__host__ __device__ constexpr bool acq_is_nei(int kind) {
    return kind == B200BO_ACQ_NEI || kind == B200BO_ACQ_LOGNEI;
}
// CNEI / LogCNEI (DESIGN.md 4.15): every GP of the call holds fantasies; served by their own kernel instantiations
__host__ __device__ constexpr bool acq_is_cnei(int kind) {
    return kind == B200BO_ACQ_CNEI || kind == B200BO_ACQ_LOGCNEI;
}
// the kinds that average over fantasies: no single mean, fp64 on the 16-warp bulk pipes and the small-batch kernels
__host__ __device__ constexpr bool acq_uses_fantasies(int kind) { return acq_is_nei(kind) || acq_is_cnei(kind); }
__host__ __device__ constexpr bool acq_kind_valid(int kind) {
    return kind == B200BO_ACQ_UCB || kind == B200BO_ACQ_EI || kind == B200BO_ACQ_POI || kind == B200BO_ACQ_NONE ||
           kind == B200BO_ACQ_MES || kind == B200BO_ACQ_LOGEI || kind == B200BO_ACQ_LOGPOI ||
           acq_uses_fantasies(kind) || kind == B200BO_ACQ_MEAN;
}
// The log-space kinds: the value is -(alpha + sum_j log p_j), the constraint factors summed as logs.  NEI = false in
// the kernels built without NEI / LogNEI (DESIGN.md 4.13), which then test for LogEI and LogPoI only.
template <bool NEI = true>
__host__ __device__ constexpr bool acq_constraints_in_log(int kind) {
    return kind == B200BO_ACQ_LOGEI || kind == B200BO_ACQ_LOGPOI || (NEI && kind == B200BO_ACQ_LOGNEI);
}
// The kinds of one GP that selection pruning bounds (prune_bound_key, predict16.cuh; DESIGN.md 4.9)
__host__ __device__ constexpr bool acq_prunable(int kind) {
    return kind == B200BO_ACQ_EI || kind == B200BO_ACQ_UCB || kind == B200BO_ACQ_POI ||
           acq_constraints_in_log<false>(kind);
}

// ---- input transform (B200BO_XFORM_*, include/b200bo.h) -----------------------------------
// The reference's per-dimension np.round (half to even: rint), then sklearn's division by the length scale before
// differencing: cdist(X / length_scale, Y / length_scale) (SK/gaussian_process/kernels.py:1716-1720).  Training rows and
// candidates go through the same rule, or every K* entry is wrong.  xform: [d] transform codes, or nullptr (identity).
// Each use tests xform for null itself: behind a bool-valued helper the two tests compile to a materialised flag and an
// extra branch in every kernel that stages coordinates.
__host__ __device__ constexpr bool xform_rounds(int code) { return code == B200BO_XFORM_ROUND; }
__device__ __forceinline__ double scale_input(double v, const int* xform, const double* ls, int j) {
    if (xform && xform_rounds(xform[j])) v = rint(v);
    return v / ls[j];
}

// ---- branch-free fp64 primitives for the covariance functions -----------------------------
// The kernel-matrix builders evaluate sqrt and exp for every (training point, candidate) pair
// with only a few resident warps, so data-dependent slow-path branches (libm special cases) and
// their code size hurt more than the arithmetic.  Both routines are within 2 ulp of libm on their
// domain (checked against numpy over 3e5 random arguments), far inside the 1e-5 parity bar.  Composed into a
// covariance, exp amplifies the relative error of its argument k by k, so cov_eval is within a few ulp times (1 + k)
// of sklearn's formula evaluated exactly (tests/test_gpu_illcond.py holds it to 4 (1 + k) ulp up to k = 700).

// Polynomial / reduction constants live in constant memory: an fp64 immediate costs two uniform
// moves every time it is used, a constant-bank operand is free.
__constant__ double kExpC[14] = {
    1.6059043836821613e-10, 2.0876756987868100e-09, 2.5052108385441720e-08, 2.7557319223985893e-07,
    2.7557319223985888e-06, 2.4801587301587302e-05, 1.9841269841269841e-04, 1.3888888888888889e-03,
    8.3333333333333332e-03, 4.1666666666666664e-02, 1.6666666666666666e-01, 0.5, 1.0, 1.0};
__constant__ double kExpR[4] = {1.4426950408889634074, -6.93147180369123816490e-01,
                                -1.90821492927058770002e-10, 700.0};

// sqrt(x) for x >= 0.  Arguments below about 1e-30 are treated as about 1e-30 (|error| <= 1e-15 absolute), arguments
// above about 1e38 as about 1e38: the float seed of one above FLT_MAX is rsqrtf(inf) = 0, which made the result 0 and
// a Matern covariance at a huge distance its maximum.  The result there, about 1e19, lies far inside exp_neg's clamp,
// so every covariance built on it is still its limit 0 (below 1e-265).  Both clamps act on the high word of the bits
// (an integer min/max: the order of non-negative doubles is the order of their high words), so they stay off the
// fp64 pipe that bounds phase A; between the clamps the argument is used unchanged.
__device__ __forceinline__ double sqrt_pos(double x) {
    const int hi = min(max(__double2hiint(x), 0x39B4484B /* high word of 1e-30 */), 0x47D2CED3 /* of 1e38 */);
    const double xc = __hiloint2double(hi, __double2loint(x));
    double y = (double)rsqrtf((float)xc);  // 2^-23 seed
    const double h = 0.5 * xc;
    y = y * fma(-h * y, y, 1.5);
    y = y * fma(-h * y, y, 1.5);
    double s = xc * y;
    s = fma(fma(-s, s, xc), 0.5 * y, s);
    return s;
}

// x / 3.0 correctly rounded, without the division: q = RN(x RN(1/3)) is within 1 ulp of x/3, so one Markstein
// correction RN(q + RN(x - 3q) RN(1/3)) gives RN(x/3) (the residual x - 3q is exact in the FMA).  Valid for normal x
// far from overflow; the callers pass k^2 with k from sqrt_pos, i.e. x in [1e-30, 5e38].  The IEEE division it replaces
// carried a conditional call to its slow path per pair, which cut phase A's unrolled row block into branch regions
// the scheduler could not interleave.  Bit-identical to x / 3.0 (tests/test_covariance_primitives_cpu.py).
__device__ __forceinline__ double div3_rn(double x) {
    constexpr double third = 0.33333333333333331483;  // RN(1/3)
    const double q = __dmul_rn(x, third);
    const double r = fma(-q, 3.0, x);
    return fma(r, third, q);
}

// exp(-k) for k >= 0 (k > 700 is clamped: the result, < 1e-304, is irrelevant at fp64 scale).
// n = rint(-k log2e) comes from the 1.5 2^52 shift: the rounded product plus 1.5 2^52 lies in [2^52, 2^53), where the
// add rounds it to an integer half to even exactly as rint does, and the low word of the sum is n.  2^n is applied by
// an integer add to the exponent field of p (p in [sqrt(1/2), sqrt(2)], n in [-1010, 0]: the product is normal and the
// multiply it replaces was exact).  Same bits as rint / (long long) / p * 2^n, without FRND, F2I and the multiply.
__device__ __forceinline__ double exp_neg(double k) {
    constexpr double shift = 6755399441055744.0;  // 1.5 * 2^52
    k = fmin(k, kExpR[3]);
    const double t = __dadd_rn(__dmul_rn(-k, kExpR[0]), shift);
    const double n = __dsub_rn(t, shift);
    double r = fma(n, kExpR[1], -k);
    r = fma(n, kExpR[2], r);
    // degree-13 Taylor polynomial (|r| <= ln2/2: truncation 4e-18) in Estrin form: dependent
    // depth 4 instead of 13, so the few resident warps keep the fp64 pipe fed.  a_k = kExpC[13-k].
    const double r2 = r * r;
    const double b0 = fma(kExpC[12], r, kExpC[13]), b1 = fma(kExpC[10], r, kExpC[11]);
    const double b2 = fma(kExpC[8], r, kExpC[9]), b3 = fma(kExpC[6], r, kExpC[7]);
    const double b4 = fma(kExpC[4], r, kExpC[5]), b5 = fma(kExpC[2], r, kExpC[3]);
    const double b6 = fma(kExpC[0], r, kExpC[1]);
    const double r4 = r2 * r2;
    const double c0 = fma(b1, r2, b0), c1 = fma(b3, r2, b2), c2 = fma(b5, r2, b4);
    const double r8 = r4 * r4;
    const double d0 = fma(c1, r4, c0), d1 = fma(b6, r4, c2);
    const double p = fma(d1, r8, d0);
    const int e = (int)((unsigned)__double2loint(t) << 20);  // n in the exponent field of the high word
    return __hiloint2double(__double2hiint(p) + e, __double2loint(p));
}

// ---- covariance functions -------------------------------------------------------------
// COV codes: 0 = Matern nu=0.5, 1 = nu=1.5, 2 = nu=2.5, 3 = RBF / Matern nu=inf.
// Follows SK/gaussian_process/kernels.py:1722-1731 (Matern) and :1549/:1553 (RBF) operation by
// operation: dists = sqrt(r2); nu=2.5: K = dists*sqrt(5); (1 + K + K^2/3) * exp(-K).
template <int COV>
__device__ __forceinline__ double cov_eval(double r2) {
    if (COV == 3) return exp_neg(0.5 * r2);
    const double dist = sqrt_pos(r2);
    if (COV == 2) {
        const double k = dist * 2.23606797749978969641;  // math.sqrt(5)
        return (1.0 + k + div3_rn(k * k)) * exp_neg(k);
    }
    if (COV == 1) {
        const double k = dist * 1.73205080756887729353;  // math.sqrt(3)
        return (1.0 + k) * exp_neg(k);
    }
    return exp_neg(dist);
}

__host__ __device__ __forceinline__ int cov_code(int family, int nu) {
    return (family == B200BO_KERNEL_RBF || nu == B200BO_NU_INF) ? 3 : nu;
}

__device__ __forceinline__ double cov_from_r2(double r2, int family, int nu) {
    switch (cov_code(family, nu)) {
        case 0: return cov_eval<0>(r2);
        case 1: return cov_eval<1>(r2);
        case 2: return cov_eval<2>(r2);
        default: return cov_eval<3>(r2);
    }
}

// h(r) = -(1/r) dk/dr of the unit covariance k(r), from r^2: the input gradient of k(|xs - Xs_n|) is
// -h(r) (xs - Xs_n).  RBF: k; Matern 2.5: (5/3)(1 + sqrt5 r) exp(-sqrt5 r); 1.5: 3 exp(-sqrt3 r); 0.5: exp(-r)/r.
// Matern 0.5 has a kink at a training input (h unbounded as r -> 0, the gradient's direction undefined at 0):
// h := 0 at r = 0, so that row contributes nothing.
template <int COV>
__device__ __forceinline__ double cov_dh_eval(double r2) {
    if (COV == 3) return exp_neg(0.5 * r2);
    const double dist = sqrt_pos(r2);
    if (COV == 2) {
        const double k = dist * 2.23606797749978969641;
        return (5.0 / 3.0) * (1.0 + k) * exp_neg(k);
    }
    if (COV == 1) return 3.0 * exp_neg(dist * 1.73205080756887729353);
    return r2 == 0.0 ? 0.0 : exp_neg(dist) / dist;
}

__device__ __forceinline__ double cov_dh_from_r2(double r2, int family, int nu) {
    switch (cov_code(family, nu)) {
        case 0: return cov_dh_eval<0>(r2);
        case 1: return cov_dh_eval<1>(r2);
        case 2: return cov_dh_eval<2>(r2);
        default: return cov_dh_eval<3>(r2);
    }
}

// scipy.special.ndtr (cephes ndtr.c), which scipy.stats.norm.cdf evaluates
// (SP/stats/_continuous_distns.py:370-371).
__device__ __forceinline__ double ndtr(double a) {
    if (isnan(a)) return a;
    const double x = a * 0.70710678118654752440;
    const double z = fabs(x);
    if (z < 0.70710678118654752440) return 0.5 + 0.5 * erf(x);
    double y = 0.5 * erfc(z);
    if (x > 0) y = 1.0 - y;
    return y;
}

// norm.pdf: exp(-x^2/2)/sqrt(2*pi) (SP/stats/_continuous_distns.py:362-363)
__device__ __forceinline__ double norm_pdf(double x) {
    return exp(-(x * x) / 2.0) / 2.50662827463100050242;
}

// log Psi(g) and the inverse Mills ratio psi(g) / Psi(g) of the standard normal (psi: pdf, Psi: cdf), finite and
// accurate for every finite g.  Naive log(ndtr(g)) is -inf below g ~ -38 and psi/Psi is 0/0 there, so below 0 both
// come from the scaled complementary error function: Psi(g) = erfcx(-g/sqrt2) exp(-g^2/2) / 2, hence
//   log Psi(g) = log(erfcx(-g/sqrt2) / 2) - g^2/2,    psi(g) / Psi(g) = sqrt(2/pi) / erfcx(-g/sqrt2).
// At and above 0, Psi = ndtr(g) >= 1/2 and log Psi = log1p(-ndtr(-g)) keeps the digits of a Psi close to 1.
__device__ __forceinline__ double log_ndtr(double g) {
    if (g < 0.0) return log(0.5 * erfcx(-g * 0.70710678118654752440)) - 0.5 * (g * g);
    return log1p(-ndtr(-g));
}
__device__ __forceinline__ double inv_mills(double g) {
    if (g < 0.0) return 0.79788456080286535588 / erfcx(-g * 0.70710678118654752440);
    return norm_pdf(g) / ndtr(g);
}

// log(1 - e^x) for x <= 0 in its two stable branches (Maechler, "Accurately Computing log(1 - exp(-|a|))", 2012):
// log(-expm1(x)) above -ln 2, log1p(-exp(x)) below.
__device__ __forceinline__ double log1mexp(double x) {
    return x > -0.69314718055994530942 ? log(-expm1(x)) : log1p(-exp(x));
}

// log h(z), h(z) = phi(z) + z Phi(z), the expected improvement in units of sigma, in the three branches of Ament et
// al. (NeurIPS 2023, eq. 9).  Below z = -1, h = phi(z) w(z) with w = 1 - sqrt(pi/2) |z| erfcx(-z/sqrt2) (Phi = phi
// sqrt(pi/2) erfcx(-z/sqrt2)), so log h = log phi + log1mexp(log(erfcx |z|) + log(pi/2)/2).  Below -1/sqrt(eps) = -2^26
// the log1mexp argument is within rounding of 0 and the asymptote w = 1/z^2 takes over.
constexpr double kLogHTail = -67108864.0;
__device__ __forceinline__ double log_h_tail_arg(double z) {
    return log(erfcx(-z * 0.70710678118654752440) * -z) + 0.22579135264472743236;
}
__device__ __forceinline__ double log_h(double z) {
    if (z > -1.0) return log(norm_pdf(z) + z * ndtr(z));
    const double log_phi = -0.5 * (z * z) - 0.91893853320467274178;
    if (z > kLogHTail) return log_phi + log1mexp(log_h_tail_arg(z));
    return log_phi - 2.0 * log(-z);
}
// d log h / dz = Phi/h = r and phi/h = q (LogEI: d = r d mean / sigma + q d sigma / sigma), finite for every finite z
// (q = z^2 overflows beyond |z| ~ 1.3e154, where its exact value does).  Below z = -1 from the same w as log_h:
// q = 1/w, r = sqrt(pi/2) erfcx(-z/sqrt2) / w; below -2^26 r = |z| and q = z^2 (relative error 1/z^2 < eps).
__device__ __forceinline__ void log_h_ratios(double z, double& r, double& q) {
    if (z > -1.0) {
        const double pz = norm_pdf(z), cz = ndtr(z), h = pz + z * cz;
        r = cz / h;
        q = pz / h;
    } else if (z > kLogHTail) {
        const double e = erfcx(-z * 0.70710678118654752440);
        const double w = -expm1(log(e * -z) + 0.22579135264472743236);
        r = 1.25331413731550025121 * e / w;
        q = 1.0 / w;
    } else {
        r = -z;
        q = z * z;
    }
}

// frozen norm(loc, scale).cdf(b) as scipy evaluates it: NaN unless scale > 0
// (rv_continuous.cdf argcheck), else ndtr((b - loc)/scale).
__device__ __forceinline__ double norm_cdf_loc_scale(double b, double loc, double scale) {
    if (!(scale > 0.0) || isnan(loc)) return CUDART_NAN;
    return ndtr((b - loc) / scale);
}

// order-preserving map double -> uint64 (for (value,index) selection keys)
__device__ __forceinline__ unsigned long long ordered_bits(double v) {
    if (v == 0.0) v = 0.0;  // -0.0 == +0.0 for np.argmin / np.argsort
    unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
// np.argmin: NaN is the minimum (first NaN wins)
__device__ __forceinline__ unsigned long long key_nan_first(double v) {
    return isnan(v) ? 0ull : ordered_bits(v);
}
// np.argsort: NaN sorts last
__device__ __forceinline__ unsigned long long key_nan_last(double v) {
    return isnan(v) ? 0xFFFFFFFFFFFFFFFFull : ordered_bits(v);
}

// ---- cp.async helpers -------------------------------------------------------------------
__device__ __forceinline__ void cp_async16_cg(void* smem_dst, const void* gmem_src) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

}  // namespace b200bo
