// predict16.cuh - 16-warp variant of the fused fp64 posterior-predict + acquisition kernel.
//
// Same fusion, tile (128 candidates x 128 rows of L^-1), k-tile (32), 3-stage cp.async pipeline and
// fixed-order reductions as predict_acq_kernel<DMMA> (predict_kernels.cuh), but 512 threads per CTA:
//   * phase B: warp tile 32(m) x 32(n) -> 32 fp64 accumulators (64 registers) per thread instead of 128,
//     the kernel fits in 128 registers/thread, and every SM sub-partition holds FOUR resident warps whose
//     LDS -> DMMA dependencies interleave (the 8-warp kernel has two: ncu showed ~6 % issue gaps inside the
//     DMMA loop, stalled_wait 4.8 / math_pipe_throttle 3.2 per issue);
//   * phase A (phase_a<P16_NT>: K* build, DFMA + sqrt/exp latency chains) runs with 16 warps, four row-quarters per
//     candidate column, so its latency-bound part shrinks;
//   * phase B runs on the sm_90 shape mma.sync m16n8k4 f64 (MMA = 1684, the default: twice the fp64 tensor rate of
//     the sm_80 shape m8n8k4 per SM and clock on H100); m8n8k4 (MMA = 884) stays selectable with
//     B200BO_PREDICT_MMA=884 for A/B measurements (DESIGN.md 4.1, 6, 6.1);
//   * phase B operands reach shared memory either by per-thread cp.async under CTA barriers (PIPE_CPASYNC) or by
//     bulk copies on an mbarrier ring (PIPE_BULK), with the L^-1 stages multicast across CTA pairs (PIPE_BULK_MC);
//     B200BO_PREDICT_PIPE selects (DESIGN.md 4.1, 6.1);
//   * L2 policy hints: the CTA-private K* scratch (written once, swept cyclically: LRU-hostile) is stored and
//     loaded evict_first; L^-1 (re-read by every CTA for every tile) is loaded evict_last on a fraction
//     P.linv_l2_last of its lines.  At N=4096 the L^-1 triangle is 67 MB, more than the 50 MB L2 of an H100, so
//     the fraction is a measured choice (DESIGN.md 6), not "keep it all".
// Selected with B200BO_PREDICT_WARPS=16 (A/B measurements decide the default, see DESIGN.md).
#pragma once
#include <type_traits>

#include <cooperative_groups.h>

#include "predict_kernels.cuh"

namespace b200bo {

constexpr int P16_NT = 512;
constexpr int P16_SPLIT = P16_NT / PBN;  // row quarters of every staged chunk in phase A

// evict_last on a fraction `frac` of the lines (the rest evict_unchanged); frac <= 0: evict_normal, i.e. no hint
__device__ __forceinline__ unsigned long long l2_policy_evict_last(float frac) {
    unsigned long long p;
    if (frac > 0.f)
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, %1;\n" : "=l"(p) : "f"(frac));
    else
        asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
__device__ __forceinline__ void cp_async16_cg_hint(void* smem_dst, const void* gmem_src, unsigned long long pol) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "l"(pol));
}

// ---- selection-only pruning: the bound pass ------------------------------------------------------------------
// For the selection of the k smallest closure values -acq (EI, UCB, PoI, LogEI, LogPoI on one GP; DESIGN.md 4.9,
// 4.12), a key per candidate
// that no candidate's exact key can be below: key_nan_last(v_lb) with v_lb <= -acq(mu, sigma).
//   sigma^2 = prior - k*^T K^-1 k* <= prior - max_i k*_i^2 / K_ii (Cauchy-Schwarz in the K^-1 inner product) = var_ub;
//   eps * prior absorbs the rounding of the explicit-inverse sum of squares the exact value is computed from;
//   EI and UCB (as max(mu, mu + kappa sigma)) do not decrease with sigma, nor does PoI while a = mu - y_max - xi < 0
//   (PoI <= 1 otherwise); v_lb is lowered by a relative and an absolute margin against the rounding of ndtr / pdf.
//   LogEI and LogPoI are the logs of EI and PoI, so the same monotonicity holds (LogPoI <= 0 for a >= 0).  Their
//   rounding error is absolute: up to a few ulps of |log h| + |log sigma| (the two can cancel), and in the tail of
//   log h it grows with z^2 ~ 2 |value|.  The margin is 1e-9 |value| + 1e-9 (kPruneLogAbsMargin): the floor covers
//   |log sigma| <= 745 with 1e4 headroom, the relative part the tail with about 1e6.
// mu is known as an interval [mu_lo, mu_hi] that holds the epilogue's mu (normalised units): a point (mu_lo = mu_hi,
// bit-equal to the epilogue's: the same phase A, the same order of sums) from the direct bound pass, a margin around the
// Gram form's mu from the Gram bound pass (predict_bound_gram_kernel).  Every kind above increases with mu, so v_lb is
// evaluated at mu_hi.
// Key 0 (never pruned): mu_lo, mu_hi or v_lb non-finite, or the interval of a widened by a few ulps contains 0 (sigma
// = 0 with a = 0 gives the NaN that np.argmin reports first).
constexpr double kPruneVarEps = 1e-8, kPruneRelMargin = 1e-9, kPruneAbsMargin = 1e-300, kPruneLogAbsMargin = 1e-9;

// var_ub: an upper bound of sigma^2 in normalised units, margin included:
//   max(0, min(prior, prior - r + eps * prior)) with r <= k*^T K^-1 k* (prune_var_ub)
__device__ __forceinline__ double prune_var_ub(const GpDev& G, double r) {
    return fmax(0.0, fmin(G.prior, G.prior - r + kPruneVarEps * G.prior));
}

__device__ __forceinline__ unsigned long long prune_bound_key(const PredictParams& P, const GpDev& G, double mu_lo,
                                                              double mu_hi, double var_ub) {
    const double mean = G.y_std * mu_hi + G.y_mean, mean_lo = G.y_std * mu_lo + G.y_mean;
    const double sd = sqrt(var_ub * (G.y_std * G.y_std));
    const double a = mean - P.y_max - P.xi, a_lo = mean_lo - P.y_max - P.xi;
    double base, scale;
    if (P.acq_kind == B200BO_ACQ_UCB) {
        base = fmax(mean, mean + P.kappa * sd);
        scale = fabs(mean) + fabs(P.kappa * sd);
    } else if (P.acq_kind == B200BO_ACQ_EI) {
        base = ei_term(a, sd);
        scale = fabs(base);
    } else if (acq_constraints_in_log<false>(P.acq_kind)) {
        base = (P.acq_kind == B200BO_ACQ_LOGPOI && a >= 0.0) ? 0.0 : log_acq_term(P.acq_kind, a, sd);
        scale = fabs(base) + kPruneLogAbsMargin / kPruneRelMargin;
    } else {
        base = a < 0.0 ? ndtr(a / sd) : 1.0;
        scale = fabs(base);
    }
    const double v_lb = -base - (kPruneRelMargin * scale + kPruneAbsMargin);
    const double tol = 8.0 * 2.220446049250313e-16 * (fmax(fabs(mean), fabs(mean_lo)) + fabs(P.y_max) + fabs(P.xi));
    const bool a_near_0 = P.acq_kind != B200BO_ACQ_UCB && a_lo <= tol && a >= -tol;
    if (!isfinite(mean) || !isfinite(mean_lo) || !isfinite(v_lb) || a_near_0) return 0ull;
    return key_nan_last(v_lb);
}

// One CTA per tile of PBN candidates: phase A without the K* stores, then (key, local index) per candidate; idx,
// kmax_out (max_i |K*_i|, for b200bo_acq_prune_bound_dev) and mu_out ((mu, mu) with mu = K* alpha_, the epilogue's
// value bit for bit; the refine stages key with it) may be nullptr.
template <bool DREG>
__global__ void __launch_bounds__(P16_NT) predict_bound_kernel(const PredictParams P, unsigned long long* keys,
                                                               int* idx, double* kmax_out, double2* mu_out) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ double kmax_s[P16_SPLIT][PBN];
    const long long c0 = (long long)blockIdx.x * PBN;
    const GpDev& G = P.gp[0];
    phase_a<P16_NT, DREG, KS_KMAX>(P, G, c0, nullptr, smem, mu_s, 0ull, kmax_s, nullptr, P.m, G.np);
    const int c = threadIdx.x;
    if (c < PBN && c0 + c < P.m) {
        const double mu_n = ((mu_s[0][c] + mu_s[1][c]) + mu_s[2][c]) + mu_s[3][c];
        const double kmax = fmax(fmax(kmax_s[0][c], kmax_s[1][c]), fmax(kmax_s[2][c], kmax_s[3][c]));
        keys[c0 + c] = prune_bound_key(P, G, mu_n, mu_n, prune_var_ub(G, kmax * kmax / G.kdiag));
        if (idx) idx[c0 + c] = (int)(c0 + c);
        if (mu_out) mu_out[c0 + c] = make_double2(mu_n, mu_n);
        if (kmax_out) kmax_out[c0 + c] = kmax;
    }
}

// B200BO_ACQ_MEAN (include/b200bo.h, DESIGN.md 4.17): the mean-only tile kernel.  A persistent grid of CTAs shaped as
// the direct bound pass (P16_NT threads, the same phase A without K* stores), each folding its tiles of PBN candidates
// into one running selection list.  Per tile, phase A of every GP in j order; mu = K* alpha_ in the tile kernel's order
// of the four parts and de-normalised with candidate_epilogue's expression, so mu_0 is bit-equal to the mean
// predict_acq16_kernel (b200bo_gp_predict) gives the batch; then the merit.  No K* scratch, no L^-1, no phase B.
template <bool DREG>
__global__ void __launch_bounds__(P16_NT) predict_mean_kernel(const PredictParams P) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ double mu0_s[PBN], viol_s[PBN];
    __shared__ SelShared sel_s;
    const int tid = threadIdx.x;
    if (P.sel_cta) {
        if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
        __syncthreads();
    }
    const long long ntiles = (P.m + PBN - 1) / PBN;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long c0 = tile * PBN;
        for (int g = 0; g < P.n_gps; ++g) {
            const GpDev& G = P.gp[g];
            phase_a<P16_NT, DREG, KS_NONE>(P, G, c0, nullptr, smem, mu_s, 0ull, nullptr, nullptr, P.m, G.np);
            if (tid < PBN) {
                const int c = tid;
                const long long gi = c0 + c;
                const double mu_n = ((mu_s[0][c] + mu_s[1][c]) + mu_s[2][c]) + mu_s[3][c];
                const double mean = G.y_std * mu_n + G.y_mean;
                if (g == 0) {
                    mu0_s[c] = mean;
                    viol_s[c] = 0.0;
                    if (P.mu_out && gi < P.m) P.mu_out[gi] = mean;
                } else {
                    viol_s[c] = __dadd_rn(viol_s[c], mean_viol(G, mean));
                }
                if (g == P.n_gps - 1) {
                    const double val = mean_merit_neg(mu0_s[c], viol_s[c], P.mean_T);
                    if (P.acq_out && gi < P.m) P.acq_out[gi] = val;
                    if (P.sel_cta) runsel_update<1>(sel_s, P.sel_k, tid, val, gi + P.index_base, gi < P.m);
                }
            }
            __syncthreads();
        }
    }
    if (P.sel_cta && tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
}

// failed polls before a wait gives up: seconds, against microseconds for a stage to arrive from L2 or HBM
constexpr uint32_t kPipeWaitBudget = 1u << 28;
// set by a ring wait (the bulk-copy phase B, the Gram bound pass) that ran out of its budget; the host reports it as an
// error and clears it before every launch.  A global, not a launch parameter, so that the k-loop holds no register for
// it.
__device__ unsigned long long g_pipe_timeout;

// ---- selection-only pruning: the Gram bound pass (DESIGN.md 4.9) ----------------------------------------------------
// The direct pass spends about 40 % (d = 16) to 55 % (d = 32) of its fp64 instructions per (candidate, training row)
// pair on the distance.  Here the distance comes from the fp64 tensor pipe in the Gram form
//   r~^2 = [x, |x|^2, 1] . [-2y, 1, |y|^2]     (x = candidate / ls, y = Xs_i; K = d + 2 terms)
// as one m16n8k4 f64 GEMM per tile, and the covariance, the mu sum and the |k| max are all that is left on the CUDA
// cores.  The Gram form cancels (DESIGN.md 7), so mu and max |k| come out as intervals around the exact path's values:
//   r^2      Every DMMA product-add is assumed IEEE-rounded, in any order (tests/test_gpu_prune_gram.py checks the
//            device's r~^2 against this bound).  With S = |x|^2 + Ymax from the rounded norms, u = 2^-53 and
//            g_n = n u / (1 - n u):  Gram sum <= g_K sum|a_k b_k| <= 2 g_K S (1 + g_d),  rounded norms <= g_d S,
//            and phase A's direct sum of squared differences (the value compared against) <= (g_d + 2u) 2 S, so
//            |r~^2 - r^2_direct| <= 5 g_{d+2} S (1 + O(g)) <= kGramCg g_{d+2} S = dr2.
//   k        |dk/d(r^2)| <= Lip (Matern-2.5: 5/6, Matern-1.5: 3/2, RBF: 1/2 - plus e^{dr2/2} for r~^2 < 0, inside the
//            slack below; Matern-0.5 is unbounded at r = 0 and keeps the direct pass).  cov_eval is within
//            4 (1 + k) ulp of the formula (common.cuh), under 8 u for RBF, 12 u for Matern-1.5, 15 u for Matern-2.5
//            in absolute terms, so both evaluations and the product with constv stay under kGramCcov u:
//            dk = constv (Lip dr2 + kGramCcov u) bounds |k~_i - k_i| for every row i.
//   mu       |mu~ - mu| <= A1 dk + (rounding of both sums, any order of np terms: 2 g_np A1 constv, and the final
//            product with constv) <= A1 (dk + 3 g_np constv) (1 + 2^-20) = dmu, the last factor for the rounding of A1.
//   max |k|  max_i |k_i| >= constv max_i k~_i - dk = kmax_lb.
// mu_lo / mu_hi and kmax_lb are rounded outward (directed rounding).  With these, prune_bound_key and prune_var_ub
// give a key no larger than the direct pass's, so the same candidates can be pruned, less a few near the k-th key.
constexpr double kGramCg = 6.0, kGramCcov = 64.0;

// row stride (doubles) of the Gram operands: K = d + 2 rounded up to the k-step 4, then to an odd multiple of 4, so
// that the 8 rows x 4 k-columns of a fragment load fall on distinct banks within each half-warp
__host__ __device__ inline int gram_stride(int d) {
    const int k = (d + 2 + 3) / 4 * 4;
    return (k / 4) & 1 ? k : k + 4;
}

// ---- the fp32 covariance of the Gram bound pass (predict_bound_gram_kernel<COV, true>) ------------------------------
// r~^2 is rounded to fp32 and clamped to [2^-100, kF32R2Max]: above the clamp the exp argument would leave the normal
// range (2^-126), and the covariance there is below 1.2e-33 (Matern-2.5 at 1400, Matern-1.5 at 2300, RBF at 166),
// inside the absolute part of the margin; below it rsqrtf stays finite.  sqrt and exp are one rsqrtf and one exp2f
// (each within 2 ulp, CUDA C++ Programming Guide, single-precision mathematical functions), the rest is FMA-pipe work:
//   Matern-2.5: z = sqrt5 r,  k = (1 + z + z^2/3) 2^(-sqrt5 log2e r);   Matern-1.5: z = sqrt3 r, k = (1 + z) 2^(...);
//   RBF: z = s / 2, k = 2^(-log2e s / 2).
// Error against the formula at the exact r~^2 (u = 2^-24; first order, every constant and product rounded):
//   r = s rsqrtf(s) is within 5 u, z and the exp argument within 7 u, plus 1/2 u from the rounding of r~^2 to s;
//   the exp argument's error x is a relative error z x of 2^(...), so it grows with z; the Matern polynomial (positive
//   terms) is within 2 x 7.5 u + 3 u, exp2f within 4 u, the last product u.  Per row, with z~ from the pass,
//     |k~ - k| <= u k~ (R + Q z~) + (clamps: < 1e-30),
//   R = 23, 14.5, 5 and Q = 7.5, 7.5, 3 (Matern-2.5, Matern-1.5, RBF) - the constants below leave headroom and add the
//   fp32 mu partial of the kernel (alpha_ rounded to fp32, four fused products: 6 u relative to sum |alpha_ k~|).
//   tests/test_prune_f32_cpu.py restates this with rsqrtf and exp2f perturbed to their documented error and
//   tests/test_gpu_prune_f32.py checks the device function exhaustively over its fp32 arguments.
// sqrt and exp2 run as rsqrt.approx.ftz and ex2.approx.ftz: on the clamped domain their arguments and results are
// normal fp32 numbers, where these return the same bits as rsqrtf / exp2f without the denormal guards around them.
template <int COV>
struct CovF32 {
    static constexpr float r2max = COV == 1 ? 2300.f : COV == 2 ? 1400.f : 166.f;
    static constexpr float rel = COV == 1 ? 24.f : COV == 2 ? 32.f : 12.f;  // R, the mu partial included
    static constexpr float qz = COV == 3 ? 4.f : 8.f;                       // Q
    // the exp2 argument per unit s (RBF) or r (Matern): -log2e / 2, -sqrt3 log2e, -sqrt5 log2e
    static constexpr float ex2c = COV == 1 ? -2.49882102012634277344f
                                  : COV == 2 ? -3.22596406936645507812f
                                             : -0.72134751081466674805f;
};
// Conditions for the ftz forms: s >= 2^-100 keeps rsqrt's argument and result normal, and at s = r2max the exp2
// argument (-119.8, -120.7, -119.7 for Matern-1.5, Matern-2.5, RBF) stays above -126, so 2^(...) is normal too
static_assert(CovF32<3>::r2max * CovF32<3>::ex2c > -126.f, "RBF: exp2 argument below the normal range");
static_assert(CovF32<1>::r2max * CovF32<1>::ex2c * CovF32<1>::ex2c < 126.f * 126.f, "Matern-1.5: exp2 argument");
static_assert(CovF32<2>::r2max * CovF32<2>::ex2c * CovF32<2>::ex2c < 126.f * 126.f, "Matern-2.5: exp2 argument");
constexpr double kF32Abs = 1e-30;  // the clamps, per unit covariance

__device__ __forceinline__ float rsqrt_ftz(float x) {
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// s: r~^2 (fp64) rounded to fp32 and clamped to [2^-100, r2max]
template <int COV>
__device__ __forceinline__ float cov_f32_arg(double r2) {
    return fminf(fmaxf(__double2float_rn(r2), 0x1p-100f), CovF32<COV>::r2max);
}

// k~ of one pair from its clamped fp32 argument s; z: the exp argument's magnitude (natural units)
template <int COV>
__device__ __forceinline__ float cov_f32_s(float s, float& z) {
    if (COV == 3) {
        z = 0.5f * s;
        return ex2_ftz(s * CovF32<COV>::ex2c);
    }
    const float r = s * rsqrt_ftz(s);
    if (COV == 2) {
        z = r * 2.23606801033020019531f;  // sqrt5
        const float e = ex2_ftz(r * CovF32<COV>::ex2c);
        return fmaf(fmaf(z, 0.33333334326744079590f, 1.f), z, 1.f) * e;
    }
    z = r * 1.73205077648162841797f;  // sqrt3
    const float e = ex2_ftz(r * CovF32<COV>::ex2c);
    return (1.f + z) * e;
}

// k~ of one pair from r~^2 (fp64)
template <int COV>
__device__ __forceinline__ float cov_f32(double r2, float& z) {
    return cov_f32_s<COV>(cov_f32_arg<COV>(r2), z);
}

// the per-row margin weights of the register-fragment fp32 pass (predict_bound_gram_reg_kernel): (|a| R, |a| Q) in
// fp32, a = alpha_i in fp32
template <int COV>
__device__ __forceinline__ float2 gram_row_weights(float a) {
    return make_float2(fabsf(a) * CovF32<COV>::rel, fabsf(a) * CovF32<COV>::qz);
}

// training-side operand, once per fit: row i < n = [-2 Xs_i | 1 | |Xs_i|^2 | 0 ...], zero rows for i >= n; behind A1
// and Ymax, alpha_ in fp32 (0 for i >= n) for the fp32 passes, then the margin weights of the covariance cov
// (gram_row_weights; zero for Matern-0.5, which has no Gram pass)
__global__ void __launch_bounds__(256) gram_operand_kernel(const double* __restrict__ Xs, const double* __restrict__ alphav,
                                                           int n, int np, int d, int cov, double* __restrict__ img) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= np) return;
    const int str = gram_stride(d);
    float* af = reinterpret_cast<float*>(img + (size_t)np * str + 2);
    const float a = i < n ? (float)alphav[i] : 0.f;
    af[i] = a;
    reinterpret_cast<float2*>(af + np)[i] = cov == 1   ? gram_row_weights<1>(a)
                                            : cov == 2 ? gram_row_weights<2>(a)
                                            : cov == 3 ? gram_row_weights<3>(a)
                                                       : make_float2(0.f, 0.f);
    double* row = img + (size_t)i * str;
    double y2 = 0.0;
    for (int j = 0; j < d; ++j) {
        const double v = Xs[(size_t)i * d + j];
        y2 = fma(v, v, y2);
        row[j] = i < n ? -2.0 * v : 0.0;
    }
    for (int j = d; j < str; ++j) row[j] = 0.0;
    if (i < n) {
        row[d] = 1.0;
        row[d + 1] = y2;
    }
}

// A1 = sum_i |alpha_i| and Ymax = max_i |Xs_i|^2 (i < n) behind the operand image; one CTA, fixed order
__global__ void __launch_bounds__(1024) gram_stats_kernel(const double* __restrict__ alphav, int n, int d,
                                                          double* __restrict__ img, double* __restrict__ stats) {
    __shared__ double sa[1024], sy[1024];
    const int t = threadIdx.x, str = gram_stride(d);
    double a = 0.0, y = 0.0;
    for (int i = t; i < n; i += 1024) {
        a += fabs(alphav[i]);
        y = fmax(y, img[(size_t)i * str + d + 1]);
    }
    sa[t] = a;
    sy[t] = y;
    __syncthreads();
    for (int s = 512; s > 0; s >>= 1) {
        if (t < s) {
            sa[t] += sa[t + s];
            sy[t] = fmax(sy[t], sy[t + s]);
        }
        __syncthreads();
    }
    if (t == 0) {
        stats[0] = sa[0];
        stats[1] = sy[0];
    }
}

// The chunks of the Gram operand reach shared memory through a ring of kGramSlots slots, each a bulk copy of the
// chunk's PA_CHUNK operand rows and alpha_ words (fp32 for the fp32 pass, fp64 otherwise) completing on the slot's
// mbarrier, as phase B's PIPE_BULK ring: every warp counts its consumption of a slot, and the last of the 8 refills it
// with the chunk kGramSlots ahead.  No CTA barrier separates the chunks, so warps drift up to kGramSlots - 1 chunks
// apart and one warp's DMMAs issue while another's covariances do.  A CTA is 8 warps over a tile of kGramTile
// candidates, so that several CTAs (3 at d <= 16 in the fp32 pass, at most 80 registers) share an SM and hide each
// other's latencies, prologue and epilogue.  4 slots fit at d = B200BO_MAX_DIM.
constexpr int kGramSlots = 4, kGramTile = 64, kGramNT = 256;
__host__ __device__ inline size_t gram_slot_doubles(int d) { return (size_t)PA_CHUNK * (gram_stride(d) + 1); }
// dynamic shared memory of predict_bound_gram_kernel: the candidate operand [kGramTile][stride], then the ring
__host__ __device__ inline size_t gram_bound_smem(int d) {
    return sizeof(double) * ((size_t)kGramTile * gram_stride(d) + kGramSlots * gram_slot_doubles(d));
}

// The covariance, mu partial and |k| maximum of one thread's 16 pairs of a chunk (acc[mi][ni][e]: candidate
// (2 mi + (e >> 1)) * 8 + g, row ni * 8 + 2 t4 + (e & 1) of the warp's slab).  MASK: the slab holds rows >= n, whose
// covariance is taken as 0; only the last chunks can.
template <int COV, bool F32, bool MASK>
__device__ __forceinline__ void gram_chunk_cov(const double (&acc)[2][2][4], int nrow, const double* al,
                                               const float* alf, double (&macc)[4], double (&kmx)[4],
                                               float (&kmxf)[4], float (&wsum)[4]) {
    if constexpr (F32) {
        float mp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int i = 2 * mi + (e >> 1), r = ni * 8 + (e & 1);
                    float z;
                    float k = cov_f32<COV>(acc[mi][ni][e], z);
                    if (MASK && r >= nrow) k = 0.f;
                    const float a = alf[r];
                    const float w = fmaf(z, CovF32<COV>::qz, CovF32<COV>::rel);
                    mp[i] = fmaf(a, k, mp[i]);
                    wsum[i] = fmaf(fabsf(a) * k, w, wsum[i]);
                    kmxf[i] = fmaxf(kmxf[i], fmaf(k * -0x1p-24f, w, k));
                }
#pragma unroll
        for (int i = 0; i < 4; ++i) macc[i] += (double)mp[i];
    } else {
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int i = 2 * mi + (e >> 1), r = ni * 8 + (e & 1);
                    double k = cov_eval<COV>(acc[mi][ni][e]);
                    if (MASK && r >= nrow) k = 0.0;
                    macc[i] = fma(al[r], k, macc[i]);
                    kmx[i] = fmax(kmx[i], k);
                }
    }
}

// One CTA per tile of kGramTile candidates.  Warp w owns candidates (w & 1) * 32 .. +32 and rows (w >> 1) * 16 .. +16
// of every PA_CHUNK-row chunk: 2 x 2 m16n8k4 tiles (m: candidates, n: training rows) over ceil(K / 4) k-steps.  Thread
// (g, t4) accumulates candidates i * 8 + g (i < 4) of its warp over rows 2 t4, 2 t4 + 1 (+ 8) of its slab, chunks in
// ascending order; the partials are added over the quad, then over the four row slabs in a fixed order.  Outputs as
// predict_bound_kernel's; mu_out gets (mu_lo, mu_hi) and kmax_out kmax_lb.  A ring wait that runs out of its budget
// sets g_pipe_timeout.
// F32: the covariance in fp32 (cov_f32).  Per thread and chunk the four alpha_ k~ products of a candidate are summed in
// fp32 and then added to the fp64 partial; W = sum_i |alpha_i| k~_i (R + Q z~_i) (fp32) carries the relative part of
// the margin, and the |k| maximum is taken over k~_i (1 - u (R + Q z~_i)), a lower bound of the row's exact k:
//   dmu = constv (A1 (Lip dr2 + 64 u53 + kF32Abs + 3 g_np) + u W (1 + (np + 16) 2^-23)) (1 + 2^-20)
//   kmax_lb = constv (max_i k~_i (1 - u (R + Q z~_i))) (1 - 2^-22) - constv (Lip dr2 + 64 u53 + kF32Abs)
// (every fp32 sum of positive terms is within (np + 16) 2^-23 of its value; 2^-22 covers the rounding of the product).
template <int COV, bool F32>
__global__ void __launch_bounds__(kGramNT, F32 ? 3 : 2)
    predict_bound_gram_kernel(const PredictParams P, unsigned long long* keys, int* idx, double* kmax_out,
                              double2* mu_out) {
    static_assert(COV != 0, "Matern-0.5 has no Lipschitz bound in r^2");
    constexpr double lip = COV == 1 ? 1.5 : COV == 2 ? 5.0 / 6.0 : 0.5;
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[4][kGramTile];
    __shared__ double kmax_s[4][kGramTile];
    __shared__ double w_s[F32 ? 4 : 1][kGramTile];
    __shared__ uint64_t full_bar[kGramSlots];
    __shared__ unsigned done_cnt[kGramSlots];
    const GpDev& G = P.gp[0];
    const int tid = threadIdx.x, d = P.d, str = gram_stride(d), nks = (d + 2 + 3) / 4;
    const long long c0 = (long long)blockIdx.x * kGramTile;
    double* xa_s = smem;                            // [kGramTile][str]: [x | |x|^2 | 1 | 0 ...]
    double* ring = smem + (size_t)kGramTile * str;  // slot s: [PA_CHUNK][str] operand rows, then PA_CHUNK alpha_ words
    const double* stats = G.gram + (size_t)G.np * str;  // A1, Ymax, then alpha_ in fp32
    const int nch = G.np / PA_CHUNK;
    // one thread: chunk ch into the free slot s
    auto copy = [&](int ch, int s) {
        constexpr uint32_t abytes = PA_CHUNK * (F32 ? sizeof(float) : sizeof(double));
        const uint32_t obytes = PA_CHUNK * str * sizeof(double);
        double* dst = ring + s * gram_slot_doubles(d);
        tc::mbar_arrive_expect_tx(&full_bar[s], obytes + abytes);
        tc::bulk_g2s(dst, G.gram + (size_t)ch * PA_CHUNK * str, obytes, &full_bar[s]);
        const void* asrc = F32 ? (const void*)(reinterpret_cast<const float*>(stats + 2) + (size_t)ch * PA_CHUNK)
                               : (const void*)(G.alphav + (size_t)ch * PA_CHUNK);
        tc::bulk_g2s(dst + PA_CHUNK * str, asrc, abytes, &full_bar[s]);
    };
    if (tid == 0) {  // the first chunks load while the candidates are built
        for (int s = 0; s < kGramSlots; ++s) {
            tc::mbar_init(&full_bar[s], 1);
            done_cnt[s] = 0;
        }
        tc::mbar_fence_init();
        for (int s = 0; s < kGramSlots && s < nch; ++s) copy(s, s);
    }
    for (int q = tid; q < kGramTile * str; q += kGramNT) {
        const int c = q / str, j = q - c * str;
        const long long gi = c0 + c;
        double v = j == d + 1 ? 1.0 : 0.0;
        if (j < d && gi < P.m) v = scale_input(candidate_coord(P, gi, j), G.xform, G.ls, j);  // as phase A builds them
        xa_s[q] = v;
    }
    __syncthreads();  // coordinates visible
    if (tid < kGramTile) {
        double x2 = 0.0;
        for (int j = 0; j < d; ++j) x2 = fma(xa_s[tid * str + j], xa_s[tid * str + j], x2);
        xa_s[tid * str + d] = x2;
    }
    __syncthreads();  // norms |x|^2 and the ring's barriers visible
    const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
    const int cg = warp & 1, rg = warp >> 1;
    const double* xa = xa_s + (size_t)(cg * 32 + g) * str + t4;
    double macc[4], kmx[4];
    float kmxf[4], wsum[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        macc[i] = kmx[i] = 0.0;
        kmxf[i] = wsum[i] = 0.f;
    }
    // chunk ch through the DMMA Gram product and the covariance section; MASK: the chunk holds rows >= n
    auto chunk = [&](int ch, auto mask) {
        const int s = ch % kGramSlots;
        tc::mbar_wait_budget(&full_bar[s], (uint32_t)(ch / kGramSlots) & 1u, &g_pipe_timeout, kPipeWaitBudget);
        const double* buf = ring + s * gram_slot_doubles(d);
        const double* xb = buf + (size_t)(rg * 16 + g) * str + t4;
        double acc[2][2][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.0;
#pragma unroll 1  // unrolled, the k-steps take the registers that a third CTA per SM needs
        for (int ks = 0; ks < nks; ++ks) {
            double a[4], b[2];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = xa[(size_t)i * 8 * str + 4 * ks];
#pragma unroll
            for (int ni = 0; ni < 2; ++ni) b[ni] = xb[(size_t)ni * 8 * str + 4 * ks];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int ni = 0; ni < 2; ++ni)
                    dmma1684(acc[mi][ni][0], acc[mi][ni][1], acc[mi][ni][2], acc[mi][ni][3], a[2 * mi],
                             a[2 * mi + 1], b[ni]);
        }
        const double* al = buf + PA_CHUNK * str + rg * 16 + 2 * t4;
        const float* alf = reinterpret_cast<const float*>(buf + PA_CHUNK * str) + rg * 16 + 2 * t4;
        const int nrow = G.n - (ch * PA_CHUNK + rg * 16 + 2 * t4);  // slab rows r < nrow of this thread are < n
        gram_chunk_cov<COV, F32, decltype(mask)::value>(acc, nrow, al, alf, macc, kmx, kmxf, wsum);
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();  // this warp's reads of slot s happen before its count
            if ((atomicAdd(&done_cnt[s], 1u) & 7u) == 7u) {  // last of the 8 warps: refill with chunk ch + kGramSlots
                __threadfence_block();
                tc::fence_proxy_async_smem();
                if (ch + kGramSlots < nch) copy(ch + kGramSlots, s);
            }
        }
    };
    // the chunks below n / PA_CHUNK hold no padded row; the mask stays out of their loop (and its code size)
    const int nfull = G.n / PA_CHUNK;
    int ch = 0;
    for (; ch < nfull; ++ch) chunk(ch, std::false_type{});
    for (; ch < nch; ++ch) chunk(ch, std::true_type{});
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (F32) {
            wsum[i] += __shfl_xor_sync(0xffffffffu, wsum[i], 1);
            wsum[i] += __shfl_xor_sync(0xffffffffu, wsum[i], 2);
            kmx[i] = (double)kmxf[i];
        }
        macc[i] += __shfl_xor_sync(0xffffffffu, macc[i], 1);
        macc[i] += __shfl_xor_sync(0xffffffffu, macc[i], 2);
        kmx[i] = fmax(kmx[i], __shfl_xor_sync(0xffffffffu, kmx[i], 1));
        kmx[i] = fmax(kmx[i], __shfl_xor_sync(0xffffffffu, kmx[i], 2));
        if (t4 == 0) {
            mu_s[rg][cg * 32 + i * 8 + g] = macc[i];
            kmax_s[rg][cg * 32 + i * 8 + g] = kmx[i];
            if (F32) w_s[rg][cg * 32 + i * 8 + g] = wsum[i];
        }
    }
    __syncthreads();
    const int c = tid;
    if (c < kGramTile && c0 + c < P.m) {
        const double u = 0x1p-53;
        const double gk = (d + 2) * u / (1.0 - (d + 2) * u), gn = G.np * u / (1.0 - G.np * u);
        const double dr2 = __dmul_ru(kGramCg * gk, __dadd_ru(xa_s[c * str + d], stats[1]));
        const double mu = G.constv * (((mu_s[0][c] + mu_s[1][c]) + mu_s[2][c]) + mu_s[3][c]);
        const double kt = fmax(fmax(kmax_s[0][c], kmax_s[1][c]), fmax(kmax_s[2][c], kmax_s[3][c]));
        double dmu, kmax_lb;
        if constexpr (F32) {
            const double dk1 = __fma_ru(lip, dr2, kGramCcov * u + kF32Abs);  // per unit covariance and row
            const double w = __dadd_ru(__dadd_ru(w_s[0][c], w_s[1][c]), __dadd_ru(w_s[2][c], w_s[3][c]));
            const double wr = __dmul_ru(__dmul_ru(w, 0x1p-24), 1.0 + (G.np + 16) * 0x1p-23);
            dmu = __dmul_ru(__dmul_ru(G.constv, 1.0 + 0x1p-20),
                            __fma_ru(stats[0], __dadd_ru(dk1, 3.0 * gn), wr));
            kmax_lb = fmax(0.0, __dsub_rd(__dmul_rd(__dmul_rd(G.constv, kt), 1.0 - 0x1p-22), __dmul_ru(G.constv, dk1)));
        } else {
            const double dk = __dmul_ru(G.constv, __fma_ru(lip, dr2, kGramCcov * u));
            dmu = __dmul_ru(__dmul_ru(stats[0], 1.0 + 0x1p-20), __fma_ru(3.0 * gn, G.constv, dk));
            kmax_lb = fmax(0.0, __dsub_rd(__dmul_rd(G.constv, kt), dk));
        }
        const double mu_lo = __dsub_rd(mu, dmu), mu_hi = __dadd_ru(mu, dmu);
        keys[c0 + c] = prune_bound_key(P, G, mu_lo, mu_hi, prune_var_ub(G, kmax_lb * kmax_lb / G.kdiag));
        if (idx) idx[c0 + c] = (int)(c0 + c);
        if (mu_out) mu_out[c0 + c] = make_double2(mu_lo, mu_hi);
        if (kmax_out) kmax_out[c0 + c] = kmax_lb;
    }
}

// ---- the fp32 Gram bound pass with the candidate operand in registers (d <= 16; DESIGN.md 4.9) -----------------------
// predict_bound_gram_kernel<COV, true> keeps the candidate fragments in shared memory and runs each chunk as a DMMA
// phase and then a covariance phase, so a warp never has tensor and XU / FMA work ready at once.  Here, with the same
// launch contract, outputs, ring and candidate build:
//   * warp w owns candidates (w & 3) * 16 .. +16 and rows (w >> 2) * 32 .. +32 of every chunk: one m16 slab, whose
//     NKS k-step fragments (2 doubles each, NKS = ceil((d + 2) / 4) <= 5) are loaded into registers once; per chunk
//     4 n8 tiles x NKS DMMAs read only the training operand from the ring;
//   * the DMMAs of the next n8 tile (the first tile of the next chunk after the fourth) issue before the covariances of
//     the current one, so every warp has both kinds of work in flight.  Two tiles of accumulators are live (16
//     registers): with two halves of 2 tiles (32) beside the 20 fragment registers the kernel spills at 80;
//   * per pair, one FMNMX keeps the least s~ (cov_f32_arg) per candidate instead of the max of k~ (1 - u (R + Q z~));
//     the epilogue evaluates that lower bound once, at the least s~: cov_f32_s is a function of s~ alone, so it is the
//     row's own lower bound, no larger than the row's exact k and so than max_i k_i;
//   * W takes the per-row weights (|alpha_i| R, |alpha_i| Q) of the operand image: W += k~ fma(z~, |a| Q, |a| R), two
//     roundings per term before the sum as before (|a| k~ and fma(z~, Q, R)), so (np + 16) 2^-23 still covers the sum.
// The mu partial still spans four rows in fp32 (2 n8 tiles x 2 rows per thread and candidate), so R and Q are
// CovF32's.  Thread (g, t4) accumulates candidates g, g + 8 of its slab; partials are added over the quad, then over the
// two row slabs.  dmu and kmax_lb as predict_bound_gram_kernel<COV, true>'s.  A slot is counted as consumed after the
// warp's covariances of its fourth tile, its last read of the slot's operand rows, alpha_ words and weights.
constexpr int kGramRegMaxDim = 16;
// slot of the register-fragment pass: [PA_CHUNK][str] operand rows, PA_CHUNK alpha_ (fp32), PA_CHUNK weight pairs
__host__ __device__ inline size_t gram_reg_slot_doubles(int d) { return (size_t)PA_CHUNK * gram_stride(d) + PA_CHUNK * 3 / 2; }
__host__ __device__ inline size_t gram_reg_bound_smem(int d) {
    return sizeof(double) * ((size_t)kGramTile * gram_stride(d) + kGramSlots * gram_reg_slot_doubles(d));
}

// covariances of one thread's 4 pairs of an n8 tile (acc[e]: candidate g + 8 (e >> 1), row 2 t4 + (e & 1) of the tile;
// al / wt: alpha_ and weights of those two rows), into the fp32 mu partials mp; rows r >= nrow are >= n (MASK) and
// stay out of the least s~ (their alpha_ and weights are 0)
template <int COV, bool MASK>
__device__ __forceinline__ void gram_reg_tile_cov(const double (&acc)[4], const float* al, const float* wt, int nrow,
                                                  float (&mp)[2], float (&wsum)[2], float (&smin)[2]) {
    const float2 a = *reinterpret_cast<const float2*>(al);
    const float4 w = *reinterpret_cast<const float4*>(wt);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int i = e >> 1, j = e & 1;
        const float s = cov_f32_arg<COV>(acc[e]);
        float z;
        const float k = cov_f32_s<COV>(s, z);
        smin[i] = fminf(smin[i], MASK && j >= nrow ? INFINITY : s);
        mp[i] = fmaf(j ? a.y : a.x, k, mp[i]);
        wsum[i] = fmaf(k, fmaf(z, j ? w.w : w.y, j ? w.z : w.x), wsum[i]);
    }
}

template <int COV, int NKS>
__global__ void __launch_bounds__(kGramNT, 3)
    predict_bound_gram_reg_kernel(const PredictParams P, unsigned long long* keys, int* idx, double* kmax_out,
                                  double2* mu_out) {
    static_assert(COV != 0, "Matern-0.5 has no Lipschitz bound in r^2");
    static_assert(NKS >= 1 && 4 * NKS <= (kGramRegMaxDim + 2 + 3) / 4 * 4, "k-steps of d <= 16");
    constexpr double lip = COV == 1 ? 1.5 : COV == 2 ? 5.0 / 6.0 : 0.5;
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[2][kGramTile];
    __shared__ float w_s[2][kGramTile], s_s[2][kGramTile];
    __shared__ uint64_t full_bar[kGramSlots];
    __shared__ unsigned done_cnt[kGramSlots];
    const GpDev& G = P.gp[0];
    // gram_stride(d) of every d with NKS k-steps: the operand addresses fold into immediates
    constexpr int str = NKS & 1 ? 4 * NKS : 4 * NKS + 4;
    constexpr size_t slot_doubles = (size_t)PA_CHUNK * str + PA_CHUNK * 3 / 2;  // gram_reg_slot_doubles(d)
    const int tid = threadIdx.x, d = P.d;
    const long long c0 = (long long)blockIdx.x * kGramTile;
    double* xa_s = smem;                            // [kGramTile][str]: [x | |x|^2 | 1 | 0 ...]
    double* ring = smem + (size_t)kGramTile * str;  // slot s: gram_reg_slot_doubles
    const double* stats = G.gram + (size_t)G.np * str;  // A1, Ymax, alpha_ in fp32, then the weight pairs
    const float* alpha32 = reinterpret_cast<const float*>(stats + 2);
    const int nch = G.np / PA_CHUNK;
    // one thread: chunk ch into the free slot s
    auto copy = [&](int ch, int s) {
        constexpr uint32_t abytes = PA_CHUNK * sizeof(float), wbytes = PA_CHUNK * sizeof(float2);
        constexpr uint32_t obytes = PA_CHUNK * str * sizeof(double);
        double* dst = ring + s * slot_doubles;
        tc::mbar_arrive_expect_tx(&full_bar[s], obytes + abytes + wbytes);
        tc::bulk_g2s(dst, G.gram + (size_t)ch * PA_CHUNK * str, obytes, &full_bar[s]);
        tc::bulk_g2s(dst + PA_CHUNK * str, alpha32 + (size_t)ch * PA_CHUNK, abytes, &full_bar[s]);
        tc::bulk_g2s(dst + PA_CHUNK * str + PA_CHUNK / 2, alpha32 + G.np + (size_t)ch * PA_CHUNK * 2, wbytes,
                     &full_bar[s]);
    };
    if (tid == 0) {  // the first chunks load while the candidates are built
        for (int s = 0; s < kGramSlots; ++s) {
            tc::mbar_init(&full_bar[s], 1);
            done_cnt[s] = 0;
        }
        tc::mbar_fence_init();
        for (int s = 0; s < kGramSlots && s < nch; ++s) copy(s, s);
    }
    for (int q = tid; q < kGramTile * str; q += kGramNT) {
        const int c = q / str, j = q - c * str;
        const long long gi = c0 + c;
        double v = j == d + 1 ? 1.0 : 0.0;
        if (j < d && gi < P.m) v = scale_input(candidate_coord(P, gi, j), G.xform, G.ls, j);  // as phase A builds them
        xa_s[q] = v;
    }
    __syncthreads();  // coordinates visible
    if (tid < kGramTile) {
        double x2 = 0.0;
        for (int j = 0; j < d; ++j) x2 = fma(xa_s[tid * str + j], xa_s[tid * str + j], x2);
        xa_s[tid * str + d] = x2;
    }
    __syncthreads();  // norms |x|^2 and the ring's barriers visible
    const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
    const int cs = warp & 3, rs = warp >> 2;
    // the thread's place in a slot: operand row rs * 32 + g, column t4 (b fragments); alpha_ / weight rows
    // rs * 32 + 2 t4 (+ 1)
    const int boff = (rs * 32 + g) * str + t4, roff = rs * 32 + 2 * t4;
    double fa[NKS][2];  // a0 / a1 of k-step ks: candidates cs * 16 + g (+ 8), column 4 ks + t4
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks) {
        fa[ks][0] = xa_s[(size_t)(cs * 16 + g) * str + 4 * ks + t4];
        fa[ks][1] = xa_s[(size_t)(cs * 16 + g + 8) * str + 4 * ks + t4];
    }
    double macc[2] = {0.0, 0.0};
    float wsum[2] = {0.f, 0.f}, smin[2] = {INFINITY, INFINITY};
    // DMMAs of n8 tile t (rows rs * 32 + t * 8 .. +8) of the chunk in slot buffer buf
    auto mma = [&](double (&acc)[4], const double* buf, int t) {
        const double* xb = buf + boff + t * 8 * str;
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] = 0.0;
#pragma unroll
        for (int ks = 0; ks < NKS; ++ks) dmma1684(acc[0], acc[1], acc[2], acc[3], fa[ks][0], fa[ks][1], xb[4 * ks]);
    };
    auto slot = [&](int ch) { return ring + (ch % kGramSlots) * slot_doubles; };
    auto wait = [&](int ch) {
        tc::mbar_wait_budget(&full_bar[ch % kGramSlots], (uint32_t)(ch / kGramSlots) & 1u, &g_pipe_timeout,
                             kPipeWaitBudget);
    };
    double acc0[4], acc1[4];
    // chunk ch, whose tile 0 DMMAs are in acc0: per tile t the DMMAs of tile t + 1 (of the next chunk's tile 0 for
    // t = 3), then tile t's covariances; the mu partial is added to macc after tiles 1 and 3, and the slot released
    // after tile 3.  MASK: the chunk holds rows >= n
    auto chunk = [&](int ch, auto mask) {
        constexpr bool M = decltype(mask)::value;
        const int s = ch % kGramSlots;
        const double* buf = slot(ch);
        const float* al = reinterpret_cast<const float*>(buf + PA_CHUNK * str) + roff;
        const float* wt = reinterpret_cast<const float*>(buf + PA_CHUNK * str + PA_CHUNK / 2) + 2 * roff;
        const int nrow = G.n - (ch * PA_CHUNK + roff);  // tile 0 rows r < nrow are < n
        float mp[2] = {0.f, 0.f};
        auto flush = [&]() {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                macc[i] += (double)mp[i];
                mp[i] = 0.f;
            }
        };
        mma(acc1, buf, 1);
        gram_reg_tile_cov<COV, M>(acc0, al, wt, nrow, mp, wsum, smin);
        mma(acc0, buf, 2);
        gram_reg_tile_cov<COV, M>(acc1, al + 8, wt + 16, nrow - 8, mp, wsum, smin);
        flush();
        mma(acc1, buf, 3);
        gram_reg_tile_cov<COV, M>(acc0, al + 16, wt + 32, nrow - 16, mp, wsum, smin);
        if (ch + 1 < nch) {
            wait(ch + 1);
            mma(acc0, slot(ch + 1), 0);
        }
        gram_reg_tile_cov<COV, M>(acc1, al + 24, wt + 48, nrow - 24, mp, wsum, smin);
        flush();
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();  // this warp's reads of slot s happen before its count
            if ((atomicAdd(&done_cnt[s], 1u) & 7u) == 7u) {  // last of the 8 warps: refill with chunk ch + kGramSlots
                __threadfence_block();
                tc::fence_proxy_async_smem();
                if (ch + kGramSlots < nch) copy(ch + kGramSlots, s);
            }
        }
    };
    wait(0);
    mma(acc0, slot(0), 0);
    // the chunks below n / PA_CHUNK hold no padded row; the mask stays out of their loop (and its code size)
    const int nfull = G.n / PA_CHUNK;
    int ch = 0;
    for (; ch < nfull; ++ch) chunk(ch, std::false_type{});
    for (; ch < nch; ++ch) chunk(ch, std::true_type{});
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        macc[i] += __shfl_xor_sync(0xffffffffu, macc[i], 1);
        macc[i] += __shfl_xor_sync(0xffffffffu, macc[i], 2);
        wsum[i] += __shfl_xor_sync(0xffffffffu, wsum[i], 1);
        wsum[i] += __shfl_xor_sync(0xffffffffu, wsum[i], 2);
        smin[i] = fminf(smin[i], __shfl_xor_sync(0xffffffffu, smin[i], 1));
        smin[i] = fminf(smin[i], __shfl_xor_sync(0xffffffffu, smin[i], 2));
        if (t4 == 0) {
            mu_s[rs][cs * 16 + i * 8 + g] = macc[i];
            w_s[rs][cs * 16 + i * 8 + g] = wsum[i];
            s_s[rs][cs * 16 + i * 8 + g] = smin[i];
        }
    }
    __syncthreads();
    const int c = tid;
    if (c < kGramTile && c0 + c < P.m) {
        const double u = 0x1p-53;
        const double gk = (d + 2) * u / (1.0 - (d + 2) * u), gn = G.np * u / (1.0 - G.np * u);
        const double dr2 = __dmul_ru(kGramCg * gk, __dadd_ru(xa_s[c * str + d], stats[1]));
        const double mu = G.constv * (mu_s[0][c] + mu_s[1][c]);
        float z;
        const float k = cov_f32_s<COV>(fminf(s_s[0][c], s_s[1][c]), z);
        const double kt = (double)fmaf(k * -0x1p-24f, fmaf(z, CovF32<COV>::qz, CovF32<COV>::rel), k);
        const double dk1 = __fma_ru(lip, dr2, kGramCcov * u + kF32Abs);  // per unit covariance and row
        const double w = __dadd_ru((double)w_s[0][c], (double)w_s[1][c]);
        const double wr = __dmul_ru(__dmul_ru(w, 0x1p-24), 1.0 + (G.np + 16) * 0x1p-23);
        const double dmu =
            __dmul_ru(__dmul_ru(G.constv, 1.0 + 0x1p-20), __fma_ru(stats[0], __dadd_ru(dk1, 3.0 * gn), wr));
        const double kmax_lb =
            fmax(0.0, __dsub_rd(__dmul_rd(__dmul_rd(G.constv, kt), 1.0 - 0x1p-22), __dmul_ru(G.constv, dk1)));
        const double mu_lo = __dsub_rd(mu, dmu), mu_hi = __dadd_ru(mu, dmu);
        keys[c0 + c] = prune_bound_key(P, G, mu_lo, mu_hi, prune_var_ub(G, kmax_lb * kmax_lb / G.kdiag));
        if (idx) idx[c0 + c] = (int)(c0 + c);
        if (mu_out) mu_out[c0 + c] = make_double2(mu_lo, mu_hi);
        if (kmax_out) kmax_out[c0 + c] = kmax_lb;
    }
}

// words of PredictParams::prune_ctl
enum {
    kCtlTile = 0,     // next tile of predict_acq16_kernel's prune mode, in bound order
    kCtlKth = 1,      // least k-th key a full CTA list has published
    kCtlEval = 2,     // candidates that went through the full phase B
    kCtlRefTile = 3,  // next tile of the refine stage, in bound order
    kCtlSurv = 4,     // candidates the refine stage let through
    kCtlRefined = 5,  // candidates the refine stage looked at
    kCtlUnit = 6,      // next unit of the lead stage, the current level launch or the current final round
    kCtlKthLead = 7,   // the k-th key as it was before the lead stage
    kCtlKthRound = 8,  // the k-th key as it was before the current final round (written by merge_kth_run)
    kCtlLevel = 9,     // candidates the refine level let through
    kCtlWords = 10
};

// Prune mode of predict_acq16_kernel: thread 0 claims the next tile in bound order and stops the CTA (returns ntiles)
// once the tile's best bound key is above the least k-th key any CTA has published: every later tile's keys are
// larger still, and a CTA's k-th key bounds the global k-th key from above.  Counts the candidates it lets through.
__device__ __forceinline__ long long prune_claim(const PredictParams& P, long long ntiles, long long& tile_s) {
    if (threadIdx.x == 0) {
        long long t = (long long)atomicAdd(P.prune_ctl + kCtlTile, 1ull);
        if (t < ntiles && P.perm_key[t * PBN] > *reinterpret_cast<volatile unsigned long long*>(P.prune_ctl + kCtlKth))
            t = ntiles;
        if (t < ntiles) atomicAdd(P.prune_ctl + kCtlEval, (unsigned long long)min((long long)PBN, P.m - t * PBN));
        tile_s = t;
    }
    __syncthreads();
    return tile_s;
}

// stage loader: BK k-rows x 128 doubles of LinvT (evict_last) and of K* (evict_first), 512 threads.  NJ = 1: of K*
// only the 32 columns cb .. cb + 31 of a column group (one 16-byte copy per thread)
template <int NJ = 4>
__device__ __forceinline__ void predict16_load_stage(double* as, double* bs, const double* Ag, const double* Bg,
                                                     int np, unsigned long long pol_last,
                                                     unsigned long long pol_first, int cb = 0) {
    constexpr int STR = PSTR_DMMA, BK = PBK_DMMA;
    static_assert(NJ == 4 || BK * 16 == P16_NT, "one column-group copy per thread");
    const int tid = threadIdx.x;
#pragma unroll
    for (int t = 0; t < BK * 64 / P16_NT; ++t) {
        const int q = tid + t * P16_NT;
        const int kk = q >> 6, m2 = (q & 63) * 2;
        cp_async16_cg_hint(as + kk * STR + m2, Ag + (size_t)kk * np + m2, pol_last);
        if constexpr (NJ == 4) cp_async16_cg_hint(bs + kk * STR + m2, Bg + kk * PBN + m2, pol_first);
    }
    if constexpr (NJ == 1) {
        const int kk = tid >> 4, m2 = cb + (tid & 15) * 2;
        cp_async16_cg_hint(bs + kk * STR + m2, Bg + kk * PBN + m2, pol_first);
    }
}

// ---- phase B: mma.sync f64; 16 warps, warp tile 32(m) x 32(n); red[4][PBN] ------------------------
// MMA = 1684: m16n8k4 (sm_90, DMMA.16x8x4), the default; MMA = 884: m8n8k4 (sm_80, DMMA.8x8x4) for A/B.
// Both load the same fragments: a[i] = A(row wm*32 + i*8 + g, k-row t4), b[j] = B(k-row t4, column wn*32 + j*8 + g),
// conflict-free (PSTR_DMMA).  m16n8k4 tile mi takes a[2mi] (rows g) and a[2mi+1] (rows g+8) as its a0/a1, so its
// c0..c3 are acc[2mi][j][0..1] and acc[2mi+1][j][0..1]: acc[i][j][e] is V row wm*32 + i*8 + g, candidate
// wn*32 + j*8 + 2*t4 + e for both shapes and the epilogue is shared.
// Row blocks [ib0, ib1) of L^-1.  PART = false: red = the sums over those blocks (the whole product: 0, np / PBM).
// PART = true (predict_units_kernel): nothing is summed across row blocks; every thread stores its s(ib) (the sum of
// squares of its 4 rows, per column) to part[ib][wm][g][column], and the tile's finisher adds them in this function's
// order (unit_finish_colsq).  PART = false with `pre` (predict_refine_kernel): every thread also stores its running
// sums before the xor tree to pre[wm * 8 + g][column], the prefix a later pass carries on from row block ib1.
// NJ = 1 (PART only): the column group cg, columns cg * 32 .. cg * 32 + 31, alone.  Warp (wn, wm) then takes the n8 tile
// wn of the group (the tile j = wn of the unsplit warp wn' = cg) over the same row slab wm: the same fragments, the same
// MMAs in the same k order and the same s(ib) for every (wm, g, column) it covers, so the group's part entries are
// the unsplit ones bit for bit; four such units make up the whole part image.
template <int MMA, bool PART, int NJ = 4>
__device__ __forceinline__ void predict16_phase_b(const GpDev& G, const double* __restrict__ Ks, double* smem,
                                                  unsigned long long pol_last, unsigned long long pol_first, int ib0,
                                                  int ib1, double* __restrict__ part, double* pre = nullptr,
                                                  int cg = 0) {
    static_assert(MMA == 884 || MMA == 1684, "phase B shape");
    static_assert(NJ == 4 || (NJ == 1 && PART && MMA == 1684), "column groups: the units' m16n8k4 phase B");
    constexpr int STR = PSTR_DMMA, BK = PBK_DMMA;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // the four warps of an SM sub-partition (equal warp & 3) own the four different row slabs, so skipping the
    // structurally-zero k-tiles of the diagonal block leaves every sub-partition with the same amount of work
    const int wn = warp >> 2;
    const int wm = (warp + wn) & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int wc = NJ == 4 ? wn * 32 : cg * 32 + wn * 8;  // first column of the warp's NJ n8 tiles
    const int np = G.np;
    double* As = smem;
    double* Bs = smem + PSTAGES * BK * STR;
    double csq[NJ][2];
#pragma unroll
    for (int j = 0; j < NJ; ++j) csq[j][0] = csq[j][1] = 0.0;
    for (int ib = ib0; ib < ib1; ++ib) {
        double acc[4][NJ][2];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
        const int nks = (ib + 1) * (PBM / BK);
        const double* Abase = G.linvT + (size_t)ib * PBM;
#pragma unroll
        for (int s = 0; s < PSTAGES - 1; ++s) {
            if (s < nks)
                predict16_load_stage<NJ>(As + s * BK * STR, Bs + s * BK * STR, Abase + (size_t)(s * BK) * np,
                                         Ks + (size_t)(s * BK) * PBN, np, pol_last, pol_first, cg * 32);
            cp_async_commit();
        }
        for (int ks = 0; ks < nks; ++ks) {
            cp_async_wait<PSTAGES - 2>();
            __syncthreads();
            const int nxt = ks + PSTAGES - 1;
            const bool live = ks * BK < ib * PBM + (wm + 1) * 32;
            const double* as = As + (ks % PSTAGES) * BK * STR + wm * 32 + g;
            const double* bs = Bs + (ks % PSTAGES) * BK * STR + wc + g;
#pragma unroll
            for (int k4 = 0; k4 < BK / 4; ++k4) {
                if (k4 == 1) {
                    if (nxt < nks)
                        predict16_load_stage<NJ>(As + (nxt % PSTAGES) * BK * STR, Bs + (nxt % PSTAGES) * BK * STR,
                                                 Abase + (size_t)(nxt * BK) * np, Ks + (size_t)(nxt * BK) * PBN, np,
                                                 pol_last, pol_first, cg * 32);
                    cp_async_commit();
                }
                if (live) {
                    double a[4], b[NJ];
                    const int krow = (k4 * 4 + t4) * STR;
#pragma unroll
                    for (int i = 0; i < 4; ++i) a[i] = as[krow + i * 8];
#pragma unroll
                    for (int j = 0; j < NJ; ++j) b[j] = bs[krow + j * 8];
                    if constexpr (MMA == 1684) {
#pragma unroll
                        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                            for (int j = 0; j < NJ; ++j)
                                dmma1684(acc[2 * mi][j][0], acc[2 * mi][j][1], acc[2 * mi + 1][j][0],
                                         acc[2 * mi + 1][j][1], a[2 * mi], a[2 * mi + 1], b[j]);
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < NJ; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i], b[j]);
                    }
                }
            }
        }
        cp_async_wait<0>();
        __syncthreads();
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                s0 = fma(acc[i][j][0], acc[i][j][0], s0);
                s1 = fma(acc[i][j][1], acc[i][j][1], s1);
            }
            if constexpr (PART) {
                double* q = part + ((size_t)(ib * 4 + wm) * 8 + g) * PBN + wc + j * 8 + t4 * 2;
                *reinterpret_cast<double2*>(q) = make_double2(s0, s1);
            } else {
                csq[j][0] += s0;
                csq[j][1] += s1;
            }
        }
    }
    if constexpr (PART) return;
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            double v = csq[j][e];
            if (pre) pre[(wm * 8 + g) * PBN + wn * 32 + j * 8 + t4 * 2 + e] = v;
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            csq[j][e] = v;
        }
    double* red = smem;  // [4][PBN]: row slab wm, every column produced by exactly one warp
    if (g == 0) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            red[wm * PBN + wn * 32 + j * 8 + t4 * 2] = csq[j][0];
            red[wm * PBN + wn * 32 + j * 8 + t4 * 2 + 1] = csq[j][1];
        }
    }
    __syncthreads();
}

// ---- phase B fed by bulk copies on an mbarrier ring (PIPE_BULK, PIPE_BULK_MC) -------------------------------
// Same stages (PSTAGES x BK k-rows of L^-1 and of K*, rows padded to PSTR_DMMA), fragments, MMAs and summation order
// as predict16_phase_b<1684>, so V, and everything computed from it, is bit-equal.  Only the way the operands reach
// shared memory differs:
//   * both operands sit in global memory in the padded stage layout: L^-1 as stage images built once per fit
//     (pad_linv_stages_kernel), K* written by phase A with row stride PSTR_DMMA.  A stage is then TWO cp.async.bulk
//     of 33 KiB issued by one thread (per-row copies, 64 per stage, made the issuing warp the critical path);
//   * full[s] (one arrival + 66 KiB of transactions) replaces the CTA barrier of every k-tile.  PIPE_BULK: every
//     warp counts its consumption of a stage in done[s] (shared-memory atomic), and the last of the 16 refills the
//     slot at once with the stage three ahead, so no warp ever waits for a free slot.  The ring runs straight across
//     row blocks, so the first stages of block ib+1 load while the warps fold block ib into csq;
//   * PIPE_BULK_MC: the two CTAs of a cluster run the same L^-1 stages; each copies half of the L^-1 image of a
//     stage and multicasts it to both, so L^-1 leaves L2 once per pair.  A refill then needs both CTAs: warp 0
//     issues stage ks + 2 behind the first MMA batch of k-tile ks after waiting on empty[s], which counts the warps
//     of both CTAs (every warp arrives on its own and on the partner's barrier).
// Every warp waits on full[s] even for the k-tiles it skips (diagonal block): a count or an arrival that is not
// bounded by the fill it releases could be counted against an earlier fill.
// The ring belongs to phase B only: a CTA (MC: cluster) barrier at entry and exit keeps the copies away from the
// shared memory that phase A and the epilogue use, and `it` (stages used so far) carries the ring's phase.
// doubles before the stage image (row block ib, k-tile kt) of L^-1: row block j holds (j + 1) * PBM / PBK_DMMA k-tiles
__host__ __device__ inline size_t pad_stage_offset(int ib, int kt) {
    return ((size_t)(PBM / PBK_DMMA) * ib * (ib + 1) / 2 + kt) * PBK_DMMA * PSTR_DMMA;
}
__host__ __device__ inline size_t pad_linv_doubles(int np) { return pad_stage_offset(np / PBM, 0); }

// L^-1 (as linvT, row-major np x np) -> the stage images of the bulk-copy phase B: for row block ib (blockIdx.y) and
// k-tile kt (blockIdx.x), k-rows kt*BK .. +BK of linvT, columns ib*PBM .. +PBM, rows padded to PSTR_DMMA with zeros
__global__ void __launch_bounds__(256) pad_linv_stages_kernel(const double* __restrict__ WT, int np,
                                                              double* __restrict__ out) {
    const int kt = blockIdx.x, ib = blockIdx.y;
    if (kt >= (ib + 1) * (PBM / PBK_DMMA)) return;
    double* img = out + pad_stage_offset(ib, kt);
    for (int idx = threadIdx.x; idx < PBK_DMMA * PSTR_DMMA; idx += 256) {
        const int r = idx / PSTR_DMMA, c = idx - r * PSTR_DMMA;
        img[idx] = c < PBM ? WT[(size_t)(kt * PBK_DMMA + r) * np + (size_t)ib * PBM + c] : 0.0;
    }
}

enum { PIPE_CPASYNC = 0, PIPE_BULK = 1, PIPE_BULK_MC = 2 };

template <bool MC>
__device__ __forceinline__ void pipe_barrier() {
    if constexpr (MC)
        tc::cluster_sync();
    else
        __syncthreads();
}

// The producer re-derives its operands (policies, K* scratch, cluster rank) from the kernel parameters at every issue
// instead of holding them in registers across the k-loop: the kernel sits at 128 registers per thread.
template <bool MC>
__device__ __forceinline__ void predict16_phase_b_bulk(const PredictParams& P, const GpDev& G, double* smem,
                                                       uint64_t* full, uint64_t* empty, unsigned* done,
                                                       uint32_t& it) {
    constexpr int STR = PSTR_DMMA, BK = PBK_DMMA;
    constexpr uint32_t kStageBytes = 2 * BK * STR * sizeof(double);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wn = warp >> 2;
    const int wm = (warp + wn) & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int nb = G.np / PBM;
    double* As = smem;
    double* Bs = smem + PSTAGES * BK * STR;
    // K* (phase A's global stores) and the stage memory (phase A / epilogue) are read / overwritten by the async proxy
    tc::fence_proxy_async_global();
    tc::fence_proxy_async_smem();
    pipe_barrier<MC>();
    // one thread: stage (pib, pks) of this phase B into the free slot s
    auto copy = [&](int pib, int pks, int s) {
        {
            tc::mbar_arrive_expect_tx(&full[s], kStageBytes);
            const double* ag = G.linv_pad + pad_stage_offset(pib, pks);
            const double* bg = P.scratch + (long long)blockIdx.x * P.scratch_stride + (size_t)pks * BK * STR;
            const unsigned long long pol_last = l2_policy_evict_last(P.linv_l2_last);
            if constexpr (MC) {
                constexpr int HALF = BK / 2 * STR;
                const int r = (int)tc::cluster_ctarank();
                tc::bulk_g2s_multicast_hint(As + s * BK * STR + r * HALF, ag + r * HALF, HALF * 8, &full[s], 0x3,
                                            pol_last);
            } else {
                tc::bulk_g2s_hint(As + s * BK * STR, ag, BK * STR * 8, &full[s], pol_last);
            }
            tc::bulk_g2s_hint(Bs + s * BK * STR, bg, BK * STR * 8, &full[s], l2_policy_evict_first());
        }
    };
    // MC producer (warp 0): stage (pib, pks) into slot s once both CTAs have consumed its previous fill (parity ph ^ 1)
    auto issue = [&](int pib, int pks, int s, uint32_t ph) {
        tc::mbar_wait_budget(&empty[s], ph ^ 1, &g_pipe_timeout, kPipeWaitBudget);
        if (lane == 0) copy(pib, pks, s);
        __syncwarp();
    };
    // ring position of the next stage to consume: slot s, fill parity ph
    int s = it % PSTAGES;
    uint32_t ph = (it / PSTAGES) & 1;
    it += 2 * nb * (nb + 1);  // stages of this phase B: sum over ib of (ib + 1) * PBM / BK
    static_assert(PBM / BK == 4 && PSTAGES == 3, "ring bookkeeping");
    if constexpr (MC) {
        if (warp == 0) {  // block 0 has PBM / BK >= PSTAGES - 1 k-tiles
            issue(0, 0, s, ph);
            issue(0, 1, s == 2 ? 0 : s + 1, s == 2 ? ph ^ 1 : ph);
        }
    } else if (tid == 0) {  // every slot is free at entry; block 0 has PBM / BK >= PSTAGES k-tiles
        for (int q = 0; q < PSTAGES; ++q) copy(0, q, (s + q) % PSTAGES);
    }
    double csq[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) csq[j][0] = csq[j][1] = 0.0;
    for (int ib = 0; ib < nb; ++ib) {
        double acc[4][4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
        const int nks = (ib + 1) * (PBM / BK);
        for (int ks = 0; ks < nks; ++ks) {
            tc::mbar_wait_budget(&full[s], ph, &g_pipe_timeout, kPipeWaitBudget);
            // the fragment offsets are re-derived from a fresh %tid.x read: holding them across the loop spilled them
            const int tx = tc::tid_x(), wx = tx >> 5, wmx = (wx + (wx >> 2)) & 3, gx = (tx & 31) >> 2;
            const bool live = ks * BK < ib * PBM + (wmx + 1) * 32;
            const double* as = As + s * BK * STR + wmx * 32 + gx;
            const double* bs = Bs + s * BK * STR + (wx >> 2) * 32 + gx;
#pragma unroll
            for (int k4 = 0; k4 < BK / 4; ++k4) {
                if (MC && k4 == 1 && warp == 0) {  // stage ks + 2 goes into the slot stage ks - 1 left
                    int pib = ib, pks = ks + PSTAGES - 1;
                    if (pks >= nks) {
                        pks -= nks;
                        ++pib;
                    }
                    if (pib < nb) issue(pib, pks, s == 0 ? 2 : s - 1, s == 0 ? ph : ph ^ 1);
                }
                if (live) {
                    double a[4], b[4];
                    const int krow = (k4 * 4 + t4) * STR;
#pragma unroll
                    for (int i = 0; i < 4; ++i) a[i] = as[krow + i * 8];
#pragma unroll
                    for (int j = 0; j < 4; ++j) b[j] = bs[krow + j * 8];
#pragma unroll
                    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            dmma1684(acc[2 * mi][j][0], acc[2 * mi][j][1], acc[2 * mi + 1][j][0],
                                     acc[2 * mi + 1][j][1], a[2 * mi], a[2 * mi + 1], b[j]);
                }
            }
            __syncwarp();
            if (lane == 0) {
                if constexpr (MC) {
                    tc::mbar_arrive_cluster(&empty[s], 0);
                    tc::mbar_arrive_cluster(&empty[s], 1);
                } else {
                    __threadfence_block();  // this warp's reads of slot s happen before its count
                    if ((atomicAdd(&done[s], 1u) & 15u) == 15u) {  // last of the 16 warps: refill with stage ks + 3
                        __threadfence_block();
                        tc::fence_proxy_async_smem();
                        int pib = ib, pks = ks + PSTAGES;
                        if (pks >= nks) {
                            pks -= nks;
                            ++pib;
                        }
                        if (pib < nb) copy(pib, pks, s);
                    }
                }
            }
            if (++s == PSTAGES) {
                s = 0;
                ph ^= 1;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                s0 = fma(acc[i][j][0], acc[i][j][0], s0);
                s1 = fma(acc[i][j][1], acc[i][j][1], s1);
            }
            csq[j][0] += s0;
            csq[j][1] += s1;
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            double v = csq[j][e];
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            csq[j][e] = v;
        }
    pipe_barrier<MC>();  // every stage consumed in this CTA (MC: and in the partner) before red overwrites stage 0
    double* red = smem;  // [4][PBN]: row slab wm, every column produced by exactly one warp
    if (g == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            red[wm * PBN + wn * 32 + j * 8 + t4 * 2] = csq[j][0];
            red[wm * PBN + wn * 32 + j * 8 + t4 * 2 + 1] = csq[j][1];
        }
    }
    __syncthreads();
}

// PIPE: phase B data path; PIPE_BULK_MC is launched in clusters of 2 CTAs, and the two CTAs of a cluster run the
// same number of tiles: when the pair's second tile lies past the batch (odd tile count), the second CTA runs it
// with every column masked (c0 >= m: zero coordinates, no output, no selection entry).
// NEI: the instantiation that serves B200BO_ACQ_NEI / LOGNEI (candidate_epilogue<true>).  CNEI: the one that serves
// B200BO_ACQ_CNEI / LOGCNEI: each GP's pass hands cnei_term that GP's K* column, and the S running terms of a
// candidate wait between the passes in the CTA's scratch slot behind K* (P.carry_off, the column's stride).
template <bool DREG, int MMA, int PIPE, bool NEI = false, bool CNEI = false>
__global__ void __launch_bounds__(P16_NT, 1) predict_acq16_kernel(const PredictParams P) {
    static_assert(PIPE == PIPE_CPASYNC || MMA == 1684, "the bulk-copy phase B runs on m16n8k4");
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ double base_s[PBN];
    __shared__ double prod_s[PBN];
    __shared__ SelShared sel_s;
    __shared__ uint64_t full_bar[PSTAGES], empty_bar[PSTAGES];
    __shared__ unsigned done_cnt[PSTAGES];

    const int tid = threadIdx.x;
    double* Ks = P.scratch + (long long)blockIdx.x * P.scratch_stride;
    const long long ntiles = (P.m + PBN - 1) / PBN;
    const unsigned long long pol_last = l2_policy_evict_last(P.linv_l2_last), pol_first = l2_policy_evict_first();
    uint32_t rank = 0, it = 0;
    if constexpr (PIPE != PIPE_CPASYNC) {
        if constexpr (PIPE == PIPE_BULK_MC) rank = tc::cluster_ctarank();
        if (tid == 0) {
            for (int s = 0; s < PSTAGES; ++s) {
                tc::mbar_init(&full_bar[s], 1);
                tc::mbar_init(&empty_bar[s], (P16_NT / 32) * 2);
                done_cnt[s] = 0;
            }
            tc::mbar_fence_init();
        }
        pipe_barrier<PIPE == PIPE_BULK_MC>();  // MC: the partner's barriers exist before the first remote arrival
    }
    if (P.sel_cta) {
        if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
        __syncthreads();
    }
    // prune mode (P.perm, never with PIPE_BULK_MC): tiles claimed in bound order; `it` only crosses tile boundaries
    __shared__ long long tile_s;
    for (long long tile = P.perm ? prune_claim(P, ntiles, tile_s) : blockIdx.x; tile - rank < ntiles;
         tile = P.perm ? prune_claim(P, ntiles, tile_s) : tile + gridDim.x) {
        const long long c0 = tile * PBN;
        for (int g = 0; g < P.n_gps; ++g) {
            const GpDev& G = P.gp[g];
            if constexpr (PIPE == PIPE_CPASYNC) {
                phase_a<P16_NT, DREG, KS_F64_EF>(P, G, c0, Ks, smem, mu_s, pol_first, nullptr, P.perm, P.m, G.np);
                predict16_phase_b<MMA, false>(G, Ks, smem, pol_last, pol_first, 0, G.np / PBM, nullptr);
            } else {  // policies made where they are used: nothing extra stays live across phase B
                phase_a<P16_NT, DREG, KS_F64_EF, PSTR_DMMA>(P, G, c0, Ks, smem, mu_s, l2_policy_evict_first(), nullptr,
                                                            P.perm, P.m, G.np);
                predict16_phase_b_bulk<PIPE == PIPE_BULK_MC>(P, G, smem, full_bar, empty_bar, done_cnt, it);
            }
            const double* red = smem;
            if (tid < PBN) {
                const int c = tid;
                const double colsq = ((red[c] + red[PBN + c]) + red[2 * PBN + c]) + red[3 * PBN + c];
                const double mu_n = ((mu_s[0][c] + mu_s[1][c]) + mu_s[2][c]) + mu_s[3][c];
                const long long gi = (P.perm && c0 + c < P.m) ? (long long)P.perm[c0 + c] : c0 + c;
                double val = 0.0;
                if constexpr (CNEI)
                    candidate_epilogue<false, false, true>(P, G, g, mu_n, colsq, gi, base_s[c], prod_s[c], &val,
                                                           Ks + c, PSTR_DMMA, nullptr, Ks + P.carry_off + c);
                else
                    candidate_epilogue<NEI>(P, G, g, mu_n, colsq, gi, base_s[c], prod_s[c], &val, Ks + c,
                                            PIPE == PIPE_CPASYNC ? PBN : PSTR_DMMA);
                if (P.sel_cta && g == P.n_gps - 1) {
                    runsel_update<1>(sel_s, P.sel_k, tid, val, gi + P.index_base, c0 + c < P.m);
                    if (P.perm && tid == 0 && sel_s.list.idx[P.sel_k - 1] != SEL_NOIDX)
                        atomicMin(P.prune_ctl + kCtlKth, sel_s.list.key[P.sel_k - 1]);
                }
            }
            __syncthreads();
        }
    }
    if (P.sel_cta && tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
}

// ---- selection-only pruning: the refine stages (DESIGN.md 4.9) ------------------------------------------------------
// The tile kernel above pays one tile latency (phase B of a whole tile on one SM) for the first wave, which sets the
// k-th key, and another for whatever the single-point bound leaves.  The refine stages replace both:
//   lead    the first kLeadTiles tiles in bound order, evaluated exactly by predict_units_kernel, which splits the row
//           blocks of every tile across CTAs, so the k-th key exists after a fraction of a tile latency;
//           merge_kth_kernel then sets the k-th key from the union of the per-CTA lists;
//   refine  predict_refine_kernel: for the following tiles in bound order (same stop rule as prune_claim) the product
//           with the leading b row blocks of L^-1 only.  r_b = sum of V_i^2 over those rows is k*^T K^-1 k* of the GP
//           conditioned on the first b * PBM training points alone, and the remaining terms are squares, so
//           r_b <= k*^T K^-1 k* and prune_var_ub(r_b) bounds the variance as the single-point r does.  Candidates whose
//           refined key and single-point key are both <= the k-th key are appended to the survivor list, with the
//           running sums of their first b row blocks (the prefix);
//   level   predict_units_kernel over row blocks [b, 2b) of the survivors only: the last unit of a tile carries each
//           survivor's prefix on to 2b, keys it as the refine stage does and appends the survivors whose keys are all
//           <= the k-th key, with the new prefix, to the level's list;
//   final   the level's survivors sorted by key through the same units (final_rounds_kernel), from the carried prefix
//           on, in rounds that each skip the tiles above the k-th key merged before them.
// When more than kRefineMaxTiles tiles of survivors come up (little prunes: the refine stage stops claiming tiles as
// soon as it sees that), the final stage does nothing and the tile kernel goes on in bound order behind the lead
// tiles as it would have without these stages; otherwise the final stage closes the tile kernel's counter.
// Exact values are bit-equal to the tile kernel's: K* entries carry no order, mu comes from the one unit of a tile that
// recomputes it from the K* slot over all np rows (the same function and order of sums as phase A), and the sum of
// squares is added up by unit_finish_colsq in the order of predict16_phase_b.  The stages are kernel boundaries, the
// steps of a final round grid barriers, and within the units the last unit to arrive at a tile's counter finishes it.
constexpr int kLeadTiles = 8, kRefineMaxTiles = 128, kUnitSlots = kLeadTiles + kRefineMaxTiles;

// Tiles of final round r from tile t0 on: 8, then the rest of the kRefineMaxTiles (at C3 the level leaves 1.6 tiles),
// at most `grid` each (a round's K* slots)
__host__ __device__ inline int final_round_tiles(int r, int t0, int grid) {
    const int t = r == 0 ? 8 : kRefineMaxTiles - t0;
    return t < grid ? t : grid;
}

constexpr long long kCtlClosed = 1ll << 40;  // value of kCtlTile no batch reaches

enum { kStageLead = 0, kStageFinal = 1, kStageLevel = 2 };

struct RefineParams {
    const double2* mu;       // [m] interval (mu_lo, mu_hi) of K* alpha_ per candidate (local index), from the bound pass
    double* mu_unit;         // [kUnitSlots][PBN] K* alpha_ of a tile's candidates, from its last group's phase A
    int* surv;               // [kRefineMaxTiles * PBN] local indices the refine stage let through (final: sorted)
    unsigned long long* surv_key;  // [kRefineMaxTiles * PBN] their keys (max of single-point and refined key)
    // [kRefineMaxTiles * PBN][32] per survivor, the running sums over row blocks [0, b0) per (row slab wm, lane group
    // g), index wm * 8 + g, before the xor tree; nullptr in the lead stage (b0 = 0)
    double* prefix;
    int* surv_out;           // a level: the survivors it lets through, their keys, prefixes and slots (the values of
    unsigned long long* surv_key_out;  // the final sort)
    double* prefix_out;
    int* pos_out;
    double* part;            // [kUnitSlots][np / PBM][4][8][PBN] per-row-block partial sums of squares
    unsigned* arrive;        // [kUnitSlots] units that have delivered their part of a tile
    int blocks;              // leading row blocks of the refined bound
    int groups_max;          // most row-block groups a tile is split into
    int final_stage;         // predict_units_kernel: kStageLead, kStageFinal or kStageLevel
    int b0, b1;              // the units' row blocks [b0, b1): the lead and the final stage end at np / PBM
    int n_word;              // final stage and level: the prune_ctl word counting their candidates
    int out_word;            // the level: the prune_ctl word counting the candidates it lets through
    int t0, t1;              // final stage and level: the round's tiles [t0, t1) of the survivor list
};

// column groups of 32 columns per row-block group of a level or final round whose row-block groups alone cannot fill
// the grid
constexpr int kUnitColGroups = 4;

// The tiles of a lead stage, level launch or final round, the same in every CTA: candidates list[0, n), tiles
// [tbeg, tend) of PBN columns, partial-sum slots from slot0.  Level and final stage: too many refine survivors leave
// n = 0 (the tile kernel takes over in bound order); otherwise the final stage closes the tile kernel's counter.
struct UnitRound {
    const int* list;
    long long n, tbeg, tend;
    int slot0;
};
__device__ __forceinline__ UnitRound unit_round(const PredictParams& P, const RefineParams& R) {
    UnitRound U;
    U.list = P.perm;
    U.n = min(P.m, (long long)kLeadTiles * PBN);
    U.slot0 = 0;
    U.tbeg = 0;
    if (R.final_stage != kStageLead) {
        U.n = 0;
        if (P.prune_ctl[kCtlSurv] <= (unsigned long long)kRefineMaxTiles * PBN) {
            U.n = (long long)P.prune_ctl[R.n_word];
            if (R.final_stage == kStageFinal && blockIdx.x == 0 && threadIdx.x == 0)
                atomicExch(P.prune_ctl + kCtlTile, (unsigned long long)kCtlClosed);
        }
        U.list = R.surv;
        U.slot0 = kLeadTiles;
        U.tbeg = R.t0;
    }
    U.tend = (U.n + PBN - 1) / PBN;
    if (R.final_stage && U.tend > R.t1) U.tend = R.t1;
    return U;
}

// whether every unit of tile `tile` skips it: its best bound key is above the k-th key copied before the stage / round
__device__ __forceinline__ bool unit_skip(const PredictParams& P, const RefineParams& R, long long tile) {
    if (R.final_stage == kStageLead) return P.perm_key[tile * PBN] > P.prune_ctl[kCtlKthLead];
    if (R.final_stage == kStageLevel) return false;  // no exact value moves the k-th key during the level
    return R.surv_key[tile * PBN] > P.prune_ctl[kCtlKthRound];
}

// The k-th smallest key over the union of the per-CTA lists (sel_cta, lists carried in by a continued batch included)
// into kCtlKth, when there are k entries, and a copy of that word into kCtlKthRound for the next final round.  It is
// the k-th smallest of values already produced, so the final k-th key is <= it.  One warp: k rounds of a merge of the
// list heads.
// One warp (lane = threadIdx.x & 31); head: nlists ints of shared memory.
__device__ __forceinline__ void merge_kth_run(const SelList* __restrict__ lists, int nlists, int k,
                                              unsigned long long* ctl, int* head) {
    const int lane = threadIdx.x & 31;
    for (int l = lane; l < nlists; l += 32) head[l] = 0;
    __syncwarp();
    unsigned long long kth = 0xFFFFFFFFFFFFFFFFull;
    bool full = true;
    for (int r = 0; r < k; ++r) {
        unsigned long long bk = 0xFFFFFFFFFFFFFFFFull;
        int bl = 0x7FFFFFFF;
        for (int l = lane; l < nlists; l += 32) {
            const int h = head[l];
            if (h < k && lists[l].idx[h] != SEL_NOIDX && (lists[l].key[h] < bk || bl == 0x7FFFFFFF)) {
                bk = lists[l].key[h];
                bl = l;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, o);
            const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
            if (ol != 0x7FFFFFFF && (bl == 0x7FFFFFFF || ok < bk || (ok == bk && ol < bl))) {
                bk = ok;
                bl = ol;
            }
        }
        if (bl == 0x7FFFFFFF) {  // fewer than k entries
            full = false;
            break;
        }
        kth = bk;
        if (lane == 0) head[bl] += 1;
        __syncwarp();
    }
    if (lane == 0) {
        if (full && kth < ctl[kCtlKth]) ctl[kCtlKth] = kth;
        ctl[kCtlKthRound] = ctl[kCtlKth];
    }
}

__global__ void __launch_bounds__(32) merge_kth_kernel(const SelList* __restrict__ lists, int nlists, int k,
                                                        unsigned long long* ctl) {
    __shared__ int head[1024];
    merge_kth_run(lists, nlists, k, ctl, head);
}

// first row block of group j of G over the row blocks [b0, nb), cut so that the groups' k-tile counts (row block ib:
// ib + 1) are about equal; j = G gives nb.  Groups may be empty.
__host__ __device__ inline int unit_cut(int b0, int nb, int G, int j) {
    const long long base = (long long)b0 * (b0 + 1) / 2, total = (long long)nb * (nb + 1) / 2 - base;
    int ib = b0;
    while (ib < nb && ((long long)ib * (ib + 1) / 2 - base) * G < total * j) ++ib;
    return j >= G ? nb : ib;
}

// sum over the row blocks [ib0, nb) of a tile's partials, in the order of predict16_phase_b: per (row slab wm, lane
// group g) over ib, starting from the carried prefix of row blocks [0, ib0) (pre_in[column][wm * 8 + g]; nullptr:
// ib0 = 0, from 0), then the xor-shuffle tree over g (4, 8, 16: ((0+1)+(2+3))+((4+5)+(6+7))), written to red[wm][c];
// the caller adds the slabs.  pre_out (nullable): the sums before the tree, [wm * 8 + g][c].  Columns from ncols on
// read no prefix.  512 threads: thread = (wm, column).
__device__ __forceinline__ void unit_finish_colsq(const double* __restrict__ part, const double* __restrict__ pre_in,
                                                  long long ncols, int ib0, int nb, double* red, double* pre_out) {
    const int c = threadIdx.x & (PBN - 1), wm = threadIdx.x >> 7;
    double v[8];
#pragma unroll
    for (int g = 0; g < 8; ++g) v[g] = pre_in && c < ncols ? __ldcg(pre_in + (size_t)c * 32 + wm * 8 + g) : 0.0;
    for (int ib = ib0; ib < nb; ++ib) {
#pragma unroll
        for (int g = 0; g < 8; ++g) v[g] += __ldcg(part + ((size_t)(ib * 4 + wm) * 8 + g) * PBN + c);
    }
    if (pre_out) {
#pragma unroll
        for (int g = 0; g < 8; ++g) pre_out[(wm * 8 + g) * PBN + c] = v[g];
    }
    red[wm * PBN + c] = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
}

template <bool DREG>
__global__ void __launch_bounds__(P16_NT, 1) predict_refine_kernel(const PredictParams P, const RefineParams R) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ long long tile_s;
    const int tid = threadIdx.x;
    const GpDev& G = P.gp[0];
    double* Ks = P.scratch + (long long)blockIdx.x * P.scratch_stride;
    const long long ntiles = (P.m + PBN - 1) / PBN;
    const unsigned long long pol_last = l2_policy_evict_last(P.linv_l2_last), pol_first = l2_policy_evict_first();
    // nothing moves the k-th key while this kernel runs
    const unsigned long long kth = P.prune_ctl[kCtlKth];
    for (;;) {
        if (tid == 0) {
            long long t = ntiles;
            if (*reinterpret_cast<volatile unsigned long long*>(P.prune_ctl + kCtlSurv) <=
                (unsigned long long)kRefineMaxTiles * PBN) {
                t = (long long)atomicAdd(P.prune_ctl + kCtlRefTile, 1ull);
                if (t < ntiles && P.perm_key[t * PBN] > kth) t = ntiles;
            }
            if (t < ntiles) atomicAdd(P.prune_ctl + kCtlRefined, (unsigned long long)min((long long)PBN, P.m - t * PBN));
            tile_s = t;
        }
        __syncthreads();
        const long long tile = tile_s;
        if (tile >= ntiles) break;
        const long long c0 = tile * PBN;
        phase_a<P16_NT, DREG, KS_F64_EF>(P, G, c0, Ks, smem, mu_s, pol_first, nullptr, P.perm, P.m, R.blocks * PBM);
        double* pre = smem + 4 * PBN;  // [32][PBN] behind red
        predict16_phase_b<1684, false>(G, Ks, smem, pol_last, pol_first, 0, R.blocks, nullptr, pre);
        const double* red = smem;
        if (tid < PBN && c0 + tid < P.m) {
            const int c = tid, li = P.perm[c0 + c];
            const double r = ((red[c] + red[PBN + c]) + red[2 * PBN + c]) + red[3 * PBN + c];
            const double2 mu = R.mu[li];
            const unsigned long long key = prune_bound_key(P, G, mu.x, mu.y, prune_var_ub(G, r));
            const unsigned long long key1 = P.perm_key[c0 + c];
            if (key <= kth && key1 <= kth) {
                const unsigned long long pos = atomicAdd(P.prune_ctl + kCtlSurv, 1ull);
                if (pos < (unsigned long long)kRefineMaxTiles * PBN) {
                    R.surv[pos] = li;
                    R.surv_key[pos] = key > key1 ? key : key1;  // both are lower bounds
#pragma unroll 4
                    for (int q = 0; q < 32; ++q) R.prefix[pos * 32 + q] = pre[q * PBN + c];
                }
            }
        }
        __syncthreads();
    }
}

// K* rows [0, PBM * b1) of the tiles of a lead stage, level or final round (unit_round, unit_skip), each into its own
// scratch slot (tile - tbeg; a round has at most gridDim.x tiles), with phase_a's arithmetic: items (tile, chunks [ch0, ch1)), the
// chunks of a tile cut so that there are about gridDim.x items.  Plain stores: every unit of the tile reads the slot.
template <bool DREG>
__device__ __forceinline__ void ks_build_run(const PredictParams& P, const RefineParams& R, double* smem,
                                             double (*mu_s)[PBN]) {
    const GpDev& G = P.gp[0];
    const UnitRound U = unit_round(P, R);
    const long long nt = U.tend - U.tbeg;
    if (nt <= 0) return;
    const int nch = R.b1 * PBM / PA_CHUNK;
    const int per = (int)max(1ll, (nch * nt + gridDim.x - 1) / gridDim.x), items = (nch + per - 1) / per;
    for (long long it = blockIdx.x; it < nt * items; it += gridDim.x) {
        const long long tile = U.tbeg + it / items;
        const int ch0 = (int)(it % items) * per, ch1 = min(nch, ch0 + per);
        if (unit_skip(P, R, tile)) continue;
        double* Ks = P.scratch + (tile - U.tbeg) * P.scratch_stride;
        phase_a<P16_NT, DREG, KS_F64>(P, G, tile * PBN, Ks, smem, mu_s, 0ull, nullptr, U.list, U.n, ch1 * PA_CHUNK,
                                      ch0 * PA_CHUNK);
    }
}

template <bool DREG>
__global__ void __launch_bounds__(P16_NT, 1) ks_build_kernel(const PredictParams P, const RefineParams R) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    ks_build_run<DREG>(P, R, smem, mu_s);
}

// K* alpha_ of a tile from its K* slot, in phase_a's order: thread (part, column) runs one fma chain over the chunks in
// ascending order, rows part * 16 .. part * 16 + 15 of each, so mu_s[part][c] is phase A's bit for bit.
__device__ __forceinline__ void unit_mu_from_ks(const GpDev& G, const double* __restrict__ Ks,
                                                double (*mu_s)[PBN]) {
    constexpr int ROWS = PA_CHUNK / P16_SPLIT;
    const int c = threadIdx.x & (PBN - 1), part = threadIdx.x >> 7;
    double mu = 0.0;
    for (int n0 = part * ROWS; n0 < G.np; n0 += PA_CHUNK) {
#pragma unroll
        for (int q = 0; q < ROWS; ++q) mu = fma(__ldg(G.alphav + n0 + q), __ldcg(Ks + (size_t)(n0 + q) * PBN + c), mu);
    }
    mu_s[part][c] = mu;
}

// k-tile groups of row-block group j of G over [b0, nb) (unit_cut): sum of ib + 1 over its row blocks
__host__ __device__ inline long long unit_cost(int b0, int nb, int G, int j) {
    const long long a = unit_cut(b0, nb, G, j), b = unit_cut(b0, nb, G, j + 1);
    return (b * (b + 1) - a * (a + 1)) / 2;
}

// Exact evaluation in units of (tile, group of consecutive row blocks of [b0, b1), column group).  Lead stage: the
// tiles are the first kLeadTiles of P.perm, each skipped when its best bound key is above the k-th key carried into this
// launch (a continued batch; read from kCtlKthLead, which does not move, so that all units of a tile decide alike).
// Final stage: the tiles [t0, t1) of the survivor list, each skipped when its first key is above kCtlKthRound.  The
// level: the tiles [t0, t1) of its survivor list, none skipped.  The level and the final rounds cut [b0, b1) into up to
// one row block per group (at most 32 groups, about 2 * gridDim.x units) and split every row-block group into
// kUnitColGroups column groups of 32 columns when their tiles' row-block groups alone cannot fill the grid.  At C3 the
// final round has 2 tiles over row blocks [8, 32): 24 groups of 4 column groups, the heaviest unit a quarter of the
// last row block (8 of its 32 k-tiles) where 16 whole-column groups made a group of two row blocks, 59 k-tiles, the
// round's latency.  The part image and the arrival count are the same either way.  Units are claimed row-block
// group descending (the single large row blocks first), tiles innermost.  A unit reads the tile's K* from the
// slot that ks_build_kernel filled, runs phase B over its row blocks and columns, and the last unit to arrive finishes
// the tile: from the survivors' carried prefix on, as the tile kernel's epilogue does (lead, final), or as the refine
// stage keys its candidates at b1 row blocks (the level).  In the lead and the final stage the first column group of the
// row-block group with the fewest k-tiles (an empty one if any) also computes the tile's mu from the slot.
// The units of one launch or round, between the CTA's runsel_begin and runsel_store (sel_s: its running list).
__device__ __forceinline__ void units_run(const PredictParams& P, const RefineParams& R, double* smem,
                                          double (*mu_s)[PBN], SelShared& sel_s) {
    __shared__ long long unit_s;
    __shared__ int last_s, mu_grp_s;
    const int tid = threadIdx.x;
    const GpDev& G = P.gp[0];
    const int nb = G.np / PBM;
    const unsigned long long pol_last = l2_policy_evict_last(P.linv_l2_last);
    const UnitRound U = unit_round(P, R);
    const int* list = U.list;
    const long long n = U.n, nt = U.tend - U.tbeg;
    unsigned long long* claim = P.prune_ctl + kCtlUnit;
    const int b0 = R.b0, b1 = R.b1;
    int groups = R.groups_max, cgs = 1;
    if (R.final_stage != kStageLead && nt > 0) {
        const int gmax = min(32, b1 - b0);  // up to one row block per group
        if (nt * gmax < 2ll * gridDim.x) cgs = kUnitColGroups;
        groups = (int)max(1ll, min((long long)gmax, 2ll * gridDim.x / (nt * cgs)));
    }
    if (tid < 32) {  // the row-block group with the fewest k-tiles, the lowest such on ties
        long long c = tid < groups ? unit_cost(b0, b1, groups, tid) : 0x7FFFFFFFFFFFFFFFll;
        int j = tid;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const long long oc = __shfl_xor_sync(0xffffffffu, c, o);
            const int oj = __shfl_xor_sync(0xffffffffu, j, o);
            if (oc < c || (oc == c && oj < j)) {
                c = oc;
                j = oj;
            }
        }
        if (tid == 0) mu_grp_s = j;
    }
    __syncthreads();
    const int mu_grp = R.final_stage == kStageLevel ? -1 : mu_grp_s;  // the level keys from the stored mu interval
    const long long units = nt * groups * cgs;
    for (;;) {
        if (tid == 0) unit_s = (long long)atomicAdd(claim, 1ull);
        __syncthreads();
        const long long unit = unit_s;
        if (unit >= units) break;
        const long long tile = U.tbeg + unit % nt, r = unit / nt;
        const long long c0 = tile * PBN;
        if (unit_skip(P, R, tile)) {
            __syncthreads();
            continue;
        }
        const int grp = groups - 1 - (int)(r / cgs), cg = (int)(r % cgs);
        const int ib0 = unit_cut(b0, b1, groups, grp), ib1 = unit_cut(b0, b1, groups, grp + 1);
        const int slot = U.slot0 + (int)tile;
        double* part = R.part + (size_t)slot * nb * 32 * PBN;
        const double* Ks = P.scratch + (tile - U.tbeg) * P.scratch_stride;
        const bool mu_unit = grp == mu_grp && cg == 0;
        if (mu_unit) unit_mu_from_ks(G, Ks, mu_s);
        if (ib1 > ib0) {
            if (cgs == 1)
                predict16_phase_b<1684, true>(G, Ks, smem, pol_last, l2_policy_evict_last(0.f), ib0, ib1, part);
            else
                predict16_phase_b<1684, true, 1>(G, Ks, smem, pol_last, l2_policy_evict_last(0.f), ib0, ib1, part,
                                                 nullptr, cg);
        }
        if (mu_unit) {  // mu_s holds the tile kernel's K* alpha_ parts (phase A over all np rows)
            __syncthreads();
            if (tid < PBN)
                R.mu_unit[(size_t)slot * PBN + tid] = ((mu_s[0][tid] + mu_s[1][tid]) + mu_s[2][tid]) + mu_s[3][tid];
        }
        __threadfence();  // this unit's partials and mu before its arrival
        __syncthreads();
        if (tid == 0) last_s = atomicAdd(R.arrive + slot, 1u) == (unsigned)(groups * cgs) - 1;
        __syncthreads();
        if (last_s) {
            __threadfence();
            if (tid == 0) R.arrive[slot] = 0u;  // every unit of the tile has arrived: the slot's next level starts at 0
            double* red = smem;
            double* pre = R.final_stage == kStageLevel ? smem + 4 * PBN : nullptr;  // [32][PBN] behind red
            unit_finish_colsq(part, R.prefix ? R.prefix + c0 * 32 : nullptr, n - c0, b0, b1, red, pre);
            __syncthreads();
            if (R.final_stage == kStageLevel) {
                if (tid < PBN && c0 + tid < n) {
                    const int c = tid, li = list[c0 + c];
                    const double r = ((red[c] + red[PBN + c]) + red[2 * PBN + c]) + red[3 * PBN + c];
                    const double2 mu = R.mu[li];
                    const unsigned long long key = prune_bound_key(P, G, mu.x, mu.y, prune_var_ub(G, r));
                    const unsigned long long key1 = R.surv_key[c0 + c], kth = P.prune_ctl[kCtlKth];
                    if (key <= kth && key1 <= kth) {
                        const unsigned long long pos = atomicAdd(P.prune_ctl + R.out_word, 1ull);
                        R.surv_out[pos] = li;
                        R.surv_key_out[pos] = key > key1 ? key : key1;  // every key is a lower bound
                        R.pos_out[pos] = (int)pos;
#pragma unroll 4
                        for (int q = 0; q < 32; ++q) R.prefix_out[pos * 32 + q] = pre[q * PBN + c];
                    }
                }
            } else if (tid < PBN) {
                const int c = tid;
                const bool valid = c0 + c < n;
                const long long gi = valid ? (long long)list[c0 + c] : P.m;
                const double colsq = ((red[c] + red[PBN + c]) + red[2 * PBN + c]) + red[3 * PBN + c];
                double val = 0.0, base, prod;
                const double mu_n = valid ? __ldcg(R.mu_unit + (size_t)slot * PBN + c) : 0.0;
                candidate_epilogue(P, G, 0, mu_n, colsq, gi, base, prod, &val);
                runsel_update<1>(sel_s, P.sel_k, tid, val, gi + P.index_base, valid);
                if (tid == 0) {
                    if (sel_s.list.idx[P.sel_k - 1] != SEL_NOIDX)
                        atomicMin(P.prune_ctl + kCtlKth, sel_s.list.key[P.sel_k - 1]);
                    atomicAdd(P.prune_ctl + kCtlEval, (unsigned long long)min((long long)PBN, n - c0));
                }
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(P16_NT, 1) predict_units_kernel(const PredictParams P, const RefineParams R) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ SelShared sel_s;
    const int tid = threadIdx.x;
    if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
    units_run(P, R, smem, mu_s, sel_s);
    if (tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
}

// The rounds of the final stage in one cooperative launch (one CTA per SM, every CTA resident): per round the K*
// build, a grid barrier, the units, a grid barrier, the merge of the k-th key by CTA 0 (which also resets the units'
// claim counter), and a grid barrier.  The same work and arithmetic as ks_build_kernel, predict_units_kernel and
// merge_kth_kernel launched round by round, without their launches: a round with no tiles left (at C3 the second)
// costs its barriers only, and once the rounds are past the survivors every CTA leaves together (the survivor count
// does not move during the stage, so all CTAs decide alike).  The rounds' tiles come from final_round_tiles, so any
// grid size runs in this one launch.
template <bool DREG>
__global__ void __launch_bounds__(P16_NT, 1) final_rounds_kernel(const PredictParams P, RefineParams R) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[P16_SPLIT][PBN];
    __shared__ SelShared sel_s;
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const int tid = threadIdx.x;
    if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
    __syncthreads();
    for (int r = 0, t0 = 0; t0 < kRefineMaxTiles; ++r, t0 = R.t1) {
        R.t0 = t0;
        R.t1 = t0 + final_round_tiles(r, t0, gridDim.x);
        const UnitRound U = unit_round(P, R);
        if (U.tbeg >= (U.n + PBN - 1) / PBN) break;  // this and every later round has no tile
        ks_build_run<DREG>(P, R, smem, mu_s);
        __threadfence();
        grid.sync();
        units_run(P, R, smem, mu_s, sel_s);
        if (tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
        __threadfence();
        grid.sync();
        if (blockIdx.x == 0 && tid < 32) {
            merge_kth_run(P.sel_cta, gridDim.x, P.sel_k, P.prune_ctl, reinterpret_cast<int*>(smem));
            if (tid == 0) P.prune_ctl[kCtlUnit] = 0ull;
            __threadfence();
        }
        grid.sync();
    }
}

}  // namespace b200bo
