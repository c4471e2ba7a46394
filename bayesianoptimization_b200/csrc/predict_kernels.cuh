// predict_kernels.cuh - the fused posterior-predict + acquisition kernel (fp64) and the
// (value,index) selection kernel.
//
// Replaces, for a batch of M candidates, the whole chain
//   K* = kernel_(X*, X)            SK/gaussian_process/_gpr.py:446, kernels.py:1720-1729
//   mu = s_y * K* alpha_ + y_mean  :447-450
//   V  = L^-1 K*^T                 :460-462   (the N^2 M term)
//   var = diag - sum_i V_i^2, clamp, sd = sqrt(var * s_y^2)   :480-500
//   -base_acq(mu, sd) [* prod_j p_j]   R/bayes_opt/acquisition.py:199-217, :485/:660/:847,
//                                      R/bayes_opt/constraint.py:200-221
// in ONE launch.  V is formed as the triangular GEMM  V = Linv * K*^T  against the cached
// explicit inverse of the Cholesky factor (computed once at fit time), so the per-candidate
// work has no dependency chain.
//
// Decomposition: a persistent grid (one CTA per SM); each CTA owns tiles of BN = 128
// candidates.  Per tile and per GP:
//   phase A  build K*^T (np x 128) once into a CTA-private HBM/L2 scratch + accumulate K* alpha_ (phase_a, which
//            every fused predict kernel here and in predict16.cuh runs)
//   phase B  for each 128-row block of Linv: acc(128x128) = sum_{k<=rows} LinvT[k][rows]^T K*[k][:],
//            8x8 register tiles, 3-stage cp.async pipeline; then colsq += sum_rows acc^2
//   phase C  mu, sd, acquisition / constraint probability per candidate
// All reductions are fixed-order (no floating-point atomics): results are bit-reproducible and
// independent of the grid size.
#pragma once
#include "common.cuh"
#include "select.cuh"
#include "tc_common.cuh"

namespace b200bo {

struct GpDev {
    const double* Xs;      // [np][d]   transform(X)/length_scale, zero padded
    const double* linvT;   // [np][np]  (L^-1)^T row-major: linvT[k][i] = Linv[i][k]
    const double* alphav;  // [np]      alpha_, zero padded
    const double* ls;      // [d]       length scales (replicated when isotropic)
    const int* xform;      // [d] or nullptr
    const uint8_t* linv_tc;  // fp32 mode: L^-1 as tf32 (hi,lo) wgmma operand images, or nullptr
    const double* linv_pad;  // bulk-copy phase B of predict_acq16_kernel: L^-1 as padded stage images, or nullptr
    // Gram bound pass of pruning: [np][gram_stride(d)] training operand, then A1 and Ymax (predict16.cuh), or nullptr
    const double* gram;
    int n, np, family, nu;
    double constv, y_mean, y_std, lb, ub;
    double prior;  // prior variance kernel_.diag(x*) = constv + WhiteKernel noise_level
    double kdiag;  // diagonal of the factorised training covariance: constv + noise_level + alpha
};

struct PredictParams {
    GpDev gp[B200BO_MAX_GPS];
    int n_gps, d, acq_kind, pad0;
    double kappa, xi, y_max;
    double ystar[B200BO_MAX_PATHS];  // MES: the samples y*_k of the maximum (data units), k < n_ystar
    int n_ystar, pad1;
    const double* Xc;  // [m][d], or nullptr: candidates generated in-kernel (Philox, select.cuh)
    const double* pbounds;  // Philox mode: [2][d] = lo_j, (hi_j - lo_j)
    unsigned long long seed;  // Philox key
    long long index_base;  // global index of this launch's candidate 0 (Philox row / selection index)
    SelList* sel_cta;  // [gridDim.x] per-CTA running selection, or nullptr (no fused selection)
    int sel_k, sel_resume;  // resume: continue the lists of the previous launch (chunked batches)
    long long m;
    double* acq_out;   // [m] or nullptr
    double* mu_out;    // [m] or nullptr (target GP)
    double* sd_out;    // [m] or nullptr (target GP)
    double* scratch;   // gridDim.x * scratch_stride doubles
    long long scratch_stride;
    unsigned long long* clamp_count;  // nullable; [0] negative variances clamped to 0, [1] non-finite candidate coordinates
    float linv_l2_last;  // predict_acq16_kernel: evict_last fraction of the L^-1 loads; <= 0: evict_normal
    // selection-only pruning (predict16.cuh, DESIGN.md 4.9), or nullptr: tile t of predict_acq16_kernel is the
    // candidates perm[t * PBN ..] (local indices sorted by the key of a lower bound on their value, perm_key)
    const int* perm;
    const unsigned long long* perm_key;
    unsigned long long* prune_ctl;  // [0] next tile to claim, [1] least k-th key of a full CTA list, [2] evaluated
    // NEI / LogNEI (DESIGN.md 4.13): A = K0^-1 F of gps[0], [np][n_ystar] row-major, then best_0 .. best_{n_ystar-1}
    const double* fant_a;
    // CNEI / LogCNEI (DESIGN.md 4.15): A_g = K0_g^-1 F_g of every GP g ([np][n_ystar]); fant_a is gps[0]'s, best_s
    // behind it.  Here rather than in GpDev, so that the struct every other kernel reads keeps its layout.
    const double* fant_a_gp[B200BO_MAX_GPS];
    // predict_acq16_kernel: offset (doubles) of each CTA's per-sample carry [n_ystar][PSTR_DMMA] in its scratch slot
    long long carry_off;
    // B200BO_ACQ_MEAN (DESIGN.md 4.17): T = 2 B + 1 of the merit, B >= |mu_0| (0 without constraint GPs: unused)
    double mean_T;
};

// coordinate j of candidate gi (local index) as the reference's x_tries[gi, j]
// A non-finite coordinate is counted in clamp_count[1]: the host entry points turn it into the ValueError
// ("Input X contains NaN or infinity") sklearn's validate_data raises - checked where the data is read anyway instead
// of a separate pass over the batch on the host (10 ms per 2^20 x 16 batch).
// Params: PredictParams or any launch-parameter struct with the same candidate-source fields (paths.cuh).
template <class Params>
__device__ __forceinline__ double candidate_coord(const Params& P, long long gi, int j) {
    if (P.Xc) {
        const double v = P.Xc[gi * P.d + j];
        if (!isfinite(v) && P.clamp_count) atomicAdd(P.clamp_count + 1, 1ull);
        return v;
    }
    return philox_coord(P.seed, gi + P.index_base, j, P.pbounds[j], P.pbounds[P.d + j]);
}

constexpr int PBM = 128, PBN = 128, PBK = 16, PSTAGES = 3, PNT = 256;
// smem row stride (doubles) of the A/B k-tiles.  DFMA variant: dense rows (conflict-free 16-byte
// fragment loads).  DMMA variant: +4 doubles: an LDS.64 is served per half-warp (4 k-rows x 4
// columns of an m8n8k4 fragment); a row stride of 264 words = 8 (mod 32) puts the four k-rows of
// each half-warp on disjoint bank octets -> 2 wavefronts per request, the minimum for 256 bytes.
constexpr int PSTR_DFMA = 128, PSTR_DMMA = 132;
// phase A needs (128 + 2*64) * d doubles (d <= 64 -> 128 KiB); phase B (DFMA) 96 KiB
constexpr int kPredictSmemBytesDfma = 133120;  // + 1 KiB staged alpha_
constexpr int PBK_DMMA = 32;  // k-tile of the DMMA variant (one CTA barrier per 32 k)
constexpr int kPredictSmemBytesDmma = PSTAGES * PBK_DMMA * 2 * PSTR_DMMA * 8;  // 202752
constexpr int kPredictMaxDimRegs = 16;  // candidates held in registers when d <= 16

enum { PREDICT_IMPL_DFMA = 0, PREDICT_IMPL_DMMA = 1, PREDICT_IMPL_TF32 = 2 };

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// sm_90 shape (SASS DMMA.16x8x4): twice the fp64 tensor rate of m8n8k4 per SM and clock on H100, the same rate as
// m16n8k8 / m16n8k16 (tools/dmma_shapes.cu, DESIGN.md 6) with the fragment registers of m8n8k4.
// Fragments (PTX ISA, .f64), g = lane/4, t4 = lane%4:
//   A 16x4: a0 (g, t4), a1 (g+8, t4)    B 4x8: b0 (t4, g)
//   C 16x8: c0 (g, 2t4), c1 (g, 2t4+1), c2 (g+8, 2t4), c3 (g+8, 2t4+1)
__device__ __forceinline__ void dmma1684(double& c0, double& c1, double& c2, double& c3, double a0, double a1,
                                         double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
                 : "d"(a0), "d"(a1), "d"(b));
}

// The out-of-line terms below and candidate_epilogue take a GRAD flag.  GRAD = false is the value alone: the
// out-pointers are unused and dropped, so the value keeps its scalar-and-pointer signature and the predict kernels
// compile as without them.  GRAD = true (small_finish_grad_kernel) also writes, from the same evaluation, the term's
// coefficients of d mean and d sd (data units): d term = cm d mean + cs d sd.  Callers pass the out-pointers through
// grad_out, so that no local's address reaches a value-form call: an escaping address alone changes the code the
// value kernels compile to.
template <bool GRAD>
__device__ __forceinline__ double* grad_out(double& x) {
    return GRAD ? &x : nullptr;
}

// One sample's term of max-value entropy search (Wang & Jegelka, ICML 2017, eq. 6) at g = (y*_k - mu) / sigma:
//   t(g) = g psi(g) / (2 Psi(g)) - log Psi(g)
// Out of line (DESIGN.md 4.8): inlined into the 16-warp kernel, which runs at its 128-register cap, the term's
// libdevice code made ptxas place spill code in the clustered kernel's phase-B k-loop; as a call, the spill code the
// MES branch adds in every predict kernel lies outside the phase-B k-loops.  For finite g the product is finite (psi
// underflows to 0 above g ~ 38.6); the guard keeps g = +inf (sigma underflowing against y* - mu) at its limit 0.
// GRAD: dt = t'(g).  With lambda = psi / Psi (inv_mills), lambda' = -lambda (g + lambda), so
// t' = -lambda/2 - g lambda (g + lambda)/2; lambda = 0 is the limit 0.
template <bool GRAD = false>
__device__ __noinline__ double mes_term(double g, double* dt = nullptr) {
    const double r = inv_mills(g);
    const double a = (r == 0.0) ? 0.0 : 0.5 * g * r;
    if constexpr (GRAD) *dt = (r == 0.0) ? 0.0 : -0.5 * r - 0.5 * g * r * (g + r);
    return a - log_ndtr(g);
}

// EI at a = mean - y_max - xi; GRAD: cm = Phi(z), cs = phi(z).  The compiler contracts the sum into one FMA, and
// which product it fuses depends on the surrounding code (see the gradient form of candidate_epilogue).
template <bool GRAD = false>
__device__ __forceinline__ double ei_term(double a, double sd, double* cm = nullptr, double* cs = nullptr) {
    const double z = a / sd;
    if constexpr (GRAD) {
        *cm = ndtr(z);
        *cs = norm_pdf(z);
    }
    return a * ndtr(z) + sd * norm_pdf(z);
}

// One fantasy's EI in nei_term, out of line like mes_term.
template <bool GRAD = false>
__device__ __noinline__ double nei_ei_term(double a, double sd, double* cm = nullptr, double* cs = nullptr) {
    return ei_term<GRAD>(a, sd, cm, cs);
}

// LogEI / LogPoI at a = mean - y_max - xi (include/b200bo.h), out of line like mes_term.  sigma = 0, or a sigma so
// small that z = a / sigma is infinite: the log of the EI limit max(a, 0) (log a, -inf, NaN at a = 0); log_ndtr has
// the PoI limits already (0 at z = +inf, -inf at -inf, NaN at NaN).
// GRAD: LogEI cm = r / sd, cs = q / sd (log_h_ratios); LogPoI cm = lambda / sd, cs = -z lambda / sd (inv_mills).
// sd = 0 or an infinite z: LogEI = log a for a > 0 has cm = 1/a; everything else is a constant (cm = cs = 0).
template <bool GRAD = false>
__device__ __noinline__ double log_acq_term(int kind, double a, double sd, double* cm = nullptr, double* cs = nullptr) {
    const double z = a / sd;
    if constexpr (GRAD) *cm = *cs = 0.0;
    if (kind == B200BO_ACQ_LOGPOI) {
        if (GRAD && sd > 0.0 && !isinf(z)) {
            const double lam = inv_mills(z);
            *cm = lam / sd;
            *cs = lam == 0.0 ? 0.0 : -z * lam / sd;
        }
        return log_ndtr(z);
    }
    if (sd == 0.0 || isinf(z)) {
        if (GRAD && a > 0.0) *cm = 1.0 / a;
        return a > 0.0 ? log(a) : (a < 0.0 ? -CUDART_INF : CUDART_NAN);
    }
    if constexpr (GRAD) {
        double r, q;
        log_h_ratios(z, r, q);
        *cm = r / sd;
        *cs = q / sd;
    }
    return log_h(z) + log(sd);
}

// log p of one constraint factor, p = Phi(u) - Phi(l), u = (ub - mean)/sd, l = (lb - mean)/sd: one-sided bounds
// through log_ndtr(u) / log_ndtr(-l); a pair in one tail reflected so that both arguments a <= b are <= 0, then
// log Phi(b) + log1mexp(log Phi(a) - log Phi(b)); a straddling pair directly.  A finite bound with sd <= 0 (or a NaN
// mean) is the frozen-norm NaN of norm_cdf_loc_scale.
// GRAD: cm = -(F_l + F_u) / sd, cs = -(l F_l + u F_u) / sd, with F_l, F_u the partials of log p in l and u, each ratio
// phi / p in the same tail-safe form as the value:
//   one-sided: F_u = lambda(u), F_l = -lambda(-l);   straddling: F_u = phi(u)/p, F_l = -phi(l)/p;
//   one tail, d = log Phi(a) - log Phi(b): phi(b)/p = lambda(b)/(-expm1(d)), phi(a)/p = lambda(a) e^d/(-expm1(d)),
//   with the signs of the reflection.  Where the value is NaN the coefficients are 0.
template <bool GRAD = false>
__device__ __noinline__ double log_cfactor(double lb, double ub, double mean, double sd, double* cm = nullptr,
                                           double* cs = nullptr) {
    if constexpr (GRAD) *cm = *cs = 0.0;
    const bool has_l = lb != -CUDART_INF, has_u = ub != CUDART_INF;
    if (!has_l && !has_u) return 0.0;
    if (!(sd > 0.0) || isnan(mean)) return CUDART_NAN;
    const double u = (ub - mean) / sd, l = (lb - mean) / sd;
    auto coef = [&](double fl, double fu) {
        *cm = -(fl + fu) / sd;
        *cs = -((fl == 0.0 ? 0.0 : l * fl) + (fu == 0.0 ? 0.0 : u * fu)) / sd;
    };
    if (!has_l) {
        if constexpr (GRAD) coef(0.0, inv_mills(u));
        return log_ndtr(u);
    }
    if (!has_u) {
        if constexpr (GRAD) coef(-inv_mills(-l), 0.0);
        return log_ndtr(-l);
    }
    if (l < 0.0 && u > 0.0) {
        const double p = ndtr(u) - ndtr(l);
        if constexpr (GRAD) coef(-norm_pdf(l) / p, norm_pdf(u) / p);
        return log(p);
    }
    const bool refl = l >= 0.0;
    const double a = refl ? -u : l, b = refl ? -l : u;
    const double lpb = log_ndtr(b), d = log_ndtr(a) - lpb;
    if constexpr (GRAD) {
        const double om = -expm1(d), gb = inv_mills(b) / om;
        const double la = inv_mills(a), ga = la == 0.0 ? 0.0 : -la * exp(d) / om;
        coef(refl ? -gb : ga, refl ? -ga : gb);
    }
    return lpb + log1mexp(d);
}

// p = Phi(u) - Phi(l) of one CNEI constraint factor, u = (ub - mean)/sd, l = (lb - mean)/sd: an infinite bound
// contributes 0 / 1 and a finite bound with sd <= 0 (or a NaN mean) is the frozen-norm NaN, as EI's factor.  A pair
// with l > 0 (the mean below the lower bound) is reflected, Phi(-l) - Phi(-u), so that a factor far in a constraint's
// tail keeps its digits instead of cancelling to 0 (EI's factor keeps the reference's unreflected form).
__device__ __forceinline__ double cnei_factor(double lb, double ub, double mean, double sd) {
    const bool has_l = lb != -CUDART_INF, has_u = ub != CUDART_INF;
    if (has_l && lb > mean && sd > 0.0)
        return ndtr((mean - lb) / sd) - (has_u ? ndtr((mean - ub) / sd) : 0.0);
    const double p_lo = has_l ? norm_cdf_loc_scale(lb, mean, sd) : 0.0;
    const double p_hi = has_u ? norm_cdf_loc_scale(ub, mean, sd) : 1.0;
    return p_hi - p_lo;
}

// NEI / LogNEI (DESIGN.md 4.13) of one candidate, out of line like mes_term and with scalar arguments only, so that
// the kernels that inline candidate_epilogue keep their register allocation.  The S fantasy means k*^T a_s
// (normalised units) come from the candidate's column of the K* tile the kernel already holds (kcol[i * kstr] =
// const_value k(xs, Xs_i)) and A = K0^-1 F ([np][S] row-major), each summed over the training rows in index order;
// best = best_0 .. best_{S-1} (data units).  NEI: the mean of the S EI terms in s order; LogNEI: the log of that mean
// from the LogEI terms, shifted by their maximum.
// GRAD: cms[s * kstr] (kcol's layout) = the coefficient of d mu_s, cs that of d sd:
//   NEI:    cms_s = Phi(z_s) / S,  cs = sum_s phi(z_s) / S                       (EI's cm / cs per fantasy, averaged)
//   LogNEI: cms_s = p_s cm_s,  cs = sum_s p_s cs_s,  p_s = exp(l_s - M) / sum exp(l - M)   (LogEI's, softmax-weighted)
template <bool GRAD = false>
__device__ __noinline__ double nei_term(int kind, const double* __restrict__ kcol, int kstr, int n,
                                        const double* __restrict__ A, const double* __restrict__ best, int S,
                                        double y_std, double y_mean, double xi, double sd, double* cms = nullptr,
                                        double* cs = nullptr) {
    double t[B200BO_MAX_PATHS], cm_s[B200BO_MAX_PATHS], cs_s[B200BO_MAX_PATHS];
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s) t[s] = 0.0;
    for (int i = 0; i < n; ++i) {
        const double k = kcol[(size_t)i * kstr];
        const double* a = A + (size_t)i * S;
#pragma unroll
        for (int s = 0; s < B200BO_MAX_PATHS; ++s)
            if (s < S) t[s] = fma(a[s], k, t[s]);
    }
    double c = 0.0;
    if (kind == B200BO_ACQ_NEI) {
        double sum = 0.0;
#pragma unroll
        for (int s = 0; s < B200BO_MAX_PATHS; ++s) {
            if (s < S) {
                sum += nei_ei_term<GRAD>(y_std * t[s] + y_mean - best[s] - xi, sd, grad_out<GRAD>(cm_s[s]),
                                         grad_out<GRAD>(cs_s[s]));
                if constexpr (GRAD) {
                    cms[s * kstr] = cm_s[s] / (double)S;
                    c += cs_s[s];
                }
            }
        }
        if constexpr (GRAD) *cs = c / (double)S;
        return sum / (double)S;
    }
    double mx = -CUDART_INF;
    bool nan = false;
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s) {
        if (s < S) {
            t[s] = log_acq_term<GRAD>(B200BO_ACQ_LOGEI, y_std * t[s] + y_mean - best[s] - xi, sd,
                                      grad_out<GRAD>(cm_s[s]), grad_out<GRAD>(cs_s[s]));
            nan = nan || isnan(t[s]);
            mx = fmax(mx, t[s]);
            if constexpr (GRAD) cms[s * kstr] = 0.0;
        }
    }
    if constexpr (GRAD) *cs = 0.0;
    if (nan) return CUDART_NAN;
    if (mx == -CUDART_INF) return -CUDART_INF;
    double e = 0.0;
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s)
        if (s < S) e += exp(t[s] - mx);
    if constexpr (GRAD) {
#pragma unroll
        for (int s = 0; s < B200BO_MAX_PATHS; ++s) {
            if (s < S) {
                const double p = exp(t[s] - mx) / e;
                cms[s * kstr] = p * cm_s[s];
                c += p * cs_s[s];
            }
        }
        *cs = c;
    }
    return mx + log(e) - log((double)S);
}

// CNEI / LogCNEI (DESIGN.md 4.15) of one candidate, GP g of n_gps, out of line like nei_term.  The S fantasy means
// y_std k*^T a_gs + y_mean of GP g come from its K* column kcol (kcol[i * kstr]) and A_g, summed as in nei_term.  g = 0
// forms the per-sample target terms EI_s (LogEI_s), each constraint GP multiplies in P_gs (adds log P_gs), and the
// running terms wait in carry[s * kstr] between the GP passes of a candidate.  At the last GP the terms are reduced
// over s exactly as nei_term reduces them (returned value alpha); before it the return value is unused.
__device__ __noinline__ double cnei_term(int kind, int g, int n_gps, const double* __restrict__ kcol, int kstr, int n,
                                         const double* __restrict__ A, const double* __restrict__ best, int S,
                                         double y_std, double y_mean, double xi, double lb, double ub, double sd,
                                         double* __restrict__ carry) {
    double t[B200BO_MAX_PATHS];
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s) t[s] = 0.0;
    for (int i = 0; i < n; ++i) {
        const double k = kcol[(size_t)i * kstr];
        const double* a = A + (size_t)i * S;
#pragma unroll
        for (int s = 0; s < B200BO_MAX_PATHS; ++s)
            if (s < S) t[s] = fma(a[s], k, t[s]);
    }
    const bool lg = kind == B200BO_ACQ_LOGCNEI, last = g == n_gps - 1;
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s) {
        if (s < S) {
            const double mean = y_std * t[s] + y_mean;
            double v;
            if (g == 0) {
                v = lg ? log_acq_term(B200BO_ACQ_LOGEI, mean - best[s] - xi, sd) : nei_ei_term(mean - best[s] - xi, sd);
            } else if (lg) {
                v = carry[s * kstr] + log_cfactor(lb, ub, mean, sd);
            } else {
                v = carry[s * kstr] * cnei_factor(lb, ub, mean, sd);
            }
            if (last)
                t[s] = v;
            else
                carry[s * kstr] = v;
        }
    }
    if (!last) return 0.0;
    if (!lg) {
        double sum = 0.0;
#pragma unroll
        for (int s = 0; s < B200BO_MAX_PATHS; ++s)
            if (s < S) sum += t[s];
        return sum / (double)S;
    }
    double mx = -CUDART_INF;
    bool nan = false;
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s) {
        if (s < S) {
            nan = nan || isnan(t[s]);
            mx = fmax(mx, t[s]);
        }
    }
    if (nan) return CUDART_NAN;
    if (mx == -CUDART_INF) return -CUDART_INF;
    double e = 0.0;
#pragma unroll
    for (int s = 0; s < B200BO_MAX_PATHS; ++s)
        if (s < S) e += exp(t[s] - mx);
    return mx + log(e) - log((double)S);
}

// ---- per-candidate epilogue shared by the tiled and the small-batch kernels ---------------------
// mu_n: K* alpha_ (normalised units); colsq: sum_i V_i^2.  g = 0: target GP -> base acquisition;
// g >= 1: constraint GP -> probability factor.  The last GP writes -base * prod.
// MES: base = (1/K) sum_k, in k order, mes_term((y*_k - mean) / sd); base = 0 when sd == 0 (a clamped variance:
// the predictive distribution is a point mass, an observation there teaches nothing).
// LogEI / LogPoI: base_neg = -log_acq_term, then base_neg -= log p_g per constraint GP, which is -(alpha + sum log p)
// summed in g order bit for bit (negation is exact); prod stays 1 and is not used.
// NEI (template flag, set in the kernel instantiations that serve NEI / LogNEI only, so that every other
// instantiation compiles as without these kinds): base = nei_term over the candidate's K* column kcol (stride kstr);
// constraints as for EI / LogEI.
// GRAD: *gr = this GP's term (the base acquisition for g = 0, the factor p or log p for g >= 1) and its coefficients.
// sd == 0 (a clamped or vanished variance): the caller sets d sd := 0, and the coefficients that divide by sd (PoI,
// MES, the factors) are 0 - the value there is a step or constant in x.
struct EpilogueGrad {
    double term, cm, cs;
    double* cms;  // NEI: the coefficients of d mu_s, cms[s * kstr] (nei_term); cm is 0
};

// CNEI (template flag of the instantiations that serve CNEI / LogCNEI only, value form): every GP's pass goes to
// cnei_term over GP g's K* column kcol, with the per-sample carry at carry[s * kstr]; the last GP writes -alpha.
template <bool NEI = false, bool GRAD = false, bool CNEI = false>
__device__ __forceinline__ void candidate_epilogue(const PredictParams& P, const GpDev& G, int g,
                                                   double mu_n, double colsq, long long gi,
                                                   double& base_neg, double& prod, double* final_val = nullptr,
                                                   const double* kcol = nullptr, int kstr = 0,
                                                   EpilogueGrad* gr = nullptr, double* carry = nullptr) {
    const bool logk = acq_constraints_in_log<NEI>(P.acq_kind);
    const double mean = G.y_std * mu_n + G.y_mean;
    double var = G.prior - colsq;
    if (var < 0.0) {
        var = 0.0;
        if (P.clamp_count && gi < P.m) atomicAdd(P.clamp_count, 1ull);
    }
    const double sd = sqrt(var * (G.y_std * G.y_std));
    if constexpr (CNEI) {
        static_assert(!GRAD && !NEI, "CNEI has a value form only");
        const double a = cnei_term(P.acq_kind, g, P.n_gps, kcol, kstr, G.n, P.fant_a_gp[g],
                                   P.fant_a + (size_t)P.gp[0].np * P.n_ystar, P.n_ystar, G.y_std, G.y_mean, P.xi,
                                   G.lb, G.ub, sd, carry);
        if (g == P.n_gps - 1) {
            const double val = -1.0 * a;
            if (final_val) *final_val = val;
            if (P.acq_out && gi < P.m) P.acq_out[gi] = val;
        }
        return;
    }
    double term = 0.0, cm = 0.0, cs = 0.0;
    if (g == 0) {
        if (P.acq_kind == B200BO_ACQ_UCB) {
            term = mean + P.kappa * sd;
            cm = 1.0;
            cs = P.kappa;
        } else if (P.acq_kind == B200BO_ACQ_EI) {
            const double a = mean - P.y_max - P.xi;
            if constexpr (GRAD) {
                // the FMA every value kernel contracts ei_term's sum to, written out: left to the compiler, this form
                // fuses the other product and the value loses its bits
                const double z = a / sd;
                cm = ndtr(z);
                cs = norm_pdf(z);
                term = fma(sd, cs, a * cm);
            } else {
                term = ei_term(a, sd);
            }
        } else if (P.acq_kind == B200BO_ACQ_POI) {
            const double z = (mean - P.y_max - P.xi) / sd;
            term = ndtr(z);
            if (GRAD && sd > 0.0) {
                const double pz = norm_pdf(z);
                cm = pz / sd;
                cs = pz == 0.0 ? 0.0 : -z * pz / sd;
            }
        } else if (P.acq_kind == B200BO_ACQ_MES) {
            if (sd > 0.0) {
                double s = 0.0, sm = 0.0, ss = 0.0;
                for (int k = 0; k < P.n_ystar; ++k) {
                    const double gk = (P.ystar[k] - mean) / sd;
                    double td;
                    s += mes_term<GRAD>(gk, grad_out<GRAD>(td));
                    if constexpr (GRAD) {
                        sm += td;
                        ss += td == 0.0 ? 0.0 : td * gk;
                    }
                }
                term = s / (double)P.n_ystar;
                cm = -sm / ((double)P.n_ystar * sd);
                cs = -ss / ((double)P.n_ystar * sd);
            }
        } else if (NEI && acq_is_nei(P.acq_kind)) {
            term = nei_term<GRAD>(P.acq_kind, kcol, kstr, G.n, P.fant_a, P.fant_a + (size_t)G.np * P.n_ystar,
                                  P.n_ystar, G.y_std, G.y_mean, P.xi, sd, GRAD ? gr->cms : nullptr,
                                  grad_out<GRAD>(cs));
        } else if (acq_constraints_in_log<false>(P.acq_kind)) {  // LogEI / LogPoI
            term = log_acq_term<GRAD>(P.acq_kind, mean - P.y_max - P.xi, sd, grad_out<GRAD>(cm), grad_out<GRAD>(cs));
        }
        base_neg = -1.0 * term;
        prod = 1.0;
        if (gi < P.m) {
            if (P.mu_out) P.mu_out[gi] = mean;
            if (P.sd_out) P.sd_out[gi] = sd;
        }
    } else if (logk) {
        // base_neg is read before the call, the order the value kernels have always been compiled from
        base_neg = base_neg -
                   (term = log_cfactor<GRAD>(G.lb, G.ub, mean, sd, grad_out<GRAD>(cm), grad_out<GRAD>(cs)));
    } else {
        const double p_lo = (G.lb == -CUDART_INF) ? 0.0 : norm_cdf_loc_scale(G.lb, mean, sd);
        const double p_hi = (G.ub == CUDART_INF) ? 1.0 : norm_cdf_loc_scale(G.ub, mean, sd);
        // constraint.py:208 (J=1: result = p_hi - p_lo) / :219 (result *= ...)
        prod = (g == 1) ? (p_hi - p_lo) : prod * (p_hi - p_lo);
        if constexpr (GRAD) {
            term = p_hi - p_lo;
            if (sd > 0.0) {
                if (G.lb != -CUDART_INF) {
                    const double z = (G.lb - mean) / sd, pz = norm_pdf(z);
                    cm += pz / sd;
                    cs += pz == 0.0 ? 0.0 : z * pz / sd;
                }
                if (G.ub != CUDART_INF) {
                    const double z = (G.ub - mean) / sd, pz = norm_pdf(z);
                    cm -= pz / sd;
                    cs -= pz == 0.0 ? 0.0 : z * pz / sd;
                }
            }
        }
    }
    if constexpr (GRAD) {
        gr->term = term;
        gr->cm = cm;
        gr->cs = cs;
    }
    if (g == P.n_gps - 1) {
        const double val = (P.n_gps > 1 && !logk) ? base_neg * prod : base_neg;
        if (final_val) *final_val = val;
        if (P.acq_out && gi < P.m) P.acq_out[gi] = val;
    }
}

// ---- B200BO_ACQ_MEAN: the posterior-mean merit (include/b200bo.h, DESIGN.md 4.17) -----------------------------
// Constraint GP G's violation at its posterior mean (data units): an infinite bound contributes 0 (the short-circuits
// of the constraint factors), max(0, .) propagates NaN as np.maximum does, and the explicit _rn intrinsics keep FMA
// contraction out, so that the numpy restatement reproduces the value bit for bit.
__device__ __forceinline__ double mean_pos(double x) { return (x > 0.0 || x != x) ? x : 0.0; }
__device__ __forceinline__ double mean_viol(const GpDev& G, double mean) {
    const double lo = G.lb == -CUDART_INF ? 0.0 : mean_pos(__dsub_rn(G.lb, mean));
    const double hi = G.ub == CUDART_INF ? 0.0 : mean_pos(__dsub_rn(mean, G.ub));
    return __dadd_rn(lo, hi);
}
// -merit: -mu_0 where viol = 0, else T (1 + viol) (= -(-T (1 + viol)) exactly)
__device__ __forceinline__ double mean_merit_neg(double mu0, double viol, double T) {
    return viol == 0.0 ? -mu0 : __dmul_rn(T, __dadd_rn(1.0, viol));
}

// ---- phase A: the tile's K*^T (np x PBN) + K* alpha_ -----------------------------------------------
// Every fused predict kernel builds its tile's covariances with this one function, so the tile kernels, the bound pass
// and the refine / units stages get the same K* entries and the same mu = K* alpha_, bit for bit (DESIGN.md 4.9).
// Thread = one candidate column; the NT / PBN threads of a column split the rows of every chunk into parts.  Training
// rows stream through shared memory in chunks of 64 (double-buffered cp.async), so every row read is a warp-wide
// broadcast LDS; DREG keeps the candidate's coordinates in registers (d <= 16).  COV is a template parameter so that
// the covariance is branch-free straight-line code.
constexpr int PA_CHUNK = 64;  // training rows per staged chunk

// Where phase A puts K* (KS):
//   KS_F64     fp64 [np][KSTR], plain stores (the 8-warp kernel)
//   KS_F64_EF  fp64 [np][KSTR], stores under the L2 policy pol_first (evict_first: the CTA-private scratch is written
//              once and swept cyclically, LRU-hostile).  KSTR = PBN for the cp.async phase B, PSTR_DMMA for the
//              bulk-copy phase B: the rows of a stage are then contiguous in global memory exactly as in shared memory.
//   KS_TF32    tf32 (hi, lo) pairs in the wgmma operand-image layout of tc_common.cuh ([np/32][hi|lo][16 KiB],
//              candidate = operand row, training index = K), fenced for the bulk copies that read them (fp32 mode)
//   KS_KMAX    nowhere: each thread keeps the largest |K*_i| of its rows in kmax_s[part][c] (the bound pass of pruning)
//   KS_NONE    nowhere, and no kmax: mu_s only (the mean-only kernel of B200BO_ACQ_MEAN)
// mu_s[part][c] is the part's share of K* alpha_; each caller adds the NT / PBN parts in its fixed order.
// Column c is candidate c0 + c of the first mlim, or perm[c0 + c] when perm is set (tiles in bound order); rows: the
// leading training rows to build (a multiple of PA_CHUNK; G.np for all of them - mu_s is K* alpha_ only then); row0
// (a multiple of PA_CHUNK, 0 but in ks_build_kernel): the rows before it are skipped, mu_s is then meaningless.
enum { KS_F64, KS_F64_EF, KS_TF32, KS_KMAX, KS_NONE };

__device__ __forceinline__ void st_global_hint(double* p, double v, unsigned long long pol) {
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;\n" ::"l"(p), "d"(v), "l"(pol) : "memory");
}

template <int NT, bool DREG, int KS, int KSTR, int COV>
__device__ __forceinline__ void phase_a_impl(const PredictParams& P, const GpDev& G, long long c0,
                                             double* __restrict__ Ks, double* smem, double (*mu_s)[PBN],
                                             unsigned long long pol_first, double (*kmax_s)[PBN], const int* perm,
                                             long long mlim, int rows, int row0) {
    constexpr int ROWS = PA_CHUNK / (NT / PBN);  // rows of every chunk per thread
    const int tid = threadIdx.x;
    const int d = P.d, np = G.np;
    double* xc_s = smem;                             // [d][PBN]
    double* xs_s = smem + (size_t)d * PBN;           // [2][PA_CHUNK][d]
    double* al_s = xs_s + (size_t)2 * PA_CHUNK * d;  // [2][PA_CHUNK] alpha_ of the staged rows
    for (int idx = tid; idx < PBN * d; idx += NT) {
        const int c = idx / d, j = idx - c * d;
        const long long gi = c0 + c;
        double v = 0.0;
        if (gi < mlim) v = scale_input(candidate_coord(P, perm ? (long long)perm[gi] : gi, j), G.xform, G.ls, j);
        xc_s[j * PBN + c] = v;
    }
    const int chunk_pieces = PA_CHUNK * d / 2;  // 16-byte pieces per chunk (PA_CHUNK*d is even)
    auto load_chunk = [&](int buf, int ch) {
        const double* src = G.Xs + (size_t)ch * PA_CHUNK * d;
        double* dst = xs_s + (size_t)buf * PA_CHUNK * d;
        for (int q = tid; q < chunk_pieces; q += NT) cp_async16_cg(dst + 2 * q, src + 2 * q);
        if (tid < PA_CHUNK / 2)
            cp_async16_cg(al_s + buf * PA_CHUNK + 2 * tid, G.alphav + (size_t)ch * PA_CHUNK + 2 * tid);
    };
    // The 256-thread kernels always build all np rows; they take np from G here rather than rows from the call site,
    // because where that load sits steers their instruction schedule (read at the call, fp32 mode ran 0.2 % slower on an
    // H100 80GB HBM3 at 700 W).
    const int nch = (NT == PNT ? np : rows) / PA_CHUNK, ch0 = row0 / PA_CHUNK;
    load_chunk(ch0 & 1, ch0);
    cp_async_commit();
    __syncthreads();  // xc_s visible
    const int c = tid & (PBN - 1), part = tid >> 7;  // part in [0, NT / PBN)
    double xc[kPredictMaxDimRegs];
    if (DREG) {
#pragma unroll
        for (int j = 0; j < kPredictMaxDimRegs; ++j) xc[j] = (j < d) ? xc_s[j * PBN + c] : 0.0;
    }
    double mu_acc = 0.0, kmax = 0.0;
    constexpr int R = 8;
    for (int ch = ch0; ch < nch; ++ch) {
        if (ch + 1 < nch) load_chunk((ch + 1) & 1, ch + 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        const double* xs = xs_s + (size_t)(ch & 1) * PA_CHUNK * d;
        const double* al = al_s + (ch & 1) * PA_CHUNK;
        for (int r0 = part * ROWS; r0 < (part + 1) * ROWS; r0 += R) {
            double r2[R];
#pragma unroll
            for (int q = 0; q < R; ++q) r2[q] = 0.0;
            if (DREG && (d & 1) == 0) {
#pragma unroll
                for (int j = 0; j < kPredictMaxDimRegs; j += 2) {
                    if (j < d) {
#pragma unroll
                        for (int q = 0; q < R; ++q) {
                            const double2 xv = *reinterpret_cast<const double2*>(xs + (r0 + q) * d + j);
                            const double d0 = xc[j] - xv.x, d1 = xc[j + 1] - xv.y;
                            r2[q] = fma(d0, d0, r2[q]);
                            r2[q] = fma(d1, d1, r2[q]);
                        }
                    }
                }
            } else if (DREG) {
#pragma unroll
                for (int j = 0; j < kPredictMaxDimRegs; ++j) {
                    if (j < d) {
#pragma unroll
                        for (int q = 0; q < R; ++q) {
                            const double df = xc[j] - xs[(r0 + q) * d + j];
                            r2[q] = fma(df, df, r2[q]);
                        }
                    }
                }
            } else {
                for (int j = 0; j < d; ++j) {
                    const double xv = xc_s[j * PBN + c];
#pragma unroll
                    for (int q = 0; q < R; ++q) {
                        const double df = xv - xs[(r0 + q) * d + j];
                        r2[q] = fma(df, df, r2[q]);
                    }
                }
            }
            float hi[R], lo[R];
#pragma unroll
            for (int q = 0; q < R; ++q) {
                const int n = ch * PA_CHUNK + r0 + q;
                double kv = G.constv * cov_eval<COV>(r2[q]);
                if (n >= G.n) kv = 0.0;
                if constexpr (KS == KS_F64) {
                    Ks[(size_t)n * KSTR + c] = kv;
                } else if constexpr (KS == KS_F64_EF) {
                    st_global_hint(Ks + (size_t)n * KSTR + c, kv, pol_first);
                } else if constexpr (KS == KS_TF32) {
                    hi[q] = tc::to_tf32((float)kv);
                    lo[q] = tc::to_tf32((float)(kv - (double)hi[q]));
                } else if constexpr (KS == KS_KMAX) {
                    kmax = fmax(kmax, fabs(kv));
                }
                mu_acc = fma(al[r0 + q], kv, mu_acc);
            }
            if constexpr (KS == KS_TF32) {
                const int n0 = ch * PA_CHUNK + r0;  // multiple of 8: two groups of 4 consecutive k
                uint8_t* img = reinterpret_cast<uint8_t*>(Ks) + (size_t)(n0 >> 5) * (2 * tc::kTcImgBytes);
#pragma unroll
                for (int h4 = 0; h4 < 2; ++h4) {
                    const int off = tc::tc_img_offset(c, (n0 & 31) + 4 * h4);
                    *reinterpret_cast<float4*>(img + off) =
                        make_float4(hi[4 * h4], hi[4 * h4 + 1], hi[4 * h4 + 2], hi[4 * h4 + 3]);
                    *reinterpret_cast<float4*>(img + tc::kTcImgBytes + off) =
                        make_float4(lo[4 * h4], lo[4 * h4 + 1], lo[4 * h4 + 2], lo[4 * h4 + 3]);
                }
            }
        }
        __syncthreads();  // chunk buffer free for the prefetch of chunk ch+2
    }
    cp_async_wait<0>();
    mu_s[part][c] = mu_acc;
    if constexpr (KS == KS_KMAX) kmax_s[part][c] = kmax;
    if constexpr (KS == KS_TF32) {
        tc::fence_proxy_async_global();  // scratch images will be read by bulk async copies
        tc::fence_proxy_async_smem();    // and the stage buffers overwritten by them
    }
    __threadfence_block();
    __syncthreads();
}

template <int NT, bool DREG, int KS, int KSTR = PBN>
__device__ __forceinline__ void phase_a(const PredictParams& P, const GpDev& G, long long c0, double* __restrict__ Ks,
                                        double* smem, double (*mu_s)[PBN], unsigned long long pol_first,
                                        double (*kmax_s)[PBN], const int* perm, long long mlim, int rows,
                                        int row0 = 0) {
    switch (cov_code(G.family, G.nu)) {
        case 0:
            phase_a_impl<NT, DREG, KS, KSTR, 0>(P, G, c0, Ks, smem, mu_s, pol_first, kmax_s, perm, mlim, rows, row0);
            break;
        case 1:
            phase_a_impl<NT, DREG, KS, KSTR, 1>(P, G, c0, Ks, smem, mu_s, pol_first, kmax_s, perm, mlim, rows, row0);
            break;
        case 2:
            phase_a_impl<NT, DREG, KS, KSTR, 2>(P, G, c0, Ks, smem, mu_s, pol_first, kmax_s, perm, mlim, rows, row0);
            break;
        default:
            phase_a_impl<NT, DREG, KS, KSTR, 3>(P, G, c0, Ks, smem, mu_s, pol_first, kmax_s, perm, mlim, rows, row0);
            break;
    }
}

// stage loader shared by both GEMM variants: BK k-rows x 128 doubles of LinvT and of K*
template <int STR, int BK>
__device__ __forceinline__ void predict_load_stage(double* as, double* bs, const double* Ag,
                                                   const double* Bg, int np) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int t = 0; t < BK / 4; ++t) {
        const int q = tid + t * PNT;
        const int kk = q >> 6, m2 = (q & 63) * 2;
        cp_async16_cg(as + kk * STR + m2, Ag + (size_t)kk * np + m2);
        cp_async16_cg(bs + kk * STR + m2, Bg + kk * PBN + m2);
    }
}

// ---- phase B (DFMA): 8x8 register tiles; returns per-column sums of V^2 in red[16][PBN] -------
__device__ __forceinline__ void predict_phase_b_dfma(const GpDev& G, const double* __restrict__ Ks,
                                                     double* smem) {
    constexpr int STR = PSTR_DFMA, BK = PBK;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int np = G.np;
    double* As = smem;
    double* Bs = smem + PSTAGES * BK * STR;
    double csq[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) csq[j] = 0.0;
    const int nb = np / PBM;
    for (int ib = 0; ib < nb; ++ib) {
        double acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
        const int nks = (ib + 1) * (PBM / BK);
        const double* Abase = G.linvT + (size_t)ib * PBM;
#pragma unroll
        for (int s = 0; s < PSTAGES - 1; ++s) {
            if (s < nks)
                predict_load_stage<STR, BK>(As + s * BK * STR, Bs + s * BK * STR,
                                            Abase + (size_t)(s * BK) * np, Ks + (size_t)(s * BK) * PBN, np);
            cp_async_commit();
        }
        for (int ks = 0; ks < nks; ++ks) {
            cp_async_wait<PSTAGES - 2>();
            __syncthreads();
            const int nxt = ks + PSTAGES - 1;
            if (nxt < nks)
                predict_load_stage<STR, BK>(As + (nxt % PSTAGES) * BK * STR, Bs + (nxt % PSTAGES) * BK * STR,
                                            Abase + (size_t)(nxt * BK) * np, Ks + (size_t)(nxt * BK) * PBN, np);
            cp_async_commit();
            const double* as = As + (ks % PSTAGES) * BK * STR;
            const double* bs = Bs + (ks % PSTAGES) * BK * STR;
#pragma unroll
            for (int kk = 0; kk < PBK; ++kk) {
                double a[8], b[8];
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const double2 t = *reinterpret_cast<const double2*>(as + kk * STR + p * 32 + ty * 2);
                    a[2 * p] = t.x;
                    a[2 * p + 1] = t.y;
                }
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const double2 t = *reinterpret_cast<const double2*>(bs + kk * STR + p * 32 + tx * 2);
                    b[2 * p] = t.x;
                    b[2 * p + 1] = t.y;
                }
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
            }
        }
        cp_async_wait<0>();
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < 8; ++i) s = fma(acc[i][j], acc[i][j], s);
            csq[j] += s;
        }
    }
    double* red = smem;  // [16][PBN]
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        red[ty * PBN + p * 32 + tx * 2] = csq[2 * p];
        red[ty * PBN + p * 32 + tx * 2 + 1] = csq[2 * p + 1];
    }
    __syncthreads();
}

// ---- phase B (DMMA): mma.sync m8n8k4 f64; warp tile 32(m) x 64(n); red[4][PBN] -----------------
__device__ __forceinline__ void predict_phase_b_dmma(const GpDev& G, const double* __restrict__ Ks,
                                                     double* smem) {
    constexpr int STR = PSTR_DMMA, BK = PBK_DMMA;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // warps w and w+4 share an SM sub-partition: give them row slabs s and 3-s so that skipping
    // the structurally-zero part of the diagonal block (k beyond the slab's last row) leaves every
    // sub-partition with the same amount of work
    const int wn = warp >> 2;
    const int wm = wn ? 3 - (warp & 3) : (warp & 3);
    const int g = lane >> 2, t4 = lane & 3;
    const int np = G.np;
    double* As = smem;
    double* Bs = smem + PSTAGES * BK * STR;
    double csq[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) csq[j][0] = csq[j][1] = 0.0;
    const int nb = np / PBM;
    for (int ib = 0; ib < nb; ++ib) {
        double acc[4][8][2];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
        const int nks = (ib + 1) * (PBM / BK);
        const double* Abase = G.linvT + (size_t)ib * PBM;
#pragma unroll
        for (int s = 0; s < PSTAGES - 1; ++s) {
            if (s < nks)
                predict_load_stage<STR, BK>(As + s * BK * STR, Bs + s * BK * STR,
                                            Abase + (size_t)(s * BK) * np, Ks + (size_t)(s * BK) * PBN, np);
            cp_async_commit();
        }
        for (int ks = 0; ks < nks; ++ks) {
            cp_async_wait<PSTAGES - 2>();
            __syncthreads();
            const int nxt = ks + PSTAGES - 1;
            // diagonal block of L^-1 (k in [ib*128, ib*128+128)): rows wm*32.. have zeros for
            // k > row, so the k-tiles beyond this warp's slab contribute nothing
            const bool live = ks * BK < ib * PBM + (wm + 1) * 32;
            const double* as = As + (ks % PSTAGES) * BK * STR + wm * 32 + g;
            const double* bs = Bs + (ks % PSTAGES) * BK * STR + wn * 64 + g;
#pragma unroll
            for (int k4 = 0; k4 < BK / 4; ++k4) {
                if (k4 == 1) {
                    // prefetch issued behind the first batch of MMAs so the tensor pipe is already
                    // busy while the LDGSTS addresses are generated
                    if (nxt < nks)
                        predict_load_stage<STR, BK>(As + (nxt % PSTAGES) * BK * STR, Bs + (nxt % PSTAGES) * BK * STR,
                                                    Abase + (size_t)(nxt * BK) * np, Ks + (size_t)(nxt * BK) * PBN, np);
                    cp_async_commit();
                }
                if (live) {
                    double a[4], b[8];
                    const int krow = (k4 * 4 + t4) * STR;
#pragma unroll
                    for (int i = 0; i < 4; ++i) a[i] = as[krow + i * 8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) b[j] = bs[krow + j * 8];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i], b[j]);
                }
            }
        }
        cp_async_wait<0>();
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
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
    // rows of one m8 fragment live in lanes with equal (lane & 3): butterfly over lane bits 2..4
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            double v = csq[j][e];
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            csq[j][e] = v;
        }
    double* red = smem;  // [4][PBN]
    if (g == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            red[wm * PBN + wn * 64 + j * 8 + t4 * 2] = csq[j][0];
            red[wm * PBN + wn * 64 + j * 8 + t4 * 2 + 1] = csq[j][1];
        }
    }
    __syncthreads();
}

template <int IMPL, bool DREG>
__global__ void __launch_bounds__(PNT, 1) predict_acq_kernel(const PredictParams P) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[2][PBN];
    __shared__ double base_s[PBN];
    __shared__ double prod_s[PBN];
    __shared__ SelShared sel_s;

    const int tid = threadIdx.x;
    double* Ks = P.scratch + (long long)blockIdx.x * P.scratch_stride;
    const long long ntiles = (P.m + PBN - 1) / PBN;
    constexpr int NRED = (IMPL == PREDICT_IMPL_DMMA) ? 4 : 16;
    if (P.sel_cta) {
        if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
        __syncthreads();
    }

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long c0 = tile * PBN;
        for (int g = 0; g < P.n_gps; ++g) {
            const GpDev& G = P.gp[g];
            phase_a<PNT, DREG, KS_F64>(P, G, c0, Ks, smem, mu_s, 0ull, nullptr, nullptr, P.m, G.np);
            if (IMPL == PREDICT_IMPL_DMMA)
                predict_phase_b_dmma(G, Ks, smem);
            else
                predict_phase_b_dfma(G, Ks, smem);
            const double* red = smem;

            // ---------------- phase C: per-candidate epilogue --------------------------------
            if (tid < PBN) {
                const int c = tid;
                double colsq = 0.0;
#pragma unroll
                for (int r = 0; r < NRED; ++r) colsq += red[r * PBN + c];
                double val = 0.0;
                candidate_epilogue(P, G, g, mu_s[0][c] + mu_s[1][c], colsq, c0 + c, base_s[c], prod_s[c], &val);
                if (P.sel_cta && g == P.n_gps - 1)
                    runsel_update<1>(sel_s, P.sel_k, tid, val, c0 + c + P.index_base, c0 + c < P.m);
            }
            __syncthreads();
        }
    }
    if (P.sel_cta && tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
}

// =======================================================================================
// fp32 mode: the same fused kernel with the N^2 term on the warpgroup tensor cores (wgmma).
//   V = L^-1 K*^T as 3xTF32 (a_hi*b_hi + a_hi*b_lo + a_lo*b_hi), fp32 accumulators in registers.
//   K* itself, K* alpha_ (the mean) and the whole epilogue stay fp64: only the triangular product
//   and the sum of squares run at reduced precision (tolerance of this mode: 1e-3).
// Warp roles during the GEMM phase (one CTA per SM, 256 threads):
//   warp 0 / lane 0  producer: 1-D bulk async copies (TMA engine) of pre-tiled operand images
//                    [A_hi|A_lo] (L^-1, tiled once at fit time) and [B_hi|B_lo] (written by phase A)
//                    into a ring of TC_STAGES shared-memory stages, completion on mbarriers
//   warps 4..7       one warpgroup: per 32-k stage 4 k-steps x 3 products x 2 row halves of
//                    wgmma.m64n128k8 into a 128 x 128 register accumulator; after each 128-row block
//                    of L^-1 the per-column sums of squares of the accumulator
// The operand images use the no-swizzle K-major core-matrix layout, so a stage is a verbatim
// 64 KiB byte copy - no tensor map, no swizzle bookkeeping.
// =======================================================================================
constexpr int TC_STAGES = 3;
constexpr int TC_STAGE_BYTES = 4 * tc::kTcImgBytes;                // A_hi, A_lo, B_hi, B_lo
constexpr int kPredictSmemBytesTc = TC_STAGES * TC_STAGE_BYTES;    // 196608

template <bool DREG>
__global__ void __launch_bounds__(PNT, 1) predict_acq_tc_kernel(const PredictParams P) {
    extern __shared__ __align__(16) double smem[];
    __shared__ double mu_s[2][PBN];
    __shared__ double base_s[PBN];
    __shared__ double prod_s[PBN];
    __shared__ double red_s[4][PBN];
    __shared__ uint64_t full_bar[TC_STAGES], empty_bar[TC_STAGES];
    __shared__ SelShared sel_s;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint8_t* stage_mem = reinterpret_cast<uint8_t*>(smem);
    double* Ks = P.scratch + (long long)blockIdx.x * P.scratch_stride;  // holds the B images (bytes)
    const long long ntiles = (P.m + PBN - 1) / PBN;
    if (P.sel_cta) {
        if (tid < PBN) runsel_begin(sel_s, P.sel_cta + blockIdx.x, P.sel_resume, tid);
        __syncthreads();
    }

    if (tid == 0) {
        for (int s = 0; s < TC_STAGES; ++s) {
            tc::mbar_init(&full_bar[s], 1);
            tc::mbar_init(&empty_bar[s], 4);  // one arrival per consumer warp
        }
        tc::mbar_fence_init();
    }
    __syncthreads();

    uint32_t stage_it = 0;  // stages filled / consumed so far (producer and consumers count alike)

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long c0 = tile * PBN;
        for (int g = 0; g < P.n_gps; ++g) {
            const GpDev& G = P.gp[g];
            phase_a<PNT, DREG, KS_TF32>(P, G, c0, Ks, smem, mu_s, 0ull, nullptr, nullptr, P.m, G.np);
            const int nb = G.np / PBM;
            const int nkt_row = G.np / tc::kTcK;  // images per row block in the A array
            const uint8_t* Bimg = reinterpret_cast<const uint8_t*>(Ks);

            if (warp == 0) {
                if (lane == 0) {
                    uint32_t it = stage_it;
                    for (int ib = 0; ib < nb; ++ib) {
                        const int nkt = (ib + 1) * (PBM / tc::kTcK);
                        const uint8_t* Aimg = G.linv_tc + (size_t)ib * nkt_row * (2 * tc::kTcImgBytes);
                        for (int kt = 0; kt < nkt; ++kt, ++it) {
                            const int s = it % TC_STAGES;
                            tc::mbar_wait(&empty_bar[s], ((it / TC_STAGES) & 1) ^ 1);
                            tc::mbar_arrive_expect_tx(&full_bar[s], TC_STAGE_BYTES);
                            uint8_t* dst = stage_mem + (size_t)s * TC_STAGE_BYTES;
                            tc::bulk_g2s(dst, Aimg + (size_t)kt * (2 * tc::kTcImgBytes), 2 * tc::kTcImgBytes,
                                         &full_bar[s]);
                            tc::bulk_g2s(dst + 2 * tc::kTcImgBytes, Bimg + (size_t)kt * (2 * tc::kTcImgBytes),
                                         2 * tc::kTcImgBytes, &full_bar[s]);
                        }
                    }
                }
            } else if (warp >= 4) {
                const int q = warp & 3;
                // per-thread column sums of V^2: columns 8*i + 2*(lane%4) + e
                float csq[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) csq[j] = 0.f;
                uint32_t it = stage_it;
                for (int ib = 0; ib < nb; ++ib) {
                    const int nkt = (ib + 1) * (PBM / tc::kTcK);
                    float acc[2][64];
                    int pending = -1;  // stage whose MMAs may still be reading shared memory
                    for (int kt = 0; kt < nkt; ++kt, ++it) {
                        const int s = it % TC_STAGES;
                        tc::mbar_wait(&full_bar[s], (it / TC_STAGES) & 1);
                        const uint32_t base = tc::smem_u32(stage_mem + (size_t)s * TC_STAGE_BYTES);
                        tc::wgmma_fence();
#pragma unroll
                        for (int j = 0; j < tc::kTcK / 8; ++j) {
                            const uint32_t koff = j * 2 * tc::kTcLBO;
                            const uint64_t b_hi = tc::wgmma_desc_kmajor_noswz(base + 2 * tc::kTcImgBytes + koff,
                                                                              tc::kTcLBO, tc::kTcSBO);
                            const uint64_t b_lo = tc::wgmma_desc_kmajor_noswz(base + 3 * tc::kTcImgBytes + koff,
                                                                              tc::kTcLBO, tc::kTcSBO);
#pragma unroll
                            for (int h = 0; h < 2; ++h) {  // rows 64h .. 64h+63 of the block: 8 core matrices
                                const uint32_t moff = h * 8 * tc::kTcSBO;
                                const uint64_t a_hi = tc::wgmma_desc_kmajor_noswz(base + moff + koff, tc::kTcLBO,
                                                                                  tc::kTcSBO);
                                const uint64_t a_lo = tc::wgmma_desc_kmajor_noswz(
                                    base + tc::kTcImgBytes + moff + koff, tc::kTcLBO, tc::kTcSBO);
                                tc::wgmma_m64n128k8_tf32(acc[h], a_hi, b_hi, (kt | j) ? 1u : 0u);
                                tc::wgmma_m64n128k8_tf32(acc[h], a_hi, b_lo, 1u);
                                tc::wgmma_m64n128k8_tf32(acc[h], a_lo, b_hi, 1u);
                            }
                        }
                        tc::wgmma_commit();
                        // keep this stage's MMAs in flight; the previous stage's are complete -> release it
                        tc::wgmma_wait<1>();
                        if (pending >= 0) {
                            __syncwarp();
                            if (lane == 0) tc::mbar_arrive(&empty_bar[pending]);
                        }
                        pending = s;
                    }
                    tc::wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) tc::mbar_arrive(&empty_bar[pending]);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int i = 0; i < 16; ++i)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const float v0 = acc[h][4 * i + e], v1 = acc[h][4 * i + 2 + e];
                                csq[2 * i + e] = fmaf(v1, v1, fmaf(v0, v0, csq[2 * i + e]));
                            }
                }
                // sum over the 16 rows of this warp held by lanes with equal lane%4; fp64 from here on
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    double v = (double)csq[j];
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    v += __shfl_xor_sync(0xffffffffu, v, 8);
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                    if (lane < 4) red_s[q][8 * (j >> 1) + 2 * lane + (j & 1)] = v;
                }
            }
            // every role advanced by the same amount
            for (int ib = 0; ib < nb; ++ib) stage_it += (ib + 1) * (PBM / tc::kTcK);
            __syncthreads();
            if (tid < PBN) {
                const int c = tid;
                const double colsq = ((red_s[0][c] + red_s[1][c]) + red_s[2][c]) + red_s[3][c];
                double val = 0.0;
                candidate_epilogue(P, G, g, mu_s[0][c] + mu_s[1][c], colsq, c0 + c, base_s[c], prod_s[c], &val);
                if (P.sel_cta && g == P.n_gps - 1)
                    runsel_update<1>(sel_s, P.sel_k, tid, val, c0 + c + P.index_base, c0 + c < P.m);
            }
            tc::fence_proxy_async_smem();
            __syncthreads();
        }
    }
    if (P.sel_cta && tid < PBN) runsel_store(sel_s, P.sel_cta + blockIdx.x, tid);
}

// L^-1 (fp64, row-major) -> tf32 (hi, lo) operand images [ib][kt][hi|lo][16 KiB] (lower k-tiles only)
__global__ void __launch_bounds__(256) pretile_linv_tc_kernel(const double* __restrict__ W, int np,
                                                              uint8_t* __restrict__ out) {
    const int kt = blockIdx.x, ib = blockIdx.y;
    if (kt >= (ib + 1) * (PBM / tc::kTcK)) return;
    uint8_t* img = out + ((size_t)ib * (np / tc::kTcK) + kt) * (2 * tc::kTcImgBytes);
    for (int idx = threadIdx.x; idx < PBM * tc::kTcK; idx += 256) {
        const int r = idx / tc::kTcK, k = idx % tc::kTcK;
        const double w = W[(size_t)(ib * PBM + r) * np + kt * tc::kTcK + k];
        const float hi = tc::to_tf32((float)w);
        const float lo = tc::to_tf32((float)(w - (double)hi));
        const int off = tc::tc_img_offset(r, k);
        *reinterpret_cast<float*>(img + off) = hi;
        *reinterpret_cast<float*>(img + tc::kTcImgBytes + off) = lo;
    }
}

// =======================================================================================
// Small-batch path (m <= a few hundred candidates: the single-row / finite-difference-stencil
// calls L-BFGS-B makes, R/bayes_opt/acquisition.py:366).  The tiled kernel would run one
// 128-wide tile on one SM; here the triangular product V = Linv K*^T for up to 32 candidates is
// spread over the whole GPU as fixed-size work units (64 rows x <=512 k), with fixed-order
// partial sums (deterministic).  Three launches per pass of 32 candidates and per GP:
//   small_kstar_kernel  K*[k][c] (+ per-block partials of K* alpha_)
//   small_trsv_kernel   partial V for each (row-block, k-chunk) unit
//   small_finish_kernel sum units, square, reduce rows, epilogue (all GPs)
// =======================================================================================
constexpr int SMC = 32;      // candidates per pass
constexpr int SROWS = 64;    // rows per unit
constexpr int SKCH = 512;    // k per unit
constexpr int SKT = 32;      // k sub-tile staged in smem
constexpr int SWSTR = SKT + 2;

struct SmallGp {
    const double* W;        // [np][np] Linv row-major
    double* ksm;            // [np][SMC]
    double* partial;        // [nunits][SROWS][SMC]
    double* mu_part;        // [np/128][SMC]
    double* colsq_rb;       // [np/SROWS][SMC] per pass: sum over the rows of a row block of V^2
    const int2* unit_tab;   // [nunits] (row-block, k-chunk)
    const int2* rb_tab;     // [np/SROWS] (first unit, number of units)
    // gradient calls only (b200bo_acq_value_grad), else unset: v = L^-1 k*, u = L^-T v and the work units of the
    // upper-triangular product against linvT (row block i covers k in [64 i, np))
    double* vsum;           // [np][SMC] per pass
    double* usum;           // [np][SMC] per pass
    double* partial_u;      // [nunits_u][SROWS][SMC]
    double* gpart;          // [np/128][2][d][SMC] per pass: partials of sum_n {alpha_n, u_n} c h(r_n) (xs_j - Xs_nj)
    const int2* unit_tab_u; // [nunits_u] (row-block, k-chunk counted from the block's first row)
    const int2* rb_tab_u;   // [np/SROWS]
};

// One launch group covers up to SMAXP passes (blockIdx.y / blockIdx.x of the finish kernel = pass): the
// passes of a batch run concurrently (an L-BFGS-B round of all seeds + their stencils is ~170 rows = 6
// passes: 3 launches instead of 18, and six times as many CTAs in flight).
constexpr int SMAXP = 8;

struct SmallParams {
    PredictParams P;
    SmallGp sg[B200BO_MAX_GPS];
    long long c0;  // first candidate of pass 0 of this launch group
    long long m_end;  // one past the last candidate of the batch
    int nunits[B200BO_MAX_GPS];  // work units per pass (stride of `partial` between passes)
    int nunits_u[B200BO_MAX_GPS];  // gradient calls: work units per pass of the product with linvT
    double* grad_out;  // gradient calls: [m][d]
};

__device__ __forceinline__ long long small_pass_c0(const SmallParams& S, int pass) { return S.c0 + (long long)pass * SMC; }
__device__ __forceinline__ int small_pass_mc(const SmallParams& S, int pass) {
    const long long left = S.m_end - small_pass_c0(S, pass);
    return (int)(left < SMC ? (left < 0 ? 0 : left) : SMC);
}

// K*[k][c] for one block of 128 training rows and one pass of 32 candidates (blockIdx.y = pass): thread =
// (candidate c, group of 16 rows); the training row is a warp-wide broadcast load, K* rows are written as
// coalesced 256-byte segments; per-candidate partial of K* alpha_ over the block in a fixed order.
__global__ void __launch_bounds__(256)
small_kstar_kernel(const SmallParams S, int g) {
    const GpDev& G = S.P.gp[g];
    const SmallGp& Q = S.sg[g];
    __shared__ double xc_s[SMC][B200BO_MAX_DIM + 1];
    __shared__ double wsum[8][SMC];
    const int tid = threadIdx.x, d = S.P.d;
    const int pass = blockIdx.y, mc = small_pass_mc(S, pass);
    const long long pc0 = small_pass_c0(S, pass);
    double* ksm = Q.ksm + (size_t)pass * G.np * SMC;
    double* mu_part = Q.mu_part + (size_t)pass * (G.np / 128) * SMC;
    for (int idx = tid; idx < SMC * d; idx += 256) {
        const int c = idx / d, j = idx - c * d;
        double v = 0.0;
        if (c < mc) v = scale_input(candidate_coord(S.P, pc0 + c, j), G.xform, G.ls, j);
        xc_s[c][j] = v;
    }
    __syncthreads();
    const int c = tid & 31, rg = tid >> 5;
    double mu_acc = 0.0;
    for (int q = 0; q < 16; ++q) {
        const int n = blockIdx.x * 128 + rg * 16 + q;
        double kv = 0.0;
        if (c < mc && n < G.n) {
            const double* xr = G.Xs + (size_t)n * d;
            double r2 = 0.0;
            for (int j = 0; j < d; ++j) {
                const double df = xc_s[c][j] - xr[j];
                r2 = fma(df, df, r2);
            }
            kv = G.constv * cov_from_r2(r2, G.family, G.nu);
        }
        ksm[(size_t)n * SMC + c] = kv;
        mu_acc = fma(G.alphav[n], kv, mu_acc);
    }
    wsum[rg][c] = mu_acc;
    __syncthreads();
    if (tid < SMC) {
        double t = 0.0;
#pragma unroll
        for (int r = 0; r < 8; ++r) t += wsum[r][tid];
        mu_part[(size_t)blockIdx.x * SMC + tid] = t;
    }
}

// Partial V for one work unit (64 rows x <= 512 k) and a GROUP of up to STPG passes (blockIdx.y = group): the W tile
// is staged once per k sub-tile and used for every pass of the group.  (One CTA per pass re-read L^-1 six times per
// round; all eight passes in one CTA needed 178 registers and 83 KB -> one CTA per SM, half the throughput.  Groups
// of four: ~100 registers, 49 KB -> two to three resident CTAs per SM.)
constexpr int STPG = 4;
constexpr int kSmallTrsvSmemBytes = (SROWS * SWSTR + STPG * SKT * SMC) * 8;  // 50176
// UPPER (gradient calls): the same product against linvT = L^-T, u = L^-T v: the unit's k range starts at its row
// block (k in [r0 + 512 j, min(.. + 512, np))), the right-hand side is vsum and the partials go to partial_u.
template <bool UPPER>
__global__ void __launch_bounds__(256, 2)
small_trsv_kernel(const SmallParams S, int g, int npass) {
    const GpDev& G = S.P.gp[g];
    const SmallGp& Q = S.sg[g];
    extern __shared__ __align__(16) double strsv_smem[];
    double* Wt = strsv_smem;                  // [SROWS][SWSTR]
    double* Kt = strsv_smem + SROWS * SWSTR;  // [STPG][SKT][SMC]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int p0 = blockIdx.y * STPG, pn = min(STPG, npass - p0);
    const int2 u = UPPER ? Q.unit_tab_u[blockIdx.x] : Q.unit_tab[blockIdx.x];
    const int r0 = u.x * SROWS;
    const int np = G.np;
    const int kbeg = UPPER ? r0 + u.y * SKCH : u.y * SKCH;
    const int kend = UPPER ? min(kbeg + SKCH, np) : min(kbeg + SKCH, r0 + SROWS);
    double acc[STPG][8];
#pragma unroll
    for (int p = 0; p < STPG; ++p)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[p][q] = 0.0;
    for (int k0 = kbeg; k0 < kend; k0 += SKT) {
        for (int idx = tid; idx < SROWS * SKT; idx += 256) {
            const int r = idx / SKT, kk = idx % SKT;
            Wt[r * SWSTR + kk] = (UPPER ? G.linvT : Q.W)[(size_t)(r0 + r) * np + k0 + kk];
        }
        for (int p = 0; p < pn; ++p) {
            const double* ksm = (UPPER ? Q.vsum : Q.ksm) + (size_t)(p0 + p) * np * SMC + (size_t)k0 * SMC;
            for (int idx = tid; idx < SKT * SMC; idx += 256) Kt[p * SKT * SMC + idx] = ksm[idx];
        }
        __syncthreads();
#pragma unroll 2
        for (int kk = 0; kk < SKT; kk += 2) {
            double2 w[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) w[q] = *reinterpret_cast<const double2*>(&Wt[(warp * 8 + q) * SWSTR + kk]);
#pragma unroll
            for (int p = 0; p < STPG; ++p) {
                if (p < pn) {
                    const double k0v = Kt[p * SKT * SMC + kk * SMC + lane], k1v = Kt[p * SKT * SMC + (kk + 1) * SMC + lane];
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        acc[p][q] = fma(w[q].x, k0v, acc[p][q]);
                        acc[p][q] = fma(w[q].y, k1v, acc[p][q]);
                    }
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int p = 0; p < STPG; ++p) {
        if (p < pn) {
            double* out = (UPPER ? Q.partial_u : Q.partial) +
                          ((size_t)(p0 + p) * (UPPER ? S.nunits_u[g] : S.nunits[g]) + blockIdx.x) * SROWS * SMC;
#pragma unroll
            for (int q = 0; q < 8; ++q) out[(warp * 8 + q) * SMC + lane] = acc[p][q];
        }
    }
}

// Per (row block of 64 rows, pass): sum the k-chunk partials of every row in a fixed order, square, and reduce the
// 64 rows -> colsq_rb[pass][row block][candidate].  grid (np / 64, npass).
// MODE (gradient calls): 1 also writes the summed v[n][c] to vsum (the same sums, so colsq is unchanged); 2 sums the
// partials of the product with linvT in index order into usum and forms no squares.
template <int MODE>
__global__ void __launch_bounds__(256)
small_reduce_kernel(const SmallParams S, int g) {
    const GpDev& G = S.P.gp[g];
    const SmallGp& Q = S.sg[g];
    __shared__ double red[8][SMC];
    const int tid = threadIdx.x, c = tid & 31, rg = tid >> 5;
    const int pass = blockIdx.y;
    const int2 rb = MODE == 2 ? Q.rb_tab_u[blockIdx.x] : Q.rb_tab[blockIdx.x];
    const double* partial = MODE == 2 ? Q.partial_u + (size_t)pass * S.nunits_u[g] * SROWS * SMC
                                      : Q.partial + (size_t)pass * S.nunits[g] * SROWS * SMC;
    double s = 0.0;
    for (int q = 0; q < 8; ++q) {
        const int r = rg * 8 + q;
        double v = 0.0;
        for (int j = 0; j < rb.y; ++j) v += partial[((size_t)(rb.x + j) * SROWS + r) * SMC + c];
        if (MODE != 0)
            (MODE == 2 ? Q.usum : Q.vsum)[((size_t)pass * G.np + blockIdx.x * SROWS + r) * SMC + c] = v;
        s = fma(v, v, s);
    }
    if (MODE == 2) return;
    red[rg][c] = s;
    __syncthreads();
    if (tid < SMC) {
        double t = 0.0;
#pragma unroll
        for (int r = 0; r < 8; ++r) t += red[r][tid];
        Q.colsq_rb[((size_t)pass * (G.np / SROWS) + blockIdx.x) * SMC + tid] = t;
    }
}

// Per pass: the row-block and K* alpha_ partials of every GP summed in index order into colsq_s / mu_s.  256 threads
// = 32 candidates x 8 slices of the partial lists (fixed-order two-level sum).
// COLSQ = false (B200BO_ACQ_MEAN): the K* alpha_ sums only - no triangular product ran.
template <bool COLSQ = true>
__device__ __forceinline__ void small_finish_sums(const SmallParams& S, int pass, double (*red)[SMC],
                                                  double (*colsq_s)[SMC], double (*mu_s)[SMC]) {
    const int tid = threadIdx.x, c = tid & 31, sl = tid >> 5;
    for (int g = 0; g < S.P.n_gps; ++g) {
        const GpDev& G = S.P.gp[g];
        const SmallGp& Q = S.sg[g];
        const int nrb = G.np / SROWS, nb = G.np / 128;
        const double* mu_part = Q.mu_part + (size_t)pass * nb * SMC;
        // slice sl sums a contiguous range of the lists; the 8 slice sums are then added in order
        double s = 0.0;
        if constexpr (COLSQ) {
            const double* crb = Q.colsq_rb + (size_t)pass * nrb * SMC;
            for (int b = sl * ((nrb + 7) / 8); b < min(nrb, (sl + 1) * ((nrb + 7) / 8)); ++b)
                s += crb[(size_t)b * SMC + c];
            red[sl][c] = s;
            __syncthreads();
            if (sl == 0) {
                double t = 0.0;
#pragma unroll
                for (int r = 0; r < 8; ++r) t += red[r][c];
                colsq_s[g][c] = t;
            }
            __syncthreads();
        }
        s = 0.0;
        for (int b = sl * ((nb + 7) / 8); b < min(nb, (sl + 1) * ((nb + 7) / 8)); ++b) s += mu_part[(size_t)b * SMC + c];
        red[sl][c] = s;
        __syncthreads();
        if (sl == 0) {
            double t = 0.0;
#pragma unroll
            for (int r = 0; r < 8; ++r) t += red[r][c];
            mu_s[g][c] = t;
        }
        __syncthreads();
    }
}

// Per pass (blockIdx.x): the sums above, then the per-candidate epilogue of every GP (NEI: the NEI / LogNEI kinds;
// CNEI: the CNEI / LogCNEI kinds, each GP with its own K* column and the per-sample carry in shared memory).
template <bool NEI, bool CNEI = false>
__global__ void __launch_bounds__(256)
small_finish_kernel(const SmallParams S) {
    __shared__ double red[8][SMC];
    __shared__ double colsq_s[B200BO_MAX_GPS][SMC];
    __shared__ double mu_s[B200BO_MAX_GPS][SMC];
    __shared__ double carry_s[CNEI ? B200BO_MAX_PATHS : 1][SMC];
    const int tid = threadIdx.x, c = tid & 31, sl = tid >> 5;
    const int pass = blockIdx.x, mc = small_pass_mc(S, pass);
    const long long pc0 = small_pass_c0(S, pass);
    small_finish_sums(S, pass, red, colsq_s, mu_s);
    if (sl == 0 && c < mc) {
        double base_neg = 0.0, prod = 1.0;
        const double* kcol = S.sg[0].ksm + (size_t)pass * S.P.gp[0].np * SMC + c;  // gps[0]'s K* column (NEI)
        for (int g = 0; g < S.P.n_gps; ++g) {
            if constexpr (CNEI)
                kcol = S.sg[g].ksm + (size_t)pass * S.P.gp[g].np * SMC + c;
            candidate_epilogue<NEI, false, CNEI>(S.P, S.P.gp[g], g, mu_s[g][c], colsq_s[g][c], pc0 + c, base_neg,
                                                 prod, nullptr, kcol, SMC, nullptr, CNEI ? &carry_s[0][c] : nullptr);
        }
    }
}

// ---- input gradient of the closure value (b200bo_acq_value_grad, DESIGN.md 4.10) ------------------------------
// With xs = transform(x)/ls, k*_n = c k(|xs - Xs_n|), v = L^-1 k*, u = L^-T v = K^-1 k* (normalised units):
//   d k*_n / d x_j = -c h(r_n) (xs_j - Xs_nj) / ls_j          (h: cov_dh_from_r2)
//   d mu / d x_j   = sum_n alpha_n d k*_n / d x_j,    d var / d x_j = -2 sum_n u_n d k*_n / d x_j
// small_grad_kernel: per (block of 128 training rows, pass) the partial sums
//   gpart[0][j][c] = sum_n alpha_n c h(r_n) (xs_j - Xs_nj),   gpart[1][j][c] = the same with u_n,
// by direct differences, rows in index order.  Sub-chunks of 32 rows: first thread = (candidate, 4 rows) forms the two
// coefficients of each row, then thread = (candidate, dimensions j = jg, jg + 8, ..) adds the 32 rows in order.
// NEI (gps[0] of an NEI / LogNEI call): blockIdx.z = fantasy s, the first list takes a_s = column s of A instead of
// alpha_, and gpart holds S + 1 lists per block: [b][s][j][c] for s < S, then the u list (written by s = 0).
// CNEI (every GP of a CNEI / LogCNEI call, with NEI): the same lists from GP g's own A_g (PredictParams::fant_a_gp).
// MEAN (B200BO_ACQ_MEAN, without NEI): the alpha_ list only; u = L^-T v was not formed and its slots stay unwritten.
constexpr int SGR = 32;  // rows per sub-chunk
template <bool NEI, bool CNEI = false, bool MEAN = false>
__global__ void __launch_bounds__(256)
small_grad_kernel(const SmallParams S, int g) {
    const GpDev& G = S.P.gp[g];
    const SmallGp& Q = S.sg[g];
    __shared__ double xc_s[SMC][B200BO_MAX_DIM + 1];
    __shared__ double coef[2][SGR][SMC];
    const int tid = threadIdx.x, d = S.P.d;
    const int pass = blockIdx.y, mc = small_pass_mc(S, pass);
    const long long pc0 = small_pass_c0(S, pass);
    for (int idx = tid; idx < SMC * d; idx += 256) {
        const int c = idx / d, j = idx - c * d;
        double v = 0.0;
        if (c < mc) v = scale_input(S.P.Xc[(pc0 + c) * d + j], G.xform, G.ls, j);
        xc_s[c][j] = v;
    }
    __syncthreads();
    const int c = tid & 31, rg = tid >> 5;
    constexpr int JT = B200BO_MAX_DIM / 8;
    double sa[JT], su[JT];
#pragma unroll
    for (int t = 0; t < JT; ++t) sa[t] = su[t] = 0.0;
    const double* usum = Q.usum + (size_t)pass * G.np * SMC;
    for (int sub = 0; sub < 128 / SGR; ++sub) {
        const int n0 = blockIdx.x * 128 + sub * SGR;
        for (int q = 0; q < SGR / 8; ++q) {
            const int rl = rg * (SGR / 8) + q, n = n0 + rl;
            double ca = 0.0, cu = 0.0;
            if (c < mc && n < G.n) {
                const double* xr = G.Xs + (size_t)n * d;
                double r2 = 0.0;
                for (int j = 0; j < d; ++j) {
                    const double df = xc_s[c][j] - xr[j];
                    r2 = fma(df, df, r2);
                }
                const double ch = G.constv * cov_dh_from_r2(r2, G.family, G.nu);
                if constexpr (CNEI)
                    ca = S.P.fant_a_gp[g][(size_t)n * S.P.n_ystar + blockIdx.z] * ch;
                else if constexpr (NEI)
                    ca = S.P.fant_a[(size_t)n * S.P.n_ystar + blockIdx.z] * ch;
                else
                    ca = G.alphav[n] * ch;
                if constexpr (!MEAN) cu = usum[(size_t)n * SMC + c] * ch;
            }
            coef[0][rl][c] = ca;
            coef[1][rl][c] = cu;
        }
        __syncthreads();
        for (int rl = 0; rl < SGR; ++rl) {
            const double* xr = G.Xs + (size_t)(n0 + rl) * d;
            const double ca = coef[0][rl][c], cu = coef[1][rl][c];
#pragma unroll
            for (int t = 0; t < JT; ++t) {
                const int j = rg + 8 * t;
                if (j < d) {
                    const double df = xc_s[c][j] - xr[j];
                    sa[t] = fma(ca, df, sa[t]);
                    su[t] = fma(cu, df, su[t]);
                }
            }
        }
        __syncthreads();
    }
    if constexpr (NEI) {
        const int nl = S.P.n_ystar + 1;  // lists per block
        double* out = Q.gpart + ((size_t)pass * (G.np / 128) + blockIdx.x) * nl * d * SMC;
#pragma unroll
        for (int t = 0; t < JT; ++t) {
            const int j = rg + 8 * t;
            if (j < d) {
                out[((size_t)blockIdx.z * d + j) * SMC + c] = sa[t];
                if (blockIdx.z == 0) out[((size_t)(nl - 1) * d + j) * SMC + c] = su[t];
            }
        }
    } else {
        double* out = Q.gpart + ((size_t)pass * (G.np / 128) + blockIdx.x) * 2 * d * SMC;
#pragma unroll
        for (int t = 0; t < JT; ++t) {
            const int j = rg + 8 * t;
            if (j < d) {
                out[(size_t)j * SMC + c] = sa[t];
                if constexpr (!MEAN) out[(size_t)(d + j) * SMC + c] = su[t];
            }
        }
    }
}

// Gradient finish, per pass (blockIdx.x): per candidate and GP one candidate_epilogue<NEI, true>, which forms the value
// exactly as small_finish_kernel does (same sums, same epilogue) and gives the GP's term and its coefficients; from
// them the weights of the two partial-sum lists,
//   grad_j = sum_g ( wa_g sum_b gpart_g[b][0][j] + wu_g sum_b gpart_g[b][1][j] ) / ls_gj      (blocks b in index order)
//   wa_g = -w_g cm_g s_y,   wu_g = w_g cs_g s_y / sqrt(var_g)   (0 where var_g <= 0: d sd := 0)
//   w_0 = -prod_i p_i,   w_g = -base prod_{i != g} p_i           (product rule over the GPs, g order)
//   LogEI / LogPoI: w_g = -1 (the value is -(alpha + sum_g log p_g), a plain sum)
// A rounded dimension has gradient 0; a NaN value gives a NaN row.
// NEI: gps[0] is the noiseless handle of an NEI / LogNEI call: its mean coefficient is one per fantasy (nei_term,
// held in wn_s) against the S lists of gpart, its sd coefficient multiplies the u list as usual.
template <bool NEI>
__global__ void __launch_bounds__(256)
small_finish_grad_kernel(const SmallParams S) {
    __shared__ double red[8][SMC];
    __shared__ double colsq_s[B200BO_MAX_GPS][SMC];
    __shared__ double mu_s[B200BO_MAX_GPS][SMC];
    __shared__ double wa_s[B200BO_MAX_GPS][SMC], wu_s[B200BO_MAX_GPS][SMC];
    __shared__ double val_s[SMC];
    __shared__ double wn_s[NEI ? B200BO_MAX_PATHS : 1][SMC];
    const int tid = threadIdx.x, c = tid & 31, sl = tid >> 5;
    const int pass = blockIdx.x, mc = small_pass_mc(S, pass), d = S.P.d, ng = S.P.n_gps;
    const long long pc0 = small_pass_c0(S, pass);
    small_finish_sums(S, pass, red, colsq_s, mu_s);
    if (sl == 0 && c < mc) {
        double base_neg = 0.0, prod = 1.0, val = 0.0;
        const double* kcol = S.sg[0].ksm + (size_t)pass * S.P.gp[0].np * SMC + c;
        // term_g, then w_g from the terms of the other GPs; wa_s / wu_s hold cm / cs until the second loop
        double term[B200BO_MAX_GPS];
#pragma unroll
        for (int g = 0; g < B200BO_MAX_GPS; ++g) {
            term[g] = 1.0;
            if (g < ng) {
                const GpDev& G = S.P.gp[g];
                EpilogueGrad e;
                e.cms = &wn_s[0][c];
                candidate_epilogue<NEI, true>(S.P, G, g, mu_s[g][c], colsq_s[g][c], pc0 + c, base_neg, prod, &val,
                                              kcol, SMC, &e);
                const double var = fmax(G.prior - colsq_s[g][c], 0.0);
                term[g] = e.term;
                wa_s[g][c] = -e.cm * G.y_std;
                wu_s[g][c] = var > 0.0 ? e.cs * G.y_std / sqrt(var) : 0.0;
            }
        }
        val_s[c] = val;
        // the value is -sum_g term_g: w_g = -1, no product rule
        const bool logk = acq_constraints_in_log<NEI>(S.P.acq_kind);
#pragma unroll
        for (int g = 0; g < B200BO_MAX_GPS; ++g) {
            if (g < ng) {
                double w = -1.0;
#pragma unroll
                for (int i = 0; i < B200BO_MAX_GPS; ++i)
                    if (i < ng && i != g && !logk) w *= term[i];
                wa_s[g][c] = wa_s[g][c] == 0.0 ? 0.0 : w * wa_s[g][c];
                wu_s[g][c] = wu_s[g][c] == 0.0 ? 0.0 : w * wu_s[g][c];
                if (NEI && g == 0)
                    for (int s = 0; s < S.P.n_ystar; ++s) wn_s[s][c] = wn_s[s][c] == 0.0 ? 0.0 : w * wn_s[s][c];
            }
        }
    }
    __syncthreads();
    for (int idx = tid; idx < SMC * d; idx += 256) {
        const int cc = idx & 31, j = idx >> 5;
        if (cc >= mc) continue;
        double gr = 0.0;
        for (int g = 0; g < ng; ++g) {
            const GpDev& G = S.P.gp[g];
            if (G.xform && xform_rounds(G.xform[j])) continue;
            const int nb = G.np / 128;
            if (NEI && g == 0) {  // sum_s wn_s (-y_std) sum_b list s, then the u list
                const int nl = S.P.n_ystar + 1;
                const double* gp = S.sg[0].gpart + (size_t)pass * nb * nl * d * SMC;
                double an = 0.0, u = 0.0;
                for (int s = 0; s < nl - 1; ++s) {
                    double a = 0.0;
                    for (int b = 0; b < nb; ++b) a += gp[(((size_t)b * nl + s) * d + j) * SMC + cc];
                    const double wn = wn_s[s][cc];
                    an += wn == 0.0 ? 0.0 : -G.y_std * wn * a;
                }
                for (int b = 0; b < nb; ++b) u += gp[(((size_t)b * nl + nl - 1) * d + j) * SMC + cc];
                const double wu = wu_s[0][cc];
                gr += (an + (wu == 0.0 ? 0.0 : wu * u)) / G.ls[j];
                continue;
            }
            const double* gp = S.sg[g].gpart + (size_t)pass * nb * 2 * d * SMC;
            double a = 0.0, u = 0.0;
            for (int b = 0; b < nb; ++b) {
                a += gp[((size_t)b * 2 * d + j) * SMC + cc];
                u += gp[((size_t)b * 2 * d + d + j) * SMC + cc];
            }
            const double wa = wa_s[g][cc], wu = wu_s[g][cc];
            gr += ((wa == 0.0 ? 0.0 : wa * a) + (wu == 0.0 ? 0.0 : wu * u)) / G.ls[j];
        }
        S.grad_out[(pc0 + cc) * d + j] = isnan(val_s[cc]) ? CUDART_NAN : gr;
    }
}

// B200BO_ACQ_MEAN on the small-batch path, per pass (blockIdx.x): the K* alpha_ sums of small_finish_sums (the order
// b200bo_gp_predict's small path adds them in), mu_g = y_std mu_n + y_mean as candidate_epilogue forms it, then the
// merit.  GRAD (b200bo_acq_value_grad): d acq_neg = sum_g w_g d mu_g, with d mu_g / d x_j = -y_std_g (sum_b gpart_g
// [b][0][j]) / ls_gj (small_grad_kernel<false, false, true>) and
//   w_0 = -1 where viol = 0 (the boundary included), else w_0 = 0 and w_g = -T below lb_g, +T above ub_g, 0 within.
// A rounded dimension has gradient 0; a NaN value gives a NaN row.
template <bool GRAD>
__global__ void __launch_bounds__(256)
small_finish_mean_kernel(const SmallParams S) {
    __shared__ double red[8][SMC];
    __shared__ double mu_s[B200BO_MAX_GPS][SMC];
    __shared__ double w_s[B200BO_MAX_GPS][SMC];
    __shared__ double val_s[SMC];
    const int tid = threadIdx.x, c = tid & 31, sl = tid >> 5;
    const int pass = blockIdx.x, mc = small_pass_mc(S, pass), ng = S.P.n_gps;
    const long long pc0 = small_pass_c0(S, pass);
    small_finish_sums<false>(S, pass, red, nullptr, mu_s);
    if (sl == 0 && c < mc) {
        const long long gi = pc0 + c;
        double mu0 = 0.0, viol = 0.0;
        for (int g = 0; g < ng; ++g) {
            const GpDev& G = S.P.gp[g];
            const double mean = G.y_std * mu_s[g][c] + G.y_mean;
            mu_s[g][c] = mean;
            if (g == 0) {
                mu0 = mean;
                if (S.P.mu_out) S.P.mu_out[gi] = mean;
            } else {
                viol = __dadd_rn(viol, mean_viol(G, mean));
            }
        }
        const double val = mean_merit_neg(mu0, viol, S.P.mean_T);
        if (S.P.acq_out) S.P.acq_out[gi] = val;
        if constexpr (GRAD) {
            val_s[c] = val;
            const bool feasible = viol == 0.0;
            for (int g = 0; g < ng; ++g) {
                const GpDev& G = S.P.gp[g];
                const double mean = mu_s[g][c];
                double w = 0.0;
                if (g == 0)
                    w = feasible ? -1.0 : 0.0;
                else if (!feasible && G.lb != -CUDART_INF && mean < G.lb)
                    w = -S.P.mean_T;
                else if (!feasible && G.ub != CUDART_INF && mean > G.ub)
                    w = S.P.mean_T;
                w_s[g][c] = w;
            }
        }
    }
    if constexpr (GRAD) {
        __syncthreads();
        const int d = S.P.d;
        for (int idx = tid; idx < SMC * d; idx += 256) {
            const int cc = idx & 31, j = idx >> 5;
            if (cc >= mc) continue;
            double gr = 0.0;
            for (int g = 0; g < ng; ++g) {
                const GpDev& G = S.P.gp[g];
                const double w = w_s[g][cc];
                if (w == 0.0 || (G.xform && xform_rounds(G.xform[j]))) continue;
                const int nb = G.np / 128;
                const double* gp = S.sg[g].gpart + (size_t)pass * nb * 2 * d * SMC;
                double a = 0.0;
                for (int b = 0; b < nb; ++b) a += gp[((size_t)b * 2 * d + j) * SMC + cc];
                gr += w * (-G.y_std * a) / G.ls[j];
            }
            S.grad_out[(pc0 + cc) * d + j] = isnan(val_s[cc]) ? CUDART_NAN : gr;
        }
    }
}

// CNEI / LogCNEI gradient coefficients of one candidate (b200bo_acq_value_grad, DESIGN.md 4.15), out of line: the
// value as cnei_term forms it (same means, same products in j order, same sums in s order), and
//   wn[(g * B200BO_MAX_PATHS + s) * SMC] = the coefficient of d mu_gs,   wsig[g] = that of d sigma0_g   (data units).
// CNEI = -(1/S) sum_s T_s, T_s = EI_s prod_j P_js: by the product rule per sample, without dividing by a P,
//   d T_s = prod_j P_js dEI_s + EI_s sum_j (prod_{k != j} P_ks) dP_js     (prefix and suffix products over j);
// LogCNEI = -logmeanexp_s l_s, l_s = LogEI_s + sum_j log P_js: d = -sum_s p_s d l_s, p_s = exp(l_s - M) / sum exp(l - M).
// EI_s / LogEI_s give Phi / phi (LogEI's r / sd, q / sd), the factors EI's (log_cfactor's) coefficients; sd = 0 makes a
// GP's coefficients 0.  kcol[g]: GP g's K* column (stride SMC).
__device__ __noinline__ double cnei_grad_term(const PredictParams& P, const double* const* kcol, const double* sdv,
                                              double* wn, double* wsig) {
    const int S = P.n_ystar, ng = P.n_gps;
    const bool lg = P.acq_kind == B200BO_ACQ_LOGCNEI;
    const double* best = P.fant_a + (size_t)P.gp[0].np * S;
    double T[B200BO_MAX_PATHS], cm0[B200BO_MAX_PATHS], cs0[B200BO_MAX_PATHS];
    double pf[B200BO_MAX_GPS][B200BO_MAX_PATHS], pcm[B200BO_MAX_GPS][B200BO_MAX_PATHS],
        pcs[B200BO_MAX_GPS][B200BO_MAX_PATHS];
    for (int g = 0; g < ng; ++g) {
        const GpDev& G = P.gp[g];
        const double* A = P.fant_a_gp[g];
        const double sd = sdv[g];
        wsig[g] = 0.0;
        for (int s = 0; s < S; ++s) {
            double t = 0.0;
            for (int i = 0; i < G.n; ++i) t = fma(A[(size_t)i * S + s], kcol[g][(size_t)i * SMC], t);
            const double mean = G.y_std * t + G.y_mean;
            if (g == 0) {
                T[s] = lg ? log_acq_term<true>(B200BO_ACQ_LOGEI, mean - best[s] - P.xi, sd, &cm0[s], &cs0[s])
                          : nei_ei_term<true>(mean - best[s] - P.xi, sd, &cm0[s], &cs0[s]);
                continue;
            }
            double cm = 0.0, cs = 0.0, v;
            if (lg) {
                v = log_cfactor<true>(G.lb, G.ub, mean, sd, &cm, &cs);
            } else {
                v = cnei_factor(G.lb, G.ub, mean, sd);
                if (sd > 0.0) {
                    if (G.lb != -CUDART_INF) {
                        const double z = (G.lb - mean) / sd, pz = norm_pdf(z);
                        cm += pz / sd;
                        cs += pz == 0.0 ? 0.0 : z * pz / sd;
                    }
                    if (G.ub != CUDART_INF) {
                        const double z = (G.ub - mean) / sd, pz = norm_pdf(z);
                        cm -= pz / sd;
                        cs -= pz == 0.0 ? 0.0 : z * pz / sd;
                    }
                }
            }
            pf[g][s] = v;
            pcm[g][s] = cm;
            pcs[g][s] = cs;
        }
    }
    double val;
    if (!lg) {
        double sum = 0.0;
        for (int s = 0; s < S; ++s) {
            double t = T[s];
            for (int g = 1; g < ng; ++g) t = t * pf[g][s];
            sum += t;
        }
        val = -1.0 * (sum / (double)S);
        const double w = -1.0 / (double)S;
        for (int s = 0; s < S; ++s) {
            double suf[B200BO_MAX_GPS + 1];  // suf[g] = prod_{k >= g} P_ks
            suf[ng] = 1.0;
            for (int g = ng - 1; g >= 1; --g) suf[g] = pf[g][s] * suf[g + 1];
            wn[s * SMC] = w * suf[1] * cm0[s];
            wsig[0] += w * suf[1] * cs0[s];
            double pre = T[s];  // EI_s prod_{k < g} P_ks
            for (int g = 1; g < ng; ++g) {
                const double o = w * pre * suf[g + 1];
                wn[(g * B200BO_MAX_PATHS + s) * SMC] = o * pcm[g][s];
                wsig[g] += o * pcs[g][s];
                pre = pre * pf[g][s];
            }
        }
        return val;
    }
    double mx = -CUDART_INF;
    bool nan = false;
    for (int s = 0; s < S; ++s) {
        for (int g = 1; g < ng; ++g) T[s] = T[s] + pf[g][s];
        nan = nan || isnan(T[s]);
        mx = fmax(mx, T[s]);
    }
    for (int g = 0; g < ng; ++g)
        for (int s = 0; s < S; ++s) wn[(g * B200BO_MAX_PATHS + s) * SMC] = 0.0;
    if (nan) return CUDART_NAN;
    if (mx == -CUDART_INF) return CUDART_INF;
    double e = 0.0;
    for (int s = 0; s < S; ++s) e += exp(T[s] - mx);
    for (int s = 0; s < S; ++s) {
        const double w = -exp(T[s] - mx) / e;
        wn[s * SMC] = w * cm0[s];
        wsig[0] += w * cs0[s];
        for (int g = 1; g < ng; ++g) {
            wn[(g * B200BO_MAX_PATHS + s) * SMC] = w * pcm[g][s];
            wsig[g] += w * pcs[g][s];
        }
    }
    return -1.0 * (mx + log(e) - log((double)S));
}

// Gradient finish of CNEI / LogCNEI, per pass (blockIdx.x): per candidate cnei_grad_term, then per dimension
//   grad_j = sum_g ( sum_s wn_gs (-y_std_g) sum_b list_gs[b][j] + wu_g sum_b u_g[b][j] ) / ls_gj,
//   wu_g = wsig_g y_std_g / sqrt(var_g)  (0 where var_g <= 0),
// over the S + 1 lists per block small_grad_kernel<true, true> wrote for every GP.
__global__ void __launch_bounds__(256)
small_finish_grad_cnei_kernel(const SmallParams S) {
    __shared__ double red[8][SMC];
    __shared__ double colsq_s[B200BO_MAX_GPS][SMC];
    __shared__ double mu_s[B200BO_MAX_GPS][SMC];
    __shared__ double wu_s[B200BO_MAX_GPS][SMC];
    __shared__ double val_s[SMC];
    __shared__ double wn_s[B200BO_MAX_GPS * B200BO_MAX_PATHS][SMC];
    const int tid = threadIdx.x, c = tid & 31, sl = tid >> 5;
    const int pass = blockIdx.x, mc = small_pass_mc(S, pass), d = S.P.d, ng = S.P.n_gps, nl = S.P.n_ystar + 1;
    const long long pc0 = small_pass_c0(S, pass);
    small_finish_sums(S, pass, red, colsq_s, mu_s);
    if (sl == 0 && c < mc) {
        const double* kcol[B200BO_MAX_GPS];
        double sdv[B200BO_MAX_GPS], var[B200BO_MAX_GPS], wsig[B200BO_MAX_GPS];
        for (int g = 0; g < ng; ++g) {
            const GpDev& G = S.P.gp[g];
            kcol[g] = S.sg[g].ksm + (size_t)pass * G.np * SMC + c;
            double v = G.prior - colsq_s[g][c];
            if (v < 0.0) {
                v = 0.0;
                if (S.P.clamp_count) atomicAdd(S.P.clamp_count, 1ull);
            }
            var[g] = v;
            sdv[g] = sqrt(v * (G.y_std * G.y_std));
        }
        const double val = cnei_grad_term(S.P, kcol, sdv, &wn_s[0][c], wsig);
        for (int g = 0; g < ng; ++g)
            wu_s[g][c] = var[g] > 0.0 && wsig[g] != 0.0 ? wsig[g] * S.P.gp[g].y_std / sqrt(var[g]) : 0.0;
        val_s[c] = val;
        if (S.P.acq_out) S.P.acq_out[pc0 + c] = val;
    }
    __syncthreads();
    for (int idx = tid; idx < SMC * d; idx += 256) {
        const int cc = idx & 31, j = idx >> 5;
        if (cc >= mc) continue;
        double gr = 0.0;
        for (int g = 0; g < ng; ++g) {
            const GpDev& G = S.P.gp[g];
            if (G.xform && xform_rounds(G.xform[j])) continue;
            const int nb = G.np / 128;
            const double* gp = S.sg[g].gpart + (size_t)pass * nb * nl * d * SMC;
            double an = 0.0, u = 0.0;
            for (int s = 0; s < nl - 1; ++s) {
                const double wn = wn_s[g * B200BO_MAX_PATHS + s][cc];
                if (wn == 0.0) continue;
                double a = 0.0;
                for (int b = 0; b < nb; ++b) a += gp[(((size_t)b * nl + s) * d + j) * SMC + cc];
                an += -G.y_std * wn * a;
            }
            for (int b = 0; b < nb; ++b) u += gp[(((size_t)b * nl + nl - 1) * d + j) * SMC + cc];
            const double wu = wu_s[g][cc];
            gr += (an + (wu == 0.0 ? 0.0 : wu * u)) / G.ls[j];
        }
        S.grad_out[(pc0 + cc) * d + j] = isnan(val_s[cc]) ? CUDART_NAN : gr;
    }
}

// ---------------------------------------------------------------------------------------
// Selection: record 0 = np.argmin(vals) (first NaN wins, ties -> lowest index);
// records 1..k = the k smallest by (value, index) with NaN last (np.argsort order for
// distinct values).  Single CTA of 1024 threads; k+1 fixed-order passes over vals (L2).
// (R/bayes_opt/acquisition.py:313-317)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
select_kernel(const double* __restrict__ vals, long long m, int k, SelRecord* __restrict__ out,
              long long index_base) {
    __shared__ unsigned long long skey[1024];
    __shared__ long long sidx[1024];
    __shared__ unsigned long long prev_key;
    __shared__ long long prev_idx;
    const int tid = threadIdx.x;
    for (int round = 0; round <= k; ++round) {
        const bool argmin_round = (round == 0);
        const bool bounded = (round >= 2);
        const unsigned long long pk = bounded ? prev_key : 0ull;
        const long long pi = bounded ? prev_idx : -1;
        unsigned long long bk = 0xFFFFFFFFFFFFFFFFull;
        long long bi = -1;
        for (long long i = tid; i < m; i += 1024) {
            const double v = vals[i];
            const unsigned long long key = argmin_round ? key_nan_first(v) : key_nan_last(v);
            if (bounded && (key < pk || (key == pk && i <= pi))) continue;
            if (bi < 0 || key < bk) {  // i increases, so ties keep the lowest index
                bk = key;
                bi = i;
            }
        }
        skey[tid] = bk;
        sidx[tid] = bi;
        __syncthreads();
        for (int s = 512; s > 0; s >>= 1) {
            if (tid < s) {
                const unsigned long long ok = skey[tid + s];
                const long long oi = sidx[tid + s];
                const long long mi = sidx[tid];
                const bool take = (oi >= 0) && (mi < 0 || ok < skey[tid] || (ok == skey[tid] && oi < mi));
                if (take) {
                    skey[tid] = ok;
                    sidx[tid] = oi;
                }
            }
            __syncthreads();
        }
        if (tid == 0) {
            const long long w = sidx[0];
            out[round].index = (w >= 0) ? w + index_base : -1;
            out[round].value = (w >= 0) ? vals[w] : CUDART_NAN;
            prev_key = skey[0];
            prev_idx = (w >= 0) ? w : (long long)0x7FFFFFFFFFFFFFFFll;
        }
        __syncthreads();
    }
}

}  // namespace b200bo
