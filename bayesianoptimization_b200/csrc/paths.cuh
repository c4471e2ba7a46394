// paths.cuh - posterior sample paths of a fitted GP (Thompson sampling), evaluated and ranked on the device.
//
// Pathwise conditioning (Wilson et al., ICML 2020, "Efficiently sampling functions from Gaussian process
// posteriors"), in the normalised target units of the fitted state:
//   path_p(x) = s_y * ( sum_l W[l][p] phi_l(xs) + sum_i V[i][p] k(xs, Xs_i) ) + y_mean,   xs = transform(x)/ls
//   phi_l(xs) = sqrt(2c/L) cos(omega_l . xs + b_l)        (random Fourier features of the prior, L of them)
//   V = K^-1 (y_norm - Phi(Xs) W - eps)                   (exact update, solved once per path at creation)
// The reference has no counterpart: its tutorial draws multivariate_normal(mean, cov) from
// predict(return_cov=True) on the host, O(M^3) in the number of candidates.  Here a candidate costs
// O(N d + L d) whatever M is, and q <= B200BO_MAX_PATHS paths share one candidate tile.
//
// Decomposition: a persistent grid of 256-thread CTAs, 128-candidate tiles, two threads per candidate (each
// takes half of every staged chunk).  Training rows (Xs, V) and then features (omega, W, b) stream through
// shared memory in double-buffered cp.async chunks of 64; the q sums live in registers.  The two halves are
// added in a fixed order, so a candidate's value depends on its coordinates only - not on the batch size, its
// position in the batch or the grid size (the finite-difference stencil of the L-BFGS-B refinement relies on
// that).  Output: f (m x q), and/or -f folded into one running selection list per path (select.cuh).
#pragma once
#include "common.cuh"
#include "predict_kernels.cuh"
#include "select.cuh"

namespace b200bo {

constexpr int PT_CHUNK = 64;  // training rows / features per staged chunk
constexpr int PT_NT = 256;
constexpr int PT_R = 4;       // rows per inner step (independent chains for the fp64 pipe)

struct PathsParams {
    const double* Xs;     // [np][d]  transform(X)/ls of the training rows (path-owned copy), zero padded
    const double* V;      // [np][q]  K^-1 r, zero padded
    const double* omega;  // [Lp][d]  spectral draws, zero padded
    const double* bias;   // [Lp]     phases
    const double* W;      // [Lp][q]  feature weights, zero padded
    const double* ls;     // [d]      length scales (replicated when isotropic)
    const int* xform;     // [d] or nullptr
    int n, np, d, q, Lp, sel_k, sel_resume, pad0;
    double constv, feat_scale, y_mean, y_std;
    // candidate source: the fields candidate_coord reads (predict_kernels.cuh)
    const double* Xc;         // [m][d] or nullptr (Philox)
    const double* pbounds;    // Philox: [2][d] = lo_j, hi_j - lo_j
    unsigned long long seed;  // Philox key
    long long index_base;     // global index of this launch's candidate 0
    long long m;
    unsigned long long* clamp_count;  // [1]: non-finite candidate coordinates (slot [0] unused)
    double* out;              // [m][q] ([m] with path_idx) or nullptr
    SelList* sel_cta;         // [q][gridDim.x] per-CTA running selections, or nullptr
    const int* path_idx;      // [m]: row mode (ROWS instantiation) - row i on path path_idx[i] only
    // trust-region source (select.cuh philox_tr_coord), Philox only: [d] centre in the pbounds buffer, or nullptr
    const double* tr_center;
    double tr_p;              // probability that a coordinate other than the forced one is perturbed
};

// coordinate j of candidate gi: host rows, the Philox box, or the trust-region source around tr_center
__device__ __forceinline__ double paths_coord(const PathsParams& P, long long gi, int j) {
    if (!P.Xc && P.tr_center)
        return philox_tr_coord(P.seed, gi + P.index_base, j, P.d, P.pbounds[j], P.pbounds[P.d + j], P.tr_center[j],
                               P.tr_p);
    return candidate_coord(P, gi, j);
}

// dynamic shared memory: 2 stage buffers [64][d + q + 1] | xc [d][128] | red [2][q][128] | SelShared [q]
__host__ __device__ inline size_t paths_smem_bytes(int d, int q, bool sel) {
    return sizeof(double) * ((size_t)2 * PT_CHUNK * (d + q + 1) + (size_t)d * PBN + (size_t)2 * q * PBN) +
           (sel ? sizeof(SelShared) * (size_t)q : 0);
}

// QT: register slots of the q sums (1, 4 or 16).  QT = 1, 4: 2 CTAs per SM (<= 128 registers, no spills).  QT = 16:
// one CTA per SM and 176 registers - at 128 it spilled, and on an H100 (400 W) it took 147 ms instead of 127 ms for
// 16 paths x 2^20 candidates at C3.
// ROWS (with QT = 1): row mode of the batched refinement - candidate i keeps the one sum of path P.path_idx[i] and
// writes out[i].  The stage still holds all q columns of V / W; only the column a candidate reads changes.  Its
// sums take the same operations in the same order as column path_idx[i] of the full evaluation, so the values
// are bit-equal to it.
template <int COV, int QT, bool ROWS = false>
__global__ void __launch_bounds__(PT_NT, QT == 16 ? 1 : 2) paths_eval_kernel(const PathsParams P) {
    static_assert(!ROWS || QT == 1, "row mode keeps one sum per candidate");
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, d = P.d, q = P.q;
    const int qs = ROWS ? 1 : q;  // sums per candidate
    const int c = tid & (PBN - 1), half = tid >> 7;
    const int bufsz = PT_CHUNK * (d + q + 1);
    double* stage = smem;
    double* xc_s = smem + 2 * bufsz;                // [d][PBN]
    double* red = xc_s + (size_t)d * PBN;           // [2][q][PBN]
    SelShared* sel = reinterpret_cast<SelShared*>(red + (size_t)2 * q * PBN);
    if (!ROWS && P.sel_cta) {
        if (tid < PBN)
            for (int p = 0; p < q; ++p)
                runsel_begin(sel[p], P.sel_cta + (size_t)p * gridDim.x + blockIdx.x, P.sel_resume, tid);
        __syncthreads();
    }
    const long long ntiles = (P.m + PBN - 1) / PBN;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long c0 = tile * PBN;
        // candidate coordinates, scaled exactly as scale_x_kernel scales the training rows
        for (int idx = tid; idx < PBN * d; idx += PT_NT) {
            const int cc = idx / d, j = idx - cc * d;
            const long long gi = c0 + cc;
            double v = 0.0;
            if (gi < P.m) v = scale_input(paths_coord(P, gi, j), P.xform, P.ls, j);
            xc_s[j * PBN + cc] = v;
        }
        int pc = 0;  // ROWS: the column of V / W this thread's candidate reads
        if (ROWS && c0 + c < P.m) pc = P.path_idx[c0 + c];
        double ak[QT], af[QT];
#pragma unroll
        for (int p = 0; p < QT; ++p) ak[p] = af[p] = 0.0;
        // pass 0: training rows (Xs, V) -> sum_i V[i][p] k(xs, Xs_i); pass 1: features (omega, W, b)
        for (int pass = 0; pass < 2; ++pass) {
            const double* A = pass ? P.omega : P.Xs;
            const double* B = pass ? P.W : P.V;
            const int nch = (pass ? P.Lp : P.np) / PT_CHUNK;
            auto load = [&](int buf, int ch) {
                double* dst = stage + buf * bufsz;
                const double* a = A + (size_t)ch * PT_CHUNK * d;
                for (int i = tid; i < PT_CHUNK * d / 2; i += PT_NT) cp_async16_cg(dst + 2 * i, a + 2 * i);
                const double* b = B + (size_t)ch * PT_CHUNK * q;
                for (int i = tid; i < PT_CHUNK * q / 2; i += PT_NT)
                    cp_async16_cg(dst + PT_CHUNK * d + 2 * i, b + 2 * i);
                if (pass && tid < PT_CHUNK / 2)
                    cp_async16_cg(dst + PT_CHUNK * (d + q) + 2 * tid, P.bias + (size_t)ch * PT_CHUNK + 2 * tid);
            };
            load(0, 0);
            cp_async_commit();
            for (int ch = 0; ch < nch; ++ch) {
                if (ch + 1 < nch) load((ch + 1) & 1, ch + 1);
                cp_async_commit();
                cp_async_wait<1>();
                __syncthreads();  // chunk ch (and, on the first chunk, xc_s) visible
                const double* a = stage + (ch & 1) * bufsz;
                const double* b = a + PT_CHUNK * d;
                const double* ph = b + PT_CHUNK * q;
                for (int r0 = half * (PT_CHUNK / 2); r0 < (half + 1) * (PT_CHUNK / 2); r0 += PT_R) {
                    double s[PT_R];
#pragma unroll
                    for (int t = 0; t < PT_R; ++t) s[t] = 0.0;
                    for (int j = 0; j < d; ++j) {
                        const double xv = xc_s[j * PBN + c];
#pragma unroll
                        for (int t = 0; t < PT_R; ++t) {
                            const double av = a[(r0 + t) * d + j];
                            if (pass) {
                                s[t] = fma(av, xv, s[t]);
                            } else {
                                const double df = xv - av;
                                s[t] = fma(df, df, s[t]);
                            }
                        }
                    }
#pragma unroll
                    for (int t = 0; t < PT_R; ++t) {
                        const int r = r0 + t;
                        if (pass) {
                            const double phi = cos(s[t] + ph[r]);
#pragma unroll
                            for (int p = 0; p < QT; ++p)
                                if (p < qs) af[p] = fma(b[r * q + pc + p], phi, af[p]);
                        } else {
                            double kv = P.constv * cov_eval<COV>(s[t]);
                            if (ch * PT_CHUNK + r >= P.n) kv = 0.0;
#pragma unroll
                            for (int p = 0; p < QT; ++p)
                                if (p < qs) ak[p] = fma(b[r * q + pc + p], kv, ak[p]);
                        }
                    }
                }
                __syncthreads();  // buffer (ch & 1) free for the prefetch of chunk ch + 2
            }
            cp_async_wait<0>();
        }
        // the two halves of every sum, always added in the same order
        if (half == 1) {
#pragma unroll
            for (int p = 0; p < QT; ++p)
                if (p < qs) {
                    red[p * PBN + c] = ak[p];
                    red[(q + p) * PBN + c] = af[p];
                }
        }
        __syncthreads();
        if (half == 0) {
            const long long gi = c0 + c;
            const bool valid = gi < P.m;
#pragma unroll
            for (int p = 0; p < QT; ++p) {
                if (p < qs) {
                    const double kp = ak[p] + red[p * PBN + c];
                    const double fp = af[p] + red[(q + p) * PBN + c];
                    const double f = P.y_std * fma(P.feat_scale, fp, kp) + P.y_mean;
                    if (P.out && valid) P.out[gi * qs + p] = f;
                    if (!ROWS && P.sel_cta) runsel_update<1>(sel[p], P.sel_k, tid, -f, gi + P.index_base, valid);
                }
            }
        }
        __syncthreads();  // xc_s / red reused by the next tile
    }
    if (!ROWS && P.sel_cta && tid < PBN)
        for (int p = 0; p < q; ++p) runsel_store(sel[p], P.sel_cta + (size_t)p * gridDim.x + blockIdx.x, tid);
}

// ---------------------------------------------------------------------------------------
// Input gradient of a path in row mode (b200bo_paths_grad_rows): one CTA per row i, path p = path_idx[i],
//   d path_p / d x_j = s_y ( -feat_scale sum_l W[l][p] sin(omega_l . xs + b_l) omega_lj
//                            - sum_n V[n][p] c h(r_n) (xs_j - Xs_nj) ) / ls_j          (h: cov_dh_eval)
// and 0 for a rounded dimension.  Items (training rows, then features) go through in chunks of 256: each thread
// forms the scalar coefficient of one item, then thread (j, slice s) adds its contiguous share of the chunk's items
// in index order; the slices are added in s order at the end.  No atomics: a row's gradient depends on its
// coordinates and its path only.  The value of the same row comes from the ROWS paths_eval_kernel.
// ---------------------------------------------------------------------------------------
constexpr int PG_NT = 256;

template <int COV>
__global__ void __launch_bounds__(PG_NT) paths_grad_kernel(const PathsParams P, double* __restrict__ grad) {
    __shared__ double xs_s[B200BO_MAX_DIM];
    __shared__ double coef[PG_NT];
    __shared__ double red[PG_NT];
    const int tid = threadIdx.x, d = P.d, q = P.q;
    const long long gi = blockIdx.x;
    const int p = P.path_idx[gi];
    if (tid < d) xs_s[tid] = scale_input(P.Xc[gi * d + tid], P.xform, P.ls, tid);
    __syncthreads();
    const int nsl = PG_NT / d, per = PG_NT / nsl;  // slices per dimension, items of a chunk per slice (the last
    const int j = tid % d, sl = tid / d;           // slice also takes the remainder)
    const bool worker = sl < nsl;
    const int i0 = sl * per, i1 = (sl == nsl - 1) ? PG_NT : i0 + per;
    double acc = 0.0;
    for (int pass = 0; pass < 2; ++pass) {
        const double* A = pass ? P.omega : P.Xs;
        const double* B = pass ? P.W : P.V;
        const int cnt = pass ? P.Lp : P.np;
        for (int c0 = 0; c0 < cnt; c0 += PG_NT) {
            const int it = c0 + tid;
            double cf = 0.0;
            if (it < cnt) {
                const double* a = A + (size_t)it * d;
                double s = 0.0;
                for (int jj = 0; jj < d; ++jj) {
                    if (pass) {
                        s = fma(a[jj], xs_s[jj], s);
                    } else {
                        const double df = xs_s[jj] - a[jj];
                        s = fma(df, df, s);
                    }
                }
                if (pass)
                    cf = -P.feat_scale * B[(size_t)it * q + p] * sin(s + P.bias[it]);
                else if (it < P.n)
                    cf = -P.constv * B[(size_t)it * q + p] * cov_dh_eval<COV>(s);
            }
            coef[tid] = cf;
            __syncthreads();
            if (worker) {
                const int e = min(i1, cnt - c0);
                for (int i = i0; i < e; ++i) {
                    const double av = A[(size_t)(c0 + i) * d + j];
                    acc = fma(coef[i], pass ? av : xs_s[j] - av, acc);
                }
            }
            __syncthreads();
        }
    }
    red[tid] = acc;
    __syncthreads();
    if (tid < d) {
        double t = 0.0;
        for (int s2 = 0; s2 < nsl; ++s2) t += red[s2 * d + tid];
        grad[gi * d + tid] = P.xform && xform_rounds(P.xform[tid]) ? 0.0 : P.y_std * t / P.ls[tid];
    }
}

// ---------------------------------------------------------------------------------------
// Constrained Thompson sampling (SCBO rule: Eriksson & Poloczek, AISTATS 2021).  G = 1 + J sets of q paths: set 0
// the target, set j >= 1 constraint GP j with bounds [lb_j, ub_j].  Path p of every set is one joint draw.  Per
// candidate and path, from the values paths_eval_kernel left in vals[g][i][p] (data units):
//   viol = sum_{j=1..J} (max(0, lb_j - c_j) + max(0, c_j - ub_j))         in j order
//   g    = f                       if viol == 0
//        = -T_p (1 + viol)         otherwise,   T_p = 2 B_p + 1 > 2 max|f_p|
// so every infeasible merit lies below every feasible one, and the infeasible tier still resolves viol to relative
// round-off (an additive offset T + viol would resolve it only to ulp(T)).  Explicit _rn intrinsics: no FMA
// contraction, so a numpy restatement on the raw values reproduces g bit for bit.  max() propagates NaN, as
// np.maximum does.  Output: g (m x q), the raw values (m x G x q), and/or -g folded into one list per path.
// ---------------------------------------------------------------------------------------
constexpr int CP_NT = 128;

struct CPathsParams {
    const double* vals;  // [G][stride][q]
    long long stride;    // rows per set in vals
    long long m;         // rows of this launch
    long long index_base;
    int G, q, sel_k, sel_resume;
    double lb[B200BO_MAX_GPS], ub[B200BO_MAX_GPS];  // [j], j >= 1
    double T[B200BO_MAX_PATHS];
    double* merit;      // [m][q] ([m] in row mode) or nullptr
    double* raw;        // [m][G][q] or nullptr (not in row mode)
    SelList* sel_cta;   // [q][gridDim.x] or nullptr (not in row mode)
    const int* path_idx;  // [m]: row mode - vals [G][stride] hold row i's path path_idx[i] only
};

__host__ __device__ inline size_t cpaths_smem_bytes(int q) { return sizeof(SelShared) * (size_t)q; }

__device__ __forceinline__ double cp_pos(double x) { return (x > 0.0 || x != x) ? x : 0.0; }

// ROWS: the merit of row i on path P.path_idx[i] only, from the values the ROWS paths_eval_kernel left; the same
// operations as column path_idx[i] of the full combine.
template <bool ROWS = false>
__global__ void __launch_bounds__(CP_NT) cpaths_select_kernel(const CPathsParams P) {
    extern __shared__ __align__(16) unsigned char cp_smem[];
    SelShared* sel = reinterpret_cast<SelShared*>(cp_smem);
    __shared__ double lb_s[B200BO_MAX_GPS], ub_s[B200BO_MAX_GPS], T_s[B200BO_MAX_PATHS];
    const int t = threadIdx.x, q = ROWS ? 1 : P.q, G = P.G;
    if (t == 0) {  // constant indices: the parameter arrays stay in the constant bank
#pragma unroll
        for (int j = 0; j < B200BO_MAX_GPS; ++j) {
            lb_s[j] = P.lb[j];
            ub_s[j] = P.ub[j];
        }
#pragma unroll
        for (int p = 0; p < B200BO_MAX_PATHS; ++p) T_s[p] = P.T[p];
    }
    if (!ROWS && P.sel_cta)
        for (int p = 0; p < q; ++p) runsel_begin(sel[p], P.sel_cta + (size_t)p * gridDim.x + blockIdx.x, P.sel_resume, t);
    __syncthreads();
    const long long ntiles = (P.m + CP_NT - 1) / CP_NT;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long gi = tile * CP_NT + t;
        const bool valid = gi < P.m;
        for (int p = 0; p < q; ++p) {
            double g = 0.0;
            if (valid) {
                const double f = P.vals[gi * q + p];
                double viol = 0.0;
                for (int j = 1; j < G; ++j) {
                    const double c = P.vals[((size_t)j * P.stride + gi) * q + p];
                    viol = __dadd_rn(viol, __dadd_rn(cp_pos(__dsub_rn(lb_s[j], c)), cp_pos(__dsub_rn(c, ub_s[j]))));
                    if (P.raw) P.raw[((size_t)gi * G + j) * q + p] = c;
                }
                const int pt = ROWS ? P.path_idx[gi] : p;  // the path whose T applies
                g = viol == 0.0 ? f : __dmul_rn(-T_s[pt], __dadd_rn(1.0, viol));
                if (P.raw) P.raw[(size_t)gi * G * q + p] = f;
                if (P.merit) P.merit[gi * q + p] = g;
            }
            if (!ROWS && P.sel_cta) runsel_update<1>(sel[p], P.sel_k, t, -g, gi + P.index_base, valid);
        }
    }
    if (!ROWS && P.sel_cta)
        for (int p = 0; p < q; ++p) runsel_store(sel[p], P.sel_cta + (size_t)p * gridDim.x + blockIdx.x, t);
}

}  // namespace b200bo
