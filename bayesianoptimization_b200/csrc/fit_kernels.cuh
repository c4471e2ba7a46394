// fit_kernels.cuh - kernel-matrix build, blocked Cholesky, triangular inverse, LML gradient.
// Replaces (on device) the arithmetic of GaussianProcessRegressor.fit's tail and
// log_marginal_likelihood (SK/gaussian_process/_gpr.py:349-367, :584-651).
#pragma once
#include "common.cuh"
#include "potrf_block.cuh"

namespace b200bo {

// ---------------------------------------------------------------------------------------
// Xs = transform(X) / length_scale  (rows >= n are zero padding)
// sklearn divides before differencing: cdist(X / length_scale, Y / length_scale)
// (SK/gaussian_process/kernels.py:1716-1720).
// ---------------------------------------------------------------------------------------
__global__ void scale_x_kernel(const double* __restrict__ X, const double* __restrict__ ls,
                               const int* __restrict__ xform, double* __restrict__ Xs, int n,
                               int np, int d) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)np * d) return;
    const int i = (int)(idx / d), j = (int)(idx % d);
    double v = 0.0;
    if (i < n) v = scale_input(X[idx], xform, ls, j);
    Xs[idx] = v;
}

// ---------------------------------------------------------------------------------------
// K(X,X): full symmetric np x np matrix; K_ii = const + alpha; padding = identity.
// (SK/gaussian_process/kernels.py:1716,1740-1743 + _gpr.py:350)
// ---------------------------------------------------------------------------------------
// 32x32 output tile per CTA (32x8 threads, 4 rows each); only tiles on or below the diagonal are computed
// (K is symmetric: pdist evaluates each pair once, kernels.py:1740-1743) and written twice - directly and,
// through a shared-memory transpose, mirrored - so every global store is a coalesced 256-byte row segment.
// The two 32-row slabs of Xs are staged in shared memory (row stride 65: conflict-free when lanes walk
// different rows).  COV is a template parameter: straight-line covariance code as in the predict kernel.
template <int COV>
__global__ void __launch_bounds__(256)
kbuild_kernel(const double* __restrict__ Xs, double* __restrict__ K, int n, int np, int d, double constv,
              double jitter) {
    if (blockIdx.x > blockIdx.y) return;  // strictly-upper tiles are produced by their mirror
    __shared__ double xi[32][B200BO_MAX_DIM + 1], xj[32][B200BO_MAX_DIM + 1];
    __shared__ double tile[32][33];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
    const int j0 = blockIdx.x * 32, i0 = blockIdx.y * 32;
    for (int idx = tid; idx < 32 * d; idx += 256) {
        const int r = idx / d, t = idx - r * d;
        xi[r][t] = Xs[(size_t)i0 * d + idx];
        xj[r][t] = Xs[(size_t)j0 * d + idx];
    }
    __syncthreads();
    const int j = j0 + tx;
    for (int rr = ty; rr < 32; rr += 8) {
        const int i = i0 + rr;
        double v;
        if (i >= n || j >= n) {
            v = (i == j) ? 1.0 : 0.0;
        } else if (i == j) {
            v = constv + jitter;
        } else {
            // the difference is formed as (row with the larger index) - (the other): identical bits on both
            // sides of the diagonal whichever tile produces the pair
            double r2 = 0.0;
            const double* a = (i > j) ? xi[rr] : xj[tx];
            const double* b = (i > j) ? xj[tx] : xi[rr];
            for (int t = 0; t < d; ++t) {
                const double df = a[t] - b[t];
                r2 += df * df;
            }
            v = constv * cov_eval<COV>(r2);
        }
        K[(size_t)i * np + j] = v;
        tile[rr][tx] = v;
    }
    if (blockIdx.x == blockIdx.y) return;
    __syncthreads();
    for (int rr = ty; rr < 32; rr += 8) K[(size_t)(j0 + rr) * np + i0 + tx] = tile[tx][rr];
}

// ---------------------------------------------------------------------------------------
// Generic fp64 GEMM on 64x64 tiles (fit-side building block; inner product on the fp64 tensor
// path, mma.sync m8n8k4 - the trailing SYRK/GEMM updates of the blocked Cholesky, the triangular
// inverse recursion and K^-1 all run through it):
//   C[m][n] = beta*C[m][n] + alpha * sum_k opA(m,k) * opB(k,n)
//   opA(m,k) = TA ? A[k*lda+m] : A[m*lda+k];  opB(k,n) = TB ? B[n*ldb+k] : B[k*ldb+n]
// M, N multiples of 64; K multiple of 16.  lower_only: skip tiles strictly above the diagonal.
// kmode: 0 = full K range; 1 = k in [0, m0+64)   (A or B lower-triangular in (m,k)/(k,n) sense:
//        caller guarantees contributions with k >= m0+64 vanish);
//        2 = k in [n0, K)                       (contributions with k < n0 vanish)
//        3 = k in [max(m0,n0), K)
// Batched over blockIdx.z with element strides sA/sB/sC.
// ---------------------------------------------------------------------------------------
template <bool TA, bool TB>
__global__ void __launch_bounds__(256)
dgemm64_kernel(int M, int N, int K, double alpha, const double* __restrict__ A, int lda,
               long long sA, const double* __restrict__ B, int ldb, long long sB, double beta,
               double* C, int ldc, long long sC, int lower_only, int kmode, int skip) {
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    if (lower_only && n0 > m0) return;
    if (m0 < skip && n0 < skip) return;  // leading skip x skip block of C is left untouched (look-ahead Cholesky)
    A += (long long)blockIdx.z * sA;
    B += (long long)blockIdx.z * sB;
    C += (long long)blockIdx.z * sC;
    // k-major tiles, row stride 68 doubles = 8 words (mod 32): the 4 k-rows x 4 columns an LDS.64
    // half-warp touches for an m8n8k4 fragment fall on disjoint banks
    __shared__ double As[16][68];
    __shared__ double Bs[16][68];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 3, wn = warp >> 2;  // warp tile: rows wm*16..+16, cols wn*32..+32
    const int g = lane >> 2, t4 = lane & 3;
    double acc[2][4][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    int kbeg = 0, kend = K;
    if (kmode == 1) kend = min(K, m0 + 64);
    if (kmode == 2) kbeg = n0;
    if (kmode == 3) kbeg = max(m0, n0);

    for (int k0 = kbeg; k0 < kend; k0 += 16) {
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int idx = tid + t * 256;
            if (TA) {
                const int m = idx & 63, kk = idx >> 6;
                As[kk][m] = A[(size_t)(k0 + kk) * lda + m0 + m];
            } else {
                const int kk = idx & 15, m = idx >> 4;
                As[kk][m] = A[(size_t)(m0 + m) * lda + k0 + kk];
            }
            if (TB) {
                const int kk = idx & 15, n = idx >> 4;
                Bs[kk][n] = B[(size_t)(n0 + n) * ldb + k0 + kk];
            } else {
                const int n = idx & 63, kk = idx >> 6;
                Bs[kk][n] = B[(size_t)(k0 + kk) * ldb + n0 + n];
            }
        }
        __syncthreads();
        // fp64 tensor path: mma.sync m8n8k4 (DMMA); 2 x 4 fragments per warp and k-step
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
            double a[2], b[4];
#pragma unroll
            for (int i = 0; i < 2; ++i) a[i] = As[k4 * 4 + t4][wm * 16 + i * 8 + g];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[k4 * 4 + t4][wn * 32 + j * 8 + g];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                                 : "+d"(acc[i][j][0]), "+d"(acc[i][j][1])
                                 : "d"(a[i]), "d"(b[j]));
        }
        __syncthreads();
    }
    // C fragment: row = g, columns 2*t4 + {0,1}
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                double* c = C + (size_t)(m0 + wm * 16 + i * 8 + g) * ldc + n0 + wn * 32 + j * 8 + 2 * t4 + e;
                const double v = alpha * acc[i][j][e];
                *c = (beta == 0.0) ? v : fma(beta, *c, v);
            }
}

// ---------------------------------------------------------------------------------------
// fp64 GEMM on 128x128 tiles: the workhorse of the fit side (trailing SYRK/GEMM updates of the blocked
// Cholesky, the triangular-inverse recursion, K^-1 = W^T W, predict(return_cov)).  Same contract as
// dgemm64_kernel (opA/opB, lower_only, kmode, batching) with M, N arbitrary multiples of 64 (edge tiles are
// predicated) and K a multiple of 16.  256 threads, warp tile 32(m) x 64(n), mma.sync m8n8k4 f64 (DMMA),
// k-tile 16, 3-stage 16-byte cp.async pipeline with the prefetch issued behind the first MMA batch - the
// machinery of predict_phase_b_dmma.  Each operand keeps in shared memory the orientation it has in global
// memory (so that every copy is a straight 16-byte cp.async):
//   k-major  [16][132]  (stride 264 words = 8 mod 32)   for A^T-stored / B-stored operands
//   mn-major [128][20]  (stride 40 words = 8 mod 32)    for A-stored / B^T-stored operands
// both give conflict-free LDS.64 fragment loads (an LDS.64 is served per half-warp: 4 k x 4 m).
// ---------------------------------------------------------------------------------------
constexpr int G128_BK = 16, G128_STAGES = 3;
constexpr int G128_KSTR = 132, G128_MSTR = 20;
constexpr int G128_OPER = 128 * G128_MSTR;  // doubles per operand per stage (>= 16 * 132)
constexpr int kGemm128SmemBytes = G128_STAGES * 2 * G128_OPER * 8;  // 122880

__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gmem_src, bool valid) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    const int bytes = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "r"(bytes));
}

// one operand tile: 128 (m or n) x 16 (k).  TRANS = stored [k][mn] in global (contiguous in mn).
template <bool TRANS>
__device__ __forceinline__ void g128_load_operand(double* sm, const double* __restrict__ G, int ld, int mn0,
                                                  int k0, int mn_limit) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int q = tid + t * 256;
        if (TRANS) {
            const int kk = q >> 6, c = (q & 63) * 2;
            const bool ok = mn0 + c < mn_limit;
            cp_async16_zfill(sm + kk * G128_KSTR + c, G + (size_t)(k0 + kk) * ld + (ok ? mn0 + c : 0), ok);
        } else {
            const int r = q >> 3, c = (q & 7) * 2;
            const bool ok = mn0 + r < mn_limit;
            cp_async16_zfill(sm + r * G128_MSTR + c, G + (size_t)(ok ? mn0 + r : 0) * ld + k0 + c, ok);
        }
    }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(256, 1)
dgemm128_kernel(int M, int N, int K, double alpha, const double* __restrict__ A, int lda, long long sA,
                const double* __restrict__ B, int ldb, long long sB, double beta, double* C, int ldc,
                long long sC, int lower_only, int kmode, int skip, double* __restrict__ side) {
    extern __shared__ __align__(16) double g128_smem[];
    // tile order: heaviest tiles first.  With triangular k-ranges (kmode) a tile's work is proportional to its
    // k-length; blocks are dispatched in linear order, and a full-length tile that starts in the second wave
    // determines the duration of the launch.
    int bx = blockIdx.x, by = blockIdx.y;
    {
        const int lin = blockIdx.y * gridDim.x + blockIdx.x;
        if (kmode == 2) {          // k in [n0, K): small n0 = heavy -> n-tiles become the slow index
            bx = lin / gridDim.y;
            by = lin % gridDim.y;
        } else if (kmode == 1) {   // k in [0, m0 + 128): large m0 = heavy -> descending m-tiles, slow index
            by = gridDim.y - 1 - lin / gridDim.x;
            bx = lin % gridDim.x;
        }
    }
    const int m0 = by * 128, n0 = bx * 128;
    if (lower_only && n0 > m0) return;
    A += (long long)blockIdx.z * sA;
    B += (long long)blockIdx.z * sB;
    C += (long long)blockIdx.z * sC;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 3, wn = warp >> 2;
    const int g = lane >> 2, t4 = lane & 3;
    double acc[4][8][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    int kbeg = 0, kend = K;
    if (kmode == 1) kend = min(K, m0 + 128);
    if (kmode == 2) kbeg = n0;
    if (kmode == 3) kbeg = max(m0, n0);
    const int nks = (kend - kbeg) / G128_BK;
    auto stage_a = [&](int s) { return g128_smem + (size_t)s * 2 * G128_OPER; };
    auto stage_b = [&](int s) { return g128_smem + (size_t)s * 2 * G128_OPER + G128_OPER; };
    auto load = [&](int s, int ks) {
        const int k0 = kbeg + ks * G128_BK;
        g128_load_operand<TA>(stage_a(s), A, lda, m0, k0, M);    // TA: A stored [k][m]
        g128_load_operand<!TB>(stage_b(s), B, ldb, n0, k0, N);   // !TB: B stored [k][n]
    };
#pragma unroll
    for (int s = 0; s < G128_STAGES - 1; ++s) {
        if (s < nks) load(s, s);
        cp_async_commit();
    }
    for (int ks = 0; ks < nks; ++ks) {
        cp_async_wait<G128_STAGES - 2>();
        __syncthreads();
        const int nxt = ks + G128_STAGES - 1;
        const double* as = stage_a(ks % G128_STAGES);
        const double* bs = stage_b(ks % G128_STAGES);
#pragma unroll
        for (int k4 = 0; k4 < G128_BK / 4; ++k4) {
            if (k4 == 1) {
                if (nxt < nks) load(nxt % G128_STAGES, nxt);
                cp_async_commit();
            }
            double a[4], b[8];
            const int kk = k4 * 4 + t4;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = wm * 32 + i * 8 + g;
                a[i] = TA ? as[kk * G128_KSTR + m] : as[m * G128_MSTR + kk];
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = wn * 64 + j * 8 + g;
                b[j] = TB ? bs[n * G128_MSTR + kk] : bs[kk * G128_KSTR + n];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                                 : "+d"(acc[i][j][0]), "+d"(acc[i][j][1])
                                 : "d"(a[i]), "d"(b[j]));
        }
    }
    cp_async_wait<0>();
    // C fragment: row = g, columns 2*t4 + {0,1}: one 16-byte store per fragment
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + wm * 32 + i * 8 + g;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + wn * 64 + j * 8 + 2 * t4;
            if (n >= N || (m < skip && n < skip)) continue;  // skip: see dgemm64_kernel
            double2* c = reinterpret_cast<double2*>(C + (size_t)m * ldc + n);
            double2 v = make_double2(alpha * acc[i][j][0], alpha * acc[i][j][1]);
            if (beta != 0.0) {
                const double2 o = *c;
                v.x = fma(beta, o.x, v.x);
                v.y = fma(beta, o.y, v.y);
            }
            *c = v;
            // look-ahead Cholesky: the updated block (rows 64..127, columns 0..63 of C) is also stored densely in
            // `side` - it is what the NEXT diagonal kernel needs before the bulk panel solve overwrites it in place
            if (side && m >= 64 && m < 128 && n < 64) *reinterpret_cast<double2*>(side + (size_t)(m - 64) * 64 + n) = v;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Rank-64 trailing update of the blocked Cholesky:  C[M x M] (tiles on/below the diagonal) -= P P^T with P the
// M x 64 panel (row-major, leading dimension ldp).  A 128x128 GEMM tile spends as long loading its operands and
// reading / writing C as it spends on its four k-steps of DMMA; here a CTA owns a 64(m) x 128(n) tile, the whole
// K = 64 of both operands is fetched by ONE batch of cp.async (104 KB of shared memory), and TWO CTAs are resident
// per SM (<= 128 registers: warp tile 16 x 64), so one CTA's load / C read-modify-write phase runs under the other's
// DMMA phase.  Same skip / side conventions as dgemm128_kernel.
// ---------------------------------------------------------------------------------------
constexpr int TU_STR = 68;  // row stride (doubles) of the mn-major operand tiles: 136 words = 8 (mod 32)
constexpr int kTrailSmemBytes = (64 + 128) * TU_STR * 8;  // 104448
__global__ void __launch_bounds__(256, 2)
trailing_update64_kernel(int M, const double* __restrict__ P, int ldp, double* C, int ldc, int skip,
                         double* __restrict__ side) {
    extern __shared__ __align__(16) double tu_smem[];
    double* As = tu_smem;                 // [64][TU_STR]   rows m0.. of the panel
    double* Bs = tu_smem + 64 * TU_STR;   // [128][TU_STR]  rows n0.. of the panel
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 128;
    if (n0 > m0) return;                       // tiles strictly above the diagonal
    if (m0 + 64 <= skip && n0 + 128 <= skip) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // 64 k = 32 16-byte pieces per row
    for (int q = tid; q < 64 * 32; q += 256) {
        const int r = q >> 5, c = (q & 31) * 2;
        const bool ok = m0 + r < M;
        cp_async16_zfill(As + r * TU_STR + c, P + (size_t)(ok ? m0 + r : 0) * ldp + c, ok);
    }
    for (int q = tid; q < 128 * 32; q += 256) {
        const int r = q >> 5, c = (q & 31) * 2;
        const bool ok = n0 + r < M;
        cp_async16_zfill(Bs + r * TU_STR + c, P + (size_t)(ok ? n0 + r : 0) * ldp + c, ok);
    }
    cp_async_commit();
    const int wm = warp & 3, wn = warp >> 2;
    const int g = lane >> 2, t4 = lane & 3;
    double acc[2][8][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    cp_async_wait<0>();
    __syncthreads();
#pragma unroll 4
    for (int k4 = 0; k4 < 16; ++k4) {
        double a[2], b[8];
        const int kk = k4 * 4 + t4;
#pragma unroll
        for (int i = 0; i < 2; ++i) a[i] = As[(wm * 16 + i * 8 + g) * TU_STR + kk];
#pragma unroll
        for (int j = 0; j < 8; ++j) b[j] = Bs[(wn * 64 + j * 8 + g) * TU_STR + kk];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j)
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                             : "+d"(acc[i][j][0]), "+d"(acc[i][j][1])
                             : "d"(a[i]), "d"(b[j]));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int m = m0 + wm * 16 + i * 8 + g;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + wn * 64 + j * 8 + 2 * t4;
            if (n >= M || (m < skip && n < skip)) continue;
            double2* c = reinterpret_cast<double2*>(C + (size_t)m * ldc + n);
            const double2 o = *c;
            const double2 v = make_double2(o.x - acc[i][j][0], o.y - acc[i][j][1]);
            *c = v;
            if (side && m >= 64 && m < 128 && n < 64) *reinterpret_cast<double2*>(side + (size_t)(m - 64) * 64 + n) = v;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Diagonal 64x64 block: in-place Cholesky (lower) + inverse of the factor written to Dinv.
// Single CTA, 256 threads, phases in potrf_block.cuh (8-column panels: 3 barriers per panel
// instead of 2 per column, one rsqrt per pivot instead of sqrt + divisions; inverse by recursive
// doubling instead of 64 dependent substitution steps).  Agrees with the unblocked kernel below to
// round-off.
// info: 0 or the 1-based index of the first non-positive pivot (LAPACK dpotrf convention,
// SP/linalg/_decomp_cholesky.py:58 raises LinAlgError on it).
// ---------------------------------------------------------------------------------------
constexpr int kPotrfSmemBytes = 3 * potrf::kB * potrf::kLd * 8;
// Look-ahead form (Pprev != nullptr): the block's dependence on the PREVIOUS panel is resolved inside this
// kernel, so that the factorisation chain does not wait for the bulk TRSM / trailing update of that panel:
//   X = Pprev * Dprev^T      (Pprev = A[j, j-1] before the panel solve, Dprev = inv(L_{j-1,j-1}), both 64x64)
//   S = A[j, j] - X X^T      (A[j, j] carries the updates of panels <= j-2; the bulk update of panel j-1 skips it)
// The bulk stream computes its own copy of L[j, j-1] for the final factor; X is used here only.
__global__ void __launch_bounds__(256)
potrf_diag_kernel(double* A, int ld, int j0, double* Dinv, int ldd, int* info, const double* __restrict__ Pprev,
                  const double* __restrict__ Dprev, int ldp) {
    using namespace potrf;
    extern __shared__ __align__(16) double potrf_smem[];
    double* S = potrf_smem;
    double* V = potrf_smem + kB * kLd;
    double* T = potrf_smem + 2 * kB * kLd;
    __shared__ double diag[kB], rdiag[kB];
    const int tid = threadIdx.x, warp = tid >> 5;
    for (int idx = tid; idx < kB * kB; idx += kThreads) {
        const int r = idx >> 6, c = idx & 63;
        S[r * kLd + c] = A[(size_t)(j0 + r) * ld + j0 + c];
        V[r * kLd + c] = Pprev ? Pprev[r * kB + c] : 0.0;
        if (Pprev) T[r * kLd + c] = (c <= r) ? Dprev[(size_t)r * ldp + c] : 0.0;
    }
    __syncthreads();
    if (Pprev) {
        // 4x4 register tiles with STRIDED ownership: thread (ti, tj) owns rows ti + 16 i and columns tj + 16 j.  With
        // the row stride of 65 doubles the 16 tj-lanes of a half-warp then read 16 different even banks (contiguous
        // 4-column ownership put lanes tj and tj+4 on the same banks: a 4-way conflict on every operand load).
        const int tj = tid & 15, ti = tid >> 4;
        double acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
        for (int k = 0; k < kB; ++k) {  // Dprev was loaded with zeros above its diagonal
            double p[4], dd[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) p[i] = V[(ti + 16 * i) * kLd + k];
#pragma unroll
            for (int j = 0; j < 4; ++j) dd[j] = T[(tj + 16 * j) * kLd + k];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(p[i], dd[j], acc[i][j]);
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) V[(ti + 16 * i) * kLd + tj + 16 * j] = acc[i][j];  // X over P
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
        for (int k = 0; k < kB; ++k) {
            double xr[4], xc[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xr[i] = V[(ti + 16 * i) * kLd + k];
#pragma unroll
            for (int j = 0; j < 4; ++j) xc[j] = V[(tj + 16 * j) * kLd + k];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(xr[i], xc[j], acc[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (tj + 16 * j <= ti + 16 * i) S[(ti + 16 * i) * kLd + tj + 16 * j] -= acc[i][j];  // lower part of S -= X X^T
        __syncthreads();
        for (int idx = tid; idx < kB * kB; idx += kThreads) V[(idx >> 6) * kLd + (idx & 63)] = 0.0;
        __syncthreads();
    }
    for (int c0 = 0; c0 < kB; c0 += kPw) {
        if (warp == 0) {
            const int bad = diag_factor(S, diag, rdiag, c0);
            if (bad != 0 && tid == 0 && *info == 0) *info = j0 + bad;
        }
        __syncthreads();
        if (c0 + kPw < kB) {
            panel_solve(tid, S, rdiag, c0);
            __syncthreads();
            trailing_update(tid, S, c0);
            __syncthreads();
        }
    }
    // factor back to global memory (strict upper part of the block zeroed)
    for (int idx = tid; idx < kB * kB; idx += kThreads) {
        const int r = idx >> 6, c = idx & 63;
        A[(size_t)(j0 + r) * ld + j0 + c] = (c < r) ? S[r * kLd + c] : (c == r ? diag[r] : 0.0);
    }
    diag_inverse(S, rdiag, V, warp);  // 8 warps <-> 8 diagonal 8x8 blocks
    __syncthreads();
    for (int s = kPw, l2 = 3; s < kB; s *= 2, ++l2) {
        inverse_level_t(tid, S, V, T, s, l2);
        __syncthreads();
        inverse_level_w(tid, V, T, s, l2);
        __syncthreads();
    }
    for (int idx = tid; idx < kB * kB; idx += kThreads) {
        const int r = idx >> 6, c = idx & 63;
        Dinv[(size_t)r * ldd + c] = V[r * kLd + c];
    }
}

// ---------------------------------------------------------------------------------------
// Diagonal 64x64 block, first version (kept for A/B runs: B200BO_POTRF=legacy): unblocked
// column-by-column Cholesky (two barriers per column) + inverse by forward substitution.
// Single CTA, 256 threads.  info: 0 or the 1-based index of the first non-positive pivot
// (LAPACK dpotrf convention, SP/linalg/_decomp_cholesky.py:58 raises LinAlgError on it).
// ---------------------------------------------------------------------------------------
constexpr int kPotrfLegacySmemBytes = 2 * 64 * 65 * 8;
__global__ void __launch_bounds__(256)
potrf_diag_legacy_kernel(double* A, int ld, int j0, double* Dinv, int ldd, int* info) {
    extern __shared__ __align__(16) double potrf_smem[];
    double (*S)[65] = reinterpret_cast<double (*)[65]>(potrf_smem);
    double (*V)[65] = reinterpret_cast<double (*)[65]>(potrf_smem + 64 * 65);
    const int tid = threadIdx.x;
    for (int idx = tid; idx < 64 * 64; idx += 256) {
        const int r = idx >> 6, c = idx & 63;
        S[r][c] = A[(size_t)(j0 + r) * ld + j0 + c];
    }
    __syncthreads();
    // right-looking, two barriers per column: every thread derives the pivot itself (the square
    // root goes to diag[], S[k][k] keeps the pivot so late readers still see it), the first 64
    // threads scale the column, then all 256 apply the rank-1 update to the trailing lower triangle
    __shared__ double diag[64];
    for (int k = 0; k < 64; ++k) {
        double piv = S[k][k];
        const bool bad = !(piv > 0.0);
        if (bad) piv = 1.0;
        const double lkk = sqrt(piv);
        if (tid == k) {
            diag[k] = lkk;
            if (bad && *info == 0) *info = j0 + k + 1;
        } else if (tid > k && tid < 64) {
            S[tid][k] = S[tid][k] / lkk;
        }
        __syncthreads();
        // trailing block (k+1..63)^2, lower part: S[i][j] -= S[i][k]*S[j][k]; 16x16 thread grid,
        // no integer divisions on the critical path
        for (int i = k + 1 + (tid >> 4); i < 64; i += 16) {
            const double lik = S[i][k];
            for (int j = k + 1 + (tid & 15); j <= i; j += 16) S[i][j] = fma(-lik, S[j][k], S[i][j]);
        }
        __syncthreads();
    }
    // write factor back (zero the strict upper part of the block)
    for (int idx = tid; idx < 64 * 64; idx += 256) {
        const int r = idx >> 6, c = idx & 63;
        A[(size_t)(j0 + r) * ld + j0 + c] = (c < r) ? S[r][c] : (c == r ? diag[r] : 0.0);
    }
    // inverse of the lower-triangular block: column c by forward substitution, 4 threads per
    // column share each dot product (lanes 4c..4c+3, combined with two shuffles, fixed order)
    {
        const int c = tid >> 2, q = tid & 3;
        for (int i = 0; i < 64; ++i) {
            double part = 0.0;
            for (int k = c + q; k < i; k += 4) part = fma(S[i][k], V[k][c], part);
            part += __shfl_xor_sync(0xffffffffu, part, 1);
            part += __shfl_xor_sync(0xffffffffu, part, 2);
            if (q == 0) {
                double v = 0.0;
                if (i >= c) v = (((i == c) ? 1.0 : 0.0) - part) / diag[i];
                V[i][c] = v;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    for (int idx = tid; idx < 64 * 64; idx += 256) {
        const int r = idx >> 6, c = idx & 63;
        Dinv[(size_t)r * ldd + c] = V[r][c];
    }
}

// dst[64][64] (dense) = src[64 rows][64 cols] with row stride ld: the look-ahead copy of A[j+1, j] taken
// before the bulk stream's in-place panel solve overwrites it
__global__ void __launch_bounds__(256) copy_block64_kernel(const double* __restrict__ src, int ld, double* __restrict__ dst) {
    for (int idx = threadIdx.x; idx < 64 * 64; idx += 256) dst[idx] = src[(size_t)(idx >> 6) * ld + (idx & 63)];
}

// zero the strict upper triangle (scipy.linalg.cholesky(lower=True) returns a clean factor)
__global__ void zero_upper_kernel(double* A, int np) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y * blockDim.y + threadIdx.y;
    if (i < np && j < np && j > i) A[(size_t)i * np + j] = 0.0;
}

// out[j][i] = in[i][j]  (np multiple of 32)
__global__ void transpose_kernel(const double* __restrict__ in, double* __restrict__ out, int np) {
    __shared__ double t[32][33];
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y)
        t[r][threadIdx.x] = in[(size_t)(by + r) * np + bx + threadIdx.x];
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y)
        out[(size_t)(bx + r) * np + by + threadIdx.x] = t[threadIdx.x][r];
}

// y[i] = sum_j A[i][j] * x[j], j in [jbeg(i), jend(i)); one warp per row, fixed-order reduction.
// tri: 0 full [0,ncols); 1 lower (j <= i); 2 upper (j >= i)
__global__ void gemv_rows_kernel(const double* __restrict__ A, int ld, const double* __restrict__ x,
                                 double* __restrict__ y, int nrows, int ncols, int tri) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    int jb = 0, je = ncols;
    if (tri == 1) je = min(ncols, row + 1);
    if (tri == 2) jb = row & ~31;
    double s = 0.0;
    for (int j = jb + lane; j < je; j += 32) {
        if (tri == 2 && j < row) continue;
        s = fma(A[(size_t)row * ld + j], x[j], s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) y[row] = s;
}

__global__ void diag_kernel(const double* __restrict__ A, int ld, double* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = A[(size_t)i * ld + i];
}

// r = y - r   (elementwise, n entries)
__global__ void residual_kernel(const double* __restrict__ y, double* __restrict__ r, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) r[i] = y[i] - r[i];
}
// a += b
__global__ void axpy1_kernel(double* __restrict__ a, const double* __restrict__ b, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] += b[i];
}

// ---------------------------------------------------------------------------------------
// LML gradient:  grad_p = 0.5 * sum_ij (alpha_i alpha_j - Kinv_ij) * dK_ij/dtheta_p
// (SK/gaussian_process/_gpr.py:629-651, kernels.py:1745-1786 / :1561-1573).
// theta order: [log const (if has_const)], log length_scale (1 or d).
// Each CTA reduces a 16x16 patch of (i,j) pairs in a fixed order and writes its partial
// sums to part[block][p]; the host adds the partials in index order (deterministic).
// ---------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------
// predict(return_cov=True) helpers (SK/gaussian_process/_gpr.py:464-475)
// ---------------------------------------------------------------------------------------
// Xcs = transform(Xc)/length_scale, rows >= m zero
__global__ void scale_xc_kernel(const double* __restrict__ Xc, const double* __restrict__ ls,
                                const int* __restrict__ xform, double* __restrict__ Xcs, int m, int mp, int d) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)mp * d) return;
    const int i = (int)(idx / d), j = (int)(idx % d);
    double v = 0.0;
    if (i < m) v = scale_input(Xc[idx], xform, ls, j);
    Xcs[idx] = v;
}
// Kst[k][c] = const * cov(Xs[k], Xcs[c])  (np x mp, zero for padded rows/columns)
__global__ void kcross_kernel(const double* __restrict__ Xs, const double* __restrict__ Xcs,
                              double* __restrict__ Kst, int n, int np, int m, int mp, int d, int family, int nu,
                              double constv) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int k = blockIdx.y * blockDim.y + threadIdx.y;
    if (k >= np || c >= mp) return;
    double v = 0.0;
    if (k < n && c < m) {
        const double* a = Xcs + (size_t)c * d;
        const double* b = Xs + (size_t)k * d;
        double r2 = 0.0;
        for (int t = 0; t < d; ++t) {
            const double df = a[t] - b[t];
            r2 = fma(df, df, r2);
        }
        v = constv * cov_from_r2(r2, family, nu);
    }
    Kst[(size_t)k * mp + c] = v;
}
// mu[c] = y_std * sum_k alpha[k] Kst[k][c] + y_mean
__global__ void cross_mean_kernel(const double* __restrict__ Kst, const double* __restrict__ alphav,
                                  double* __restrict__ mu, int np, int m, int mp, double y_mean, double y_std) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= m) return;
    double s = 0.0;
    for (int k = 0; k < np; ++k) s = fma(alphav[k], Kst[(size_t)k * mp + c], s);
    mu[c] = y_std * s + y_mean;
}
// cov[i][j] = (k(x_i, x_j) - (V^T V)[i][j]) * y_std^2   (m x m, contiguous)
__global__ void cov_finish_kernel(const double* __restrict__ Xcs, const double* __restrict__ VtV, int ldv,
                                  double* __restrict__ cov, int m, int d, int family, int nu, double constv,
                                  double y_std, double noise) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= m || j >= m) return;
    double kv;
    if (i == j) {
        kv = constv + noise;  // kernel_(X) with Y=None: a WhiteKernel term sits on the diagonal
    } else {
        const double* a = Xcs + (size_t)min(i, j) * d;
        const double* b = Xcs + (size_t)max(i, j) * d;
        double r2 = 0.0;
        for (int t = 0; t < d; ++t) {
            const double df = a[t] - b[t];
            r2 += df * df;
        }
        kv = constv * cov_from_r2(r2, family, nu);
    }
    cov[(size_t)i * m + j] = (kv - VtV[(size_t)i * ldv + j]) * (y_std * y_std);
}

// ---------------------------------------------------------------------------------------
// Incremental factor update at fixed hyper-parameters (SURVEY.md 8f rank 3): one training point
// is appended in O(N^2): new row of K, of L (l = L^-1 k, pivot sqrt(c+alpha-|l|^2)) and of L^-1.
// ---------------------------------------------------------------------------------------
// Xs[n] = transform(x)/ls ; kvec[i] = const*cov(Xs[i], Xs[n]) for i < n
__global__ void append_krow_kernel(const double* __restrict__ x_new, const double* __restrict__ ls,
                                   const int* __restrict__ xform, double* __restrict__ Xs, double* __restrict__ X,
                                   double* __restrict__ kvec, int n, int d, int family, int nu, double constv) {
    __shared__ double xs[B200BO_MAX_DIM];
    if (threadIdx.x < d) {
        double v = x_new[threadIdx.x];
        if (blockIdx.x == 0) X[(size_t)n * d + threadIdx.x] = v;
        v = scale_input(v, xform, ls, threadIdx.x);
        xs[threadIdx.x] = v;
        if (blockIdx.x == 0) Xs[(size_t)n * d + threadIdx.x] = v;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* a = Xs + (size_t)i * d;
    double r2 = 0.0;
    for (int t = 0; t < d; ++t) {
        const double df = a[t] - xs[t];
        r2 += df * df;
    }
    kvec[i] = constv * cov_from_r2(r2, family, nu);
}
// write row/column n of K, row n of L; pivot check.  lvec = L^-1[0:n,0:n] kvec.
__global__ void append_rows_kernel(double* __restrict__ K, double* __restrict__ L, const double* __restrict__ kvec,
                                   const double* __restrict__ lvec, int n, int np, double diag, int* info,
                                   double* __restrict__ pivot_out) {
    __shared__ double red[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) {
        const double l = lvec[i], k = kvec[i];
        s = fma(l, l, s);
        K[(size_t)n * np + i] = k;
        K[(size_t)i * np + n] = k;
        L[(size_t)n * np + i] = l;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int t = 128; t > 0; t >>= 1) {
        if (threadIdx.x < t) red[threadIdx.x] += red[threadIdx.x + t];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double piv = diag - red[0];
        if (!(piv > 0.0)) {
            *info = n + 1;
            piv = 1.0;
        }
        const double lnn = sqrt(piv);
        K[(size_t)n * np + n] = diag;
        L[(size_t)n * np + n] = lnn;
        *pivot_out = lnn;
    }
}
// row n of W = L^-1 and column n of WT:  W[n][j] = -(1/l_nn) * t[j], t = W[0:n,0:n]^T lvec ; W[n][n] = 1/l_nn
__global__ void append_winv_kernel(double* __restrict__ W, double* __restrict__ WT, const double* __restrict__ tvec,
                                   const double* __restrict__ pivot, int n, int np) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const double inv = 1.0 / *pivot;
    if (j < n) {
        const double w = -inv * tvec[j];
        W[(size_t)n * np + j] = w;
        WT[(size_t)j * np + n] = w;
    } else if (j == n) {
        W[(size_t)n * np + n] = inv;
        WT[(size_t)n * np + n] = inv;
    }
}

// NEI fantasies at a pending row n just appended to the noiseless factor (b200bo_gp_condition_fantasies): one warp per
// sample s,  F[s][n] = sum_{i<n} L[n][i] Z[s][i] + sum_{i<nreg} K[n][i] W[s][i] + L[n][n] z_s  in a fixed order (lane
// strides, then a butterfly), the joint prior draw from the grown factor plus the Matheron update over the registered
// rows.  Stores F[s][n] and Z[s][n] = z_s and raises best_s (data units) behind A: best[s] = max(best[s], y_std F + y_mean).
__global__ void fantasy_row_kernel(const double* __restrict__ K, const double* __restrict__ L, int np, int n, int nreg,
                                   const double* __restrict__ W, const double* __restrict__ zrow, double* __restrict__ Z,
                                   double* __restrict__ F, double* __restrict__ best, double y_std, double y_mean) {
    const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const double* lrow = L + (size_t)n * np;
    const double* krow = K + (size_t)n * np;
    const double* zs = Z + (size_t)s * np;
    const double* ws = W + (size_t)s * nreg;
    double acc = 0.0;
    for (int i = lane; i < n; i += 32) acc = fma(lrow[i], zs[i], acc);
    for (int i = lane; i < nreg; i += 32) acc = fma(krow[i], ws[i], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        const double z = zrow[s];
        const double f = fma(lrow[n], z, acc);
        Z[(size_t)s * np + n] = z;
        F[(size_t)s * np + n] = f;
        best[s] = fmax(best[s], y_std * f + y_mean);
    }
}
// The GPs of a constrained incumbent (b200bo_gp_set_constrained_incumbent): F ([S][np], normalised) and the y statistics
// of the target (index 0) and of each constraint, with the constraint's bounds (data units; index 0 unused).
struct IncumbentGPs {
    const double* f[B200BO_MAX_GPS];
    double y_std[B200BO_MAX_GPS], y_mean[B200BO_MAX_GPS];
    double lb[B200BO_MAX_GPS], ub[B200BO_MAX_GPS];
    int n_gps;
};
// CNEI's incumbents over the n rows of the handles (DESIGN.md 4.16): one warp per sample s.  Each value is taken to data
// units as v = y_std F + y_mean with separate roundings (the host's arithmetic, no FMA contraction); row i is eligible
// when in_bounds[i] != 0 and every constraint's v lies in [lb, ub].  best[s] = max of the target's v over the eligible
// rows, or min over all rows when none is.  max / min are exact, so the lane order does not change the result.
__global__ void fantasy_incumbent_kernel(const IncumbentGPs G, const uint8_t* __restrict__ in_bounds, int n, int np,
                                         double* __restrict__ best) {
    const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double hi = -CUDART_INF, lo = CUDART_INF;
    bool any = false;
    for (int i = lane; i < n; i += 32) {
        const size_t k = (size_t)s * np + i;
        const double v = __dadd_rn(__dmul_rn(G.y_std[0], G.f[0][k]), G.y_mean[0]);
        lo = fmin(lo, v);
        bool ok = in_bounds[i] != 0;
        for (int g = 1; g < G.n_gps && ok; ++g) {
            const double c = __dadd_rn(__dmul_rn(G.y_std[g], G.f[g][k]), G.y_mean[g]);
            ok = G.lb[g] <= c && c <= G.ub[g];
        }
        if (ok) {
            hi = fmax(hi, v);
            any = true;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    }
    any = __any_sync(0xffffffffu, any);
    if (lane == 0) best[s] = any ? hi : lo;
}
// A[i][s] = Acol[s][i] for i < n, zero for n <= i < np: the [np][S] layout the NEI kernels read
__global__ void fantasy_pack_kernel(const double* __restrict__ Acol, int np, int n, int S, double* __restrict__ A) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= np * S) return;
    const int i = idx / S, s = idx % S;
    A[idx] = i < n ? Acol[(size_t)s * np + i] : 0.0;
}

// Re-pitch of an np_src x np_src matrix into an np_dst x np_dst one (np_dst >= np_src, both multiples of 32), in one
// pass: dst[i][j] = src[i][j] inside the source block, the identity outside it - the padding invariant of K, L, L^-1
// and its transpose.  32x8 threads per 32x32 tile, 4 rows each; every store is a coalesced 256-byte row segment.
__global__ void __launch_bounds__(256)
repitch_identity_kernel(const double* __restrict__ src, int np_src, double* __restrict__ dst, int np_dst) {
    const int j = blockIdx.x * 32 + threadIdx.x;
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int i = blockIdx.y * 32 + r;
        dst[(size_t)i * np_dst + j] =
            (i < np_src && j < np_src) ? src[(size_t)i * np_src + j] : (i == j ? 1.0 : 0.0);
    }
}

constexpr int kMaxTheta = B200BO_MAX_DIM + 1;

// gradient factor such that dk/dlog(l_t) = gcommon * D_t  (D_t = scaled squared difference)
// (SK/gaussian_process/kernels.py:1761-1782 Matern, :1561-1573 RBF)
template <int COV>
__device__ __forceinline__ void cov_and_gradfactor(double r2, double& kval, double& gcommon) {
    if (COV == 3) {
        kval = exp_neg(0.5 * r2);
        gcommon = kval;  // K_gradient = D * K
    } else if (COV == 2) {
        const double tmp = sqrt_pos(5.0 * r2);
        const double e = exp_neg(tmp);
        kval = (1.0 + tmp + div3_rn(tmp * tmp)) * e;
        gcommon = 5.0 / 3.0 * (tmp + 1.0) * e;
    } else if (COV == 1) {
        const double tmp = sqrt_pos(3.0 * r2);
        const double e = exp_neg(tmp);
        kval = (1.0 + tmp) * e;
        gcommon = 3.0 * e;
    } else {  // nu = 0.5: K * D / sqrt(sum D), 0 where the distance is 0
        const double den = sqrt(r2);
        kval = exp_neg(den);
        gcommon = (den != 0.0) ? kval / den : 0.0;
    }
}

// Tiled version for d <= LG_DMAX: one CTA per 64x64 patch on or below the diagonal (K^-1 and dK/dtheta are
// symmetric: pairs i > j count twice), each thread 16 pairs, per-theta sums kept in registers, ONE fixed-order
// block reduction per theta at the end.  part[patch][p]; the host adds the patches in index order.
constexpr int LG_DMAX = 16;
template <int COV, bool ANISO>
__global__ void __launch_bounds__(256)
lml_grad_tile_kernel(const double* __restrict__ Xs, const double* __restrict__ Kinv, int ldk,
                     const double* __restrict__ alphav, int n, int d, double constv, int has_const,
                     double* __restrict__ part, int ntheta) {
    const int bj = blockIdx.x, bi = blockIdx.y;
    if (bj > bi) return;
    // patch id in row-major order over the lower block triangle
    const int bid = bi * (bi + 1) / 2 + bj;
    __shared__ double xi[64][LG_DMAX + 1], xj[64][LG_DMAX + 1];
    __shared__ double ai[64], aj[64];
    __shared__ double red[8][LG_DMAX + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = bi * 64, j0 = bj * 64;
    for (int idx = tid; idx < 64 * d; idx += 256) {
        const int r = idx / d, t = idx - r * d;
        xi[r][t] = (i0 + r < n) ? Xs[(size_t)(i0 + r) * d + t] : 0.0;
        xj[r][t] = (j0 + r < n) ? Xs[(size_t)(j0 + r) * d + t] : 0.0;
    }
    if (tid < 64) {
        ai[tid] = (i0 + tid < n) ? alphav[i0 + tid] : 0.0;
        aj[tid] = (j0 + tid < n) ? alphav[j0 + tid] : 0.0;
    }
    __syncthreads();
    double acc_c = 0.0;
    double acc[ANISO ? LG_DMAX : 1];
#pragma unroll
    for (int t = 0; t < (ANISO ? LG_DMAX : 1); ++t) acc[t] = 0.0;
    const int cj = tid & 63;         // column of the patch (coalesced Kinv reads)
    const int r0 = (tid >> 6) * 16;  // 16 consecutive rows
    const int j = j0 + cj;
    for (int rr = 0; rr < 16; ++rr) {
        const int ri = r0 + rr, i = i0 + ri;
        if (i >= n || j >= n || j > i) continue;
        double w = ai[ri] * aj[cj] - Kinv[(size_t)i * ldk + j];
        if (i != j) w *= 2.0;
        double r2 = 0.0;
        double df2[ANISO ? LG_DMAX : 1];
#pragma unroll
        for (int t = 0; t < LG_DMAX; ++t) {
            if (t < d) {
                const double df = xi[ri][t] - xj[cj][t];
                const double q = df * df;
                r2 += q;
                if (ANISO) df2[t] = q;
            }
        }
        double kval, gcommon;
        cov_and_gradfactor<COV>(r2, kval, gcommon);
        if (i == j) kval = 1.0;
        acc_c = fma(w, constv * kval, acc_c);
        const double base = w * constv * gcommon;
        if (ANISO) {
#pragma unroll
            for (int t = 0; t < LG_DMAX; ++t)
                if (t < d) acc[t] = fma(base, df2[t], acc[t]);
        } else {
            acc[0] = fma(base, r2, acc[0]);
        }
    }
    // fixed-order reduction: lanes (butterfly), then the 8 warps in index order
    const int nls = ANISO ? d : 1;
    for (int q = 0; q <= nls; ++q) {
        double v = (q == 0) ? acc_c : 0.0;
        if (q > 0) {
#pragma unroll
            for (int t = 0; t < (ANISO ? LG_DMAX : 1); ++t)
                if (t == q - 1) v = acc[t];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][q] = v;
    }
    __syncthreads();
    if (tid <= nls) {
        double s = 0.0;
        for (int w8 = 0; w8 < 8; ++w8) s += red[w8][tid];
        // theta order: [log const (if has_const)], log length_scale...
        if (tid == 0) {
            if (has_const) part[(size_t)bid * ntheta] = 0.5 * s;
        } else {
            part[(size_t)bid * ntheta + (has_const ? 1 : 0) + tid - 1] = 0.5 * s;
        }
    }
}

__global__ void __launch_bounds__(256)
lml_grad_kernel(const double* __restrict__ Xs, const double* __restrict__ Kinv, int ldk,
                const double* __restrict__ alphav, int n, int d, int family, int nu, double constv,
                int has_const, int aniso, double* __restrict__ part, int ntheta) {
    const int j = blockIdx.x * 16 + (threadIdx.x & 15);
    const int i = blockIdx.y * 16 + (threadIdx.x >> 4);
    __shared__ double red[256];
    const int bid = blockIdx.y * gridDim.x + blockIdx.x;
    // K^-1 and dK/dtheta are symmetric: only pairs i >= j are visited (K^-1's upper tiles are never
    // computed) and off-diagonal pairs count twice
    const bool valid = (i < n && j < n && j <= i);
    double w = 0.0, r2 = 0.0, kval = 0.0, gcommon = 0.0;
    const double* a = Xs + (size_t)(valid ? i : 0) * d;
    const double* b = Xs + (size_t)(valid ? j : 0) * d;
    if (valid) {
        w = alphav[i] * alphav[j] - Kinv[(size_t)i * ldk + j];
        if (i != j) w *= 2.0;
        for (int t = 0; t < d; ++t) {
            const double df = a[t] - b[t];
            r2 += df * df;
        }
        kval = (i == j) ? 1.0 : cov_from_r2(r2, family, nu);
        // gradient factor such that dk/dlog(l_t) = gcommon * D_t  (D_t = scaled squared diff)
        if (family == B200BO_KERNEL_RBF || nu == B200BO_NU_INF) {
            gcommon = kval;  // K_gradient = D * K
        } else if (nu == B200BO_NU_25) {
            const double tmp = sqrt(5.0 * r2);
            gcommon = 5.0 / 3.0 * (tmp + 1.0) * exp(-tmp);
        } else if (nu == B200BO_NU_15) {
            gcommon = 3.0 * exp(-sqrt(3.0 * r2));
        } else {  // nu = 0.5: K * D / sqrt(sum D), 0 where the distance is 0
            const double den = sqrt(r2);
            gcommon = (den != 0.0) ? kval / den : 0.0;
        }
    }
    for (int p = 0; p < ntheta; ++p) {
        double g = 0.0;
        if (valid) {
            if (has_const && p == 0) {
                g = constv * kval;
            } else if (!aniso) {
                g = constv * gcommon * r2;
            } else {
                const int t = p - has_const;
                const double df = a[t] - b[t];
                g = constv * gcommon * (df * df);
            }
        }
        red[threadIdx.x] = w * g;
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) {
            if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
            __syncthreads();
        }
        if (threadIdx.x == 0) part[(size_t)bid * ntheta + p] = 0.5 * red[0];
        __syncthreads();
    }
}

}  // namespace b200bo
