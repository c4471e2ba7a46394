// b200bo.cu - C ABI (include/b200bo.h) over the sm_90a kernels.  No CPU fallback: every
// compute entry point needs a CUDA device and reports B200BO_ERR_CUDA without one.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <dlfcn.h>
#include <nccl.h>
#include <nvtx3/nvToolsExt.h>

#include "fit_kernels.cuh"
#include "paths.cuh"
#include "predict_kernels.cuh"
#include "predict16.cuh"

using namespace b200bo;

constexpr int kDefaultPredictWarps = 16;  // measured A/B (DESIGN.md 6): 550.1 ms vs 561.7 ms per 2^20 candidates at C3
constexpr float kDefaultLinvL2Last = 1.0f;  // evict_last fraction of the L^-1 loads (DESIGN.md 6)
// phase B data path of predict_acq16_kernel: bulk copies without clusters, 4-5 % above cp.async at C3 (DESIGN.md 6)
constexpr int kDefaultPredictPipe = PIPE_BULK;

// ---------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

static int set_err(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CU(call)                                                                              \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess)                                                               \
            return set_err(B200BO_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                  \
                           cudaGetErrorString(e__), __FILE__, __LINE__);                      \
    } while (0)

#define LAUNCHED() (g_launches.fetch_add(1, std::memory_order_relaxed))

// NVTX ranges around the phases of the path (fit / lml / predict_acq / select / exchange): visible in any
// NVTX-aware profiler, free otherwise (header-only NVTX3 resolves its injection library lazily).
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

// ---------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------
// A device allocation that grows on demand and is freed with its owner (on the device current at that point).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    int reserve(size_t bytes) {
        if (bytes <= cap) return B200BO_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess)
            return set_err(B200BO_ERR_CUDA, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        cap = bytes;
        return B200BO_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

// Streamed upload of a host candidate matrix: chunk i+1 goes up on `copy` while chunk i is evaluated on `exec`
// (double-buffered device chunks, ordered by events).  Shared by the acquisition and the sample-path entry points.
struct ChunkedUpload {
    cudaStream_t copy = nullptr, exec = nullptr;
    cudaEvent_t up[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr};
    int ensure();
    void release() {
        if (copy) cudaStreamDestroy(copy);
        if (exec) cudaStreamDestroy(exec);
        for (int i = 0; i < 2; ++i) {
            if (up[i]) cudaEventDestroy(up[i]);
            if (done[i]) cudaEventDestroy(done[i]);
        }
        copy = exec = nullptr;
        up[0] = up[1] = done[0] = done[1] = nullptr;
    }
    // launch(d_chunk, rows, first_row, chunk_number, is_last) issues the work of one chunk on `exec`;
    // buf: two device buffers of chunk x d doubles.  Returns with the work enqueued, not finished.
    template <class Launch>
    int run(const double* Xc, long long m, int d, long long chunk, double* const buf[2], Launch launch);
};

struct b200bo_gp {
    int device = 0;
    int sm_count = 0;
    int pair_grid = 0;  // CTAs of predict_acq16_kernel's clustered launch: 2 x max active clusters (0: not queried yet)
    bool pipe_armed = false;  // a bulk-copy phase B ran on this handle: its timeout flag is worth reading
    long long n = 0;
    int np = 0, d = 0;
    bool has_data = false, fitted = false;
    // kernel of the last fit
    int family = 0, nu = B200BO_NU_25;
    double constv = 1.0, jitter = 0.0;  // jitter = alpha + WhiteKernel noise_level (diagonal of K)
    double noise = 0.0;
    double y_mean = 0.0, y_std = 1.0;
    std::vector<double> y_norm;  // host copy of normalised targets (n)
    std::vector<double> y_raw;   // host copy of the raw targets (n)
    bool normalize = false;
    std::vector<int> xform;      // host copy (d) or empty
    std::vector<double> ystar;   // MES samples of the maximum (b200bo_gp_set_max_values), or empty
    // NEI fantasies (b200bo_gp_set_fantasies): A = K0^-1 F ([np][S]) then best_s on the device, and the host copy of
    // best_s (empty: no fantasies)
    DevBuf fant_a;
    std::vector<double> fant_best;
    // what pending rows need (b200bo_gp_condition_fantasies), [S][np] per sample: F (normalised) and the prior draws
    // Z of the rows; W = K^-1 R over the first fant_nreg (registered) rows, [S][fant_nreg]
    DevBuf fant_f, fant_z, fant_w;
    DevBuf fant_tmp;  // b200bo_gp_condition_fantasies: the S solves ([S][np]), then the z row (S)
    DevBuf fant_mask;  // b200bo_gp_set_constrained_incumbent: the in-bounds mask of the rows (n bytes)
    int fant_nreg = 0;
    DevBuf X, Xs, y, K, L, W, WT, T, alphav, v1, v2, ls, xf, info, part;
    DevBuf tscratch;  // b200bo_gp_condition: t = W^T l of the row update (np), so that alpha_ survives it
    // predict-side scratch (used when this handle is gps[0] of a call)
    DevBuf pscratch, xc, out_acq, out_mu, out_sd, sel, clamp;
    // small-batch path scratch (per GP) + work-unit tables (rebuilt when np changes)
    DevBuf s_ksm, s_partial, s_mupart, s_unit, s_rb, s_colsq;
    int s_np = 0, s_nunits = 0;
    // gradient calls (b200bo_acq_value_grad): v, u, the partials of the product with L^-T and of the gradient sums,
    // and the upper-triangular work-unit tables (rebuilt when np or d changes)
    DevBuf s_vsum, s_usum, s_partial_u, s_gpart, s_unit_u, s_rb_u, out_grad;
    int s_grad_np = 0, s_grad_d = 0, s_nunits_u = 0;
    // fp32 mode: L^-1 as tf32 (hi,lo) wgmma operand images (built on first use after a fit)
    DevBuf tc_linv;
    bool tc_valid = false;
    // bulk-copy phase B of the fp64 kernel: L^-1 as padded stage images (built on first use after a fit)
    DevBuf pad_linv;
    bool pad_valid = false;
    // Gram bound pass of pruning: the training-side operand, A1 and Ymax, alpha_ in fp32 (built on first use after a
    // fit), and the host copy of A1 the choice between the fp64 and the fp32 pass reads
    DevBuf gram;
    bool gram_valid = false;
    double gram_a1 = 0.0;
    DevBuf cov_xc, cov_kst, cov_v, cov_c, cov_out, cov_mu;  // predict(return_cov=True) scratch
    DevBuf sel_cta;         // per-CTA running selection lists of the fused kernels
    // selection-only pruning: bound keys / local indices (two buffers each for the radix sort), its temp storage and
    // the control words of predict_acq16_kernel's prune mode
    DevBuf prune_key, prune_idx, prune_tmp, prune_ctl;
    // its refine stages: the interval of K* alpha_ per candidate from the bound pass, the survivor list and its keys
    // (the refine stage's and the level's, the level's slots and the second buffers of their sort), the survivors'
    // carried prefixes, the per-row-block partials, K* alpha_ of the tiles and the arrival counters of
    // predict_units_kernel
    DevBuf prune_mu, prune_surv, prune_surv_key, prune_prefix, prune_part, prune_mu_unit, prune_arrive;
    // candidates of the last call (chunked: all chunks) and those of them evaluated outside the prune mode; the
    // prune mode counts its own in prune_ctl[2] (prune_counted)
    long long stat_total = 0, stat_direct = 0;
    bool prune_counted = false;
    // stage boundaries of the last pruned launch on its stream: after the bound pass, the sort, the lead, refine and
    // final stages, and after the refine level (b200bo_last_prune_stage_ms, b200bo_last_prune_levels; the stages start
    // at ev0 and the tile kernel ends at ev1)
    cudaEvent_t ev_stage[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    bool stage_timed = false, stage_refined = false;
    int coop_final[2] = {-1, -1};  // final_rounds_coop per DREG: -1 not yet checked, 0 no, 1 yes
    DevBuf pbounds, prow;   // throughput mode: Philox bounds (lo, span) / regenerated winner rows
    bool replica = false;   // predict-only copy made by b200bo_gp_replicate
    // look-ahead Cholesky: bulk stream, chain/bulk events, copy of the next diagonal step's panel block
    cudaStream_t bulk_stream = nullptr;
    cudaEvent_t ev_chain = nullptr, ev_bulk = nullptr;
    DevBuf pside;
    // CUDA graph of the theta-independent part of a factorisation (run_factor)
    cudaStream_t cap_stream = nullptr;
    cudaGraphExec_t fgraph_exec = nullptr;
    unsigned long long fgraph_key[16] = {0};
    long long fgraph_nodes = 0;
    // streamed host batches: copy / execute streams and the double-buffer events
    ChunkedUpload upload;
    int precision = B200BO_PRECISION_FP64;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // fit-side work (set_data / fit / lml) of this handle is issued on this stream: the legacy default
    // stream (nullptr) unless b200bo_gp_set_private_stream gave the handle its own, so that several
    // handles driven from different host threads factorise concurrently
    cudaStream_t stream = nullptr;
};

// stream of the fit-side entry point in flight on this thread
static thread_local cudaStream_t g_st = nullptr;
struct StreamScope {
    cudaStream_t prev;
    explicit StreamScope(const b200bo_gp* gp) : prev(g_st) { g_st = gp ? gp->stream : nullptr; }
    ~StreamScope() { g_st = prev; }
};

static thread_local b200bo_gp* g_last_timed = nullptr;

// wait for the fit-side stream (the whole device when it is the legacy default stream)
static int sync_fit_stream() {
    if (g_st)
        CU(cudaStreamSynchronize(g_st));
    else
        CU(cudaDeviceSynchronize());
    return B200BO_OK;
}
// host <-> device copies ordered in the fit-side stream; d2h returns with the data on the host
static int h2d(void* dst, const void* src, size_t bytes) {
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, g_st));
    return B200BO_OK;
}
static int d2h(void* dst, const void* src, size_t bytes) {
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, g_st));
    CU(cudaStreamSynchronize(g_st));
    return B200BO_OK;
}

static inline int round_up(long long v, int m) { return (int)(((v + m - 1) / m) * m); }

extern "C" int b200bo_version(void) { return B200BO_VERSION; }
extern "C" const char* b200bo_last_error(void) { return g_err; }
extern "C" int64_t b200bo_launch_count(void) { return g_launches.load(); }

extern "C" int b200bo_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

// dynamic shared memory of the register-fragment fp32 Gram pass, every k-step count of d <= kGramRegMaxDim
template <int COV>
static cudaError_t gram_reg_attrs() {
    constexpr int attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
    const int smem = (int)gram_reg_bound_smem(kGramRegMaxDim);
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(predict_bound_gram_reg_kernel<COV, 1>, (cudaFuncAttribute)attr, smem))) return e;
    if ((e = cudaFuncSetAttribute(predict_bound_gram_reg_kernel<COV, 2>, (cudaFuncAttribute)attr, smem))) return e;
    if ((e = cudaFuncSetAttribute(predict_bound_gram_reg_kernel<COV, 3>, (cudaFuncAttribute)attr, smem))) return e;
    if ((e = cudaFuncSetAttribute(predict_bound_gram_reg_kernel<COV, 4>, (cudaFuncAttribute)attr, smem))) return e;
    return cudaFuncSetAttribute(predict_bound_gram_reg_kernel<COV, 5>, (cudaFuncAttribute)attr, smem);
}

// device properties, timing events and the opt-in shared-memory sizes of the big kernels
static int init_handle(b200bo_gp* gp) {
    CU(cudaDeviceGetAttribute(&gp->sm_count, cudaDevAttrMultiProcessorCount, gp->device));
    CU(cudaEventCreate(&gp->ev0));
    CU(cudaEventCreate(&gp->ev1));
    for (cudaEvent_t& e : gp->ev_stage) CU(cudaEventCreate(&e));
    CU(cudaFuncSetAttribute(predict_acq_kernel<PREDICT_IMPL_DFMA, false>,
                            cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_acq_kernel<PREDICT_IMPL_DFMA, true>,
                            cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_acq_kernel<PREDICT_IMPL_DMMA, false>,
                            cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq_kernel<PREDICT_IMPL_DMMA, true>,
                            cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(potrf_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            kPotrfSmemBytes));
    CU(cudaFuncSetAttribute(potrf_diag_legacy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            kPotrfLegacySmemBytes));
    CU(cudaFuncSetAttribute(predict_acq_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            kPredictSmemBytesTc));
    CU(cudaFuncSetAttribute(predict_acq_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            kPredictSmemBytesTc));
    CU(cudaFuncSetAttribute(small_trsv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmallTrsvSmemBytes));
    CU(cudaFuncSetAttribute(small_trsv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmallTrsvSmemBytes));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 884, PIPE_CPASYNC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 884, PIPE_CPASYNC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_CPASYNC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_CPASYNC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK_MC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK_MC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    // the NEI / LogNEI instantiations
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK_MC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK_MC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    // the CNEI / LogCNEI instantiations
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<true, 1684, PIPE_BULK_MC, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_acq16_kernel<false, 1684, PIPE_BULK_MC, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_bound_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_bound_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_mean_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_mean_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDfma));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(cudaFuncSetAttribute(predict_bound_gram_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gram_bound_smem(B200BO_MAX_DIM)));
    CU(gram_reg_attrs<1>());
    CU(gram_reg_attrs<2>());
    CU(gram_reg_attrs<3>());
    CU(cudaFuncSetAttribute(predict_refine_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_refine_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(predict_units_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(ks_build_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(ks_build_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(final_rounds_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(final_rounds_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPredictSmemBytesDmma));
    CU(cudaFuncSetAttribute(trailing_update64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTrailSmemBytes));
    CU(cudaFuncSetAttribute(dgemm128_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemm128SmemBytes));
    CU(cudaFuncSetAttribute(dgemm128_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemm128SmemBytes));
    CU(cudaFuncSetAttribute(dgemm128_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemm128SmemBytes));
    return B200BO_OK;
}

extern "C" int b200bo_gp_create(b200bo_gp** out, int device) {
    if (!out) return set_err(B200BO_ERR_ARG, "out is NULL");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return set_err(B200BO_ERR_CUDA,
                       "no CUDA device available (%s); this engine has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= ndev) return set_err(B200BO_ERR_ARG, "device %d out of range", device);
    CU(cudaSetDevice(device));
    b200bo_gp* gp = new b200bo_gp();
    gp->device = device;
    const int rc = init_handle(gp);
    if (rc != B200BO_OK) {
        b200bo_gp_destroy(gp);
        return rc;
    }
    *out = gp;
    return B200BO_OK;
}

extern "C" void b200bo_gp_destroy(b200bo_gp* gp) {
    if (!gp) return;
    cudaSetDevice(gp->device);  // the buffers are freed by delete, on this device
    if (gp->stream) cudaStreamDestroy(gp->stream);
    if (gp->fgraph_exec) cudaGraphExecDestroy(gp->fgraph_exec);
    if (gp->cap_stream) cudaStreamDestroy(gp->cap_stream);
    if (gp->bulk_stream) cudaStreamDestroy(gp->bulk_stream);
    if (gp->ev_chain) cudaEventDestroy(gp->ev_chain);
    if (gp->ev_bulk) cudaEventDestroy(gp->ev_bulk);
    gp->upload.release();
    if (gp->ev0) cudaEventDestroy(gp->ev0);
    if (gp->ev1) cudaEventDestroy(gp->ev1);
    for (cudaEvent_t e : gp->ev_stage)
        if (e) cudaEventDestroy(e);
    if (g_last_timed == gp) g_last_timed = nullptr;
    delete gp;
}

extern "C" int64_t b200bo_gp_n(const b200bo_gp* gp) { return gp ? gp->n : 0; }
extern "C" int b200bo_gp_dim(const b200bo_gp* gp) { return gp ? gp->d : 0; }

extern "C" int b200bo_gp_set_precision(b200bo_gp* gp, int precision) {
    if (!gp) return set_err(B200BO_ERR_ARG, "gp is NULL");
    if (precision != B200BO_PRECISION_FP64 && precision != B200BO_PRECISION_FP32)
        return set_err(B200BO_ERR_ARG, "unknown precision %d", precision);
    gp->precision = precision;
    return B200BO_OK;
}

extern "C" int b200bo_gp_set_private_stream(b200bo_gp* gp, int enable) {
    if (!gp) return set_err(B200BO_ERR_ARG, "gp is NULL");
    CU(cudaSetDevice(gp->device));
    if (enable && !gp->stream) {
        CU(cudaStreamCreate(&gp->stream));  // a blocking stream: still ordered against legacy-stream work
    } else if (!enable && gp->stream) {
        CU(cudaStreamSynchronize(gp->stream));
        CU(cudaStreamDestroy(gp->stream));
        gp->stream = nullptr;
    }
    return B200BO_OK;
}

extern "C" int b200bo_gp_set_transform(b200bo_gp* gp, const int32_t* xform, int d) {
    if (!gp) return set_err(B200BO_ERR_ARG, "gp is NULL");
    gp->xform.clear();
    if (xform) {
        if (d <= 0 || d > B200BO_MAX_DIM) return set_err(B200BO_ERR_ARG, "bad d=%d", d);
        for (int j = 0; j < d; ++j) {
            if (xform[j] != B200BO_XFORM_IDENTITY && xform[j] != B200BO_XFORM_ROUND)
                return set_err(B200BO_ERR_UNSUPPORTED, "transform code %d unsupported", xform[j]);
            gp->xform.push_back(xform[j]);
        }
    }
    gp->fitted = false;
    gp->fant_best.clear();
    return B200BO_OK;
}

extern "C" int b200bo_gp_set_max_values(b200bo_gp* gp, const double* ystar, int K) {
    if (!gp) return set_err(B200BO_ERR_ARG, "gp is NULL");
    if (K < 0 || K > B200BO_MAX_PATHS) return set_err(B200BO_ERR_ARG, "K=%d out of range [0,%d]", K, B200BO_MAX_PATHS);
    if (K > 0 && !ystar) return set_err(B200BO_ERR_ARG, "ystar is NULL");
    for (int k = 0; k < K; ++k)
        if (!std::isfinite(ystar[k])) return set_err(B200BO_ERR_ARG, "ystar[%d] is not finite", k);
    gp->ystar.assign(ystar, ystar + K);
    return B200BO_OK;
}

// ---------------------------------------------------------------------------------------
// data upload + y normalisation (SK/gaussian_process/_gpr.py:275-285)
// ---------------------------------------------------------------------------------------
// y_norm, y_mean and y_std of gp->y_raw under gp->normalize.  y statistics in the order numpy uses for small arrays
// is irrelevant at 1e-16; use a compensated sum so the result is the correctly rounded mean / population std.
static void normalize_targets(b200bo_gp* gp) {
    const std::vector<double>& y = gp->y_raw;
    const size_t n = y.size();
    double mean = 0.0, sd = 1.0;
    gp->y_norm = y;
    if (gp->normalize) {
        long double s = 0.0L;
        for (size_t i = 0; i < n; ++i) s += y[i];
        mean = (double)(s / (long double)n);
        long double q = 0.0L;
        for (size_t i = 0; i < n; ++i) {
            const long double t = (long double)y[i] - (long double)mean;
            q += t * t;
        }
        sd = (double)sqrtl(q / (long double)n);
        if (sd == 0.0) sd = 1.0;
        for (size_t i = 0; i < n; ++i) gp->y_norm[i] = (y[i] - mean) / sd;
    }
    gp->y_mean = mean;
    gp->y_std = sd;
}

extern "C" int b200bo_gp_set_data(b200bo_gp* gp, const double* X, const double* y, int64_t n, int d,
                                  int normalize_y) {
    if (!gp || !X || !y) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (n <= 0 || d <= 0 || d > B200BO_MAX_DIM)
        return set_err(B200BO_ERR_ARG, "bad shape n=%lld d=%d (d <= %d)", (long long)n, d, B200BO_MAX_DIM);
    // five np x np fp64 matrices (K, L, L^-1, its transpose, workspace) + the fp32-mode images of L^-1:
    // about 44 np^2 bytes, 64 GB at the limit - what an 80 GB H100 holds beside the candidate batches
    if (n > 38000) return set_err(B200BO_ERR_ARG, "n=%lld too large (n <= 38000)", (long long)n);
    if (!gp->xform.empty() && (int)gp->xform.size() != d)
        return set_err(B200BO_ERR_ARG, "transform has %zu entries, d=%d", gp->xform.size(), d);
    CU(cudaSetDevice(gp->device));
    StreamScope scope(gp);
    gp->fitted = false;
    gp->fant_best.clear();
    gp->replica = false;
    gp->tc_valid = false;
    gp->pad_valid = false;
    gp->gram_valid = false;
    gp->n = n;
    gp->d = d;
    gp->np = round_up(n, kPad);
    const size_t np = gp->np;
    gp->y_raw.assign(y, y + n);
    gp->normalize = normalize_y != 0;
    normalize_targets(gp);
    int rc;
    if ((rc = gp->X.reserve(sizeof(double) * np * d))) return rc;
    if ((rc = gp->Xs.reserve(sizeof(double) * np * d))) return rc;
    if ((rc = gp->y.reserve(sizeof(double) * np))) return rc;
    if ((rc = gp->alphav.reserve(sizeof(double) * np))) return rc;
    if ((rc = gp->v1.reserve(sizeof(double) * np))) return rc;
    if ((rc = gp->v2.reserve(sizeof(double) * np))) return rc;
    if ((rc = gp->ls.reserve(sizeof(double) * B200BO_MAX_DIM))) return rc;
    if ((rc = gp->xf.reserve(sizeof(int) * B200BO_MAX_DIM))) return rc;
    if ((rc = gp->info.reserve(sizeof(int)))) return rc;
    if ((rc = gp->part.reserve(sizeof(double) * 64))) return rc;
    if ((rc = gp->K.reserve(sizeof(double) * np * np))) return rc;
    if ((rc = gp->L.reserve(sizeof(double) * np * np))) return rc;
    if ((rc = gp->W.reserve(sizeof(double) * np * np))) return rc;
    if ((rc = gp->WT.reserve(sizeof(double) * np * np))) return rc;
    if ((rc = gp->T.reserve(sizeof(double) * np * np))) return rc;
    if ((rc = h2d(gp->X.p, X, sizeof(double) * n * d))) return rc;
    CU(cudaMemsetAsync(gp->y.p, 0, sizeof(double) * np, g_st));
    if ((rc = h2d(gp->y.p, gp->y_norm.data(), sizeof(double) * n))) return rc;
    if (!gp->xform.empty() && (rc = h2d(gp->xf.p, gp->xform.data(), sizeof(int) * d))) return rc;
    if ((rc = sync_fit_stream())) return rc;  // the caller may release X / y on return
    gp->has_data = true;
    return B200BO_OK;
}

static int check_kernel(const b200bo_gp* gp, const b200bo_kernel* k) {
    if (!k || !k->length_scale) return set_err(B200BO_ERR_ARG, "kernel/length_scale is NULL");
    if (k->family != B200BO_KERNEL_MATERN && k->family != B200BO_KERNEL_RBF)
        return set_err(B200BO_ERR_UNSUPPORTED, "kernel family %d unsupported", k->family);
    if (k->family == B200BO_KERNEL_MATERN && (k->nu < B200BO_NU_05 || k->nu > B200BO_NU_INF))
        return set_err(B200BO_ERR_UNSUPPORTED, "Matern nu code %d unsupported", k->nu);
    if (k->n_length_scale != 1 && k->n_length_scale != gp->d)
        return set_err(B200BO_ERR_ARG, "n_length_scale=%d must be 1 or d=%d", k->n_length_scale, gp->d);
    for (int j = 0; j < k->n_length_scale; ++j)
        if (!(k->length_scale[j] > 0.0)) return set_err(B200BO_ERR_ARG, "length_scale must be > 0");
    if (!(k->const_value > 0.0)) return set_err(B200BO_ERR_ARG, "const_value must be > 0");
    if (!(k->noise_level >= 0.0)) return set_err(B200BO_ERR_ARG, "noise_level must be >= 0");
    return B200BO_OK;
}

static int potrf_mode() {  // 0 look-ahead (default), 1 serial blocked, 2 legacy unblocked
    const char* pv = getenv("B200BO_POTRF");
    if (pv && (pv[0] == 'l' || pv[0] == 'L')) return 2;
    if (pv && (pv[0] == 's' || pv[0] == 'S')) return 1;
    return 0;
}
static int trail_kernel() {  // 1: 64x128 tiles, 2 CTAs/SM (default); 0: the generic 128x128 GEMM (B200BO_TRAIL=gemm)
    const char* e = getenv("B200BO_TRAIL");
    return (e && e[0] == 'g') ? 0 : 1;
}
static bool gemm_force64() {
    const char* e = getenv("B200BO_GEMM");
    return e && e[0] == '6';
}

static int ensure_bulk_stream(b200bo_gp* gp) {
    if (!gp->bulk_stream) {
        CU(cudaStreamCreateWithFlags(&gp->bulk_stream, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&gp->ev_chain, cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&gp->ev_bulk, cudaEventDisableTiming));
    }
    return B200BO_OK;
}

template <bool TA, bool TB>
static int gemm(int M, int N, int K, double alpha, const double* A, int lda, long long sA,
                const double* B, int ldb, long long sB, double beta, double* C, int ldc,
                long long sC, int batch, int lower_only, int kmode, int skip = 0, const cudaStream_t* stp = nullptr,
                double* side = nullptr) {
    if (M <= 0 || N <= 0 || K <= 0 || batch <= 0) return B200BO_OK;
    const cudaStream_t st = stp ? *stp : g_st;
    // 128x128 pipelined tiles wherever a tile can be filled; the 64x64 kernel for narrow panels / small blocks
    if (M >= 128 && N >= 128 && !gemm_force64()) {
        dim3 grid((N + 127) / 128, (M + 127) / 128, batch);
        dgemm128_kernel<TA, TB><<<grid, 256, kGemm128SmemBytes, st>>>(M, N, K, alpha, A, lda, sA, B, ldb, sB, beta,
                                                                      C, ldc, sC, lower_only, kmode, skip, side);
    } else {
        dim3 grid(N / 64, M / 64, batch);
        dgemm64_kernel<TA, TB><<<grid, 256, 0, st>>>(M, N, K, alpha, A, lda, sA, B, ldb, sB, beta, C, ldc, sC,
                                                     lower_only, kmode, skip);
    }
    LAUNCHED();
    CU(cudaGetLastError());
    return B200BO_OK;
}

// K build + Cholesky + explicit triangular inverse.  On return L holds the clean lower factor,
// W = L^-1 (lower).  *info_out = 0 or the failing pivot (1-based).
static int transpose_W(b200bo_gp* gp);
static int solve_alpha(b200bo_gp* gp);

// Everything of a factorisation whose kernel ARGUMENTS do not depend on the hyper-parameters: K -> L, blocked
// Cholesky, zeroing of the upper triangle, L^-1 by recursive doubling, its transpose, alpha_ = K^-1 y.  Issued on g_st
// (+ the bulk stream of the look-ahead); no host synchronisation, no allocation: the sequence is CUDA-graph capturable.
// A non-positive pivot is replaced by 1 inside the diagonal kernel (arithmetic stays finite) and reported through
// gp->info, which the caller reads afterwards.
static int factor_body(b200bo_gp* gp) {
    const int np = gp->np;
    int rc;
    double* L = gp->L.as<double>();
    double* W = gp->W.as<double>();
    double* T = gp->T.as<double>();
    CU(cudaMemcpyAsync(L, gp->K.p, sizeof(double) * (size_t)np * np, cudaMemcpyDeviceToDevice, g_st));
    CU(cudaMemsetAsync(W, 0, sizeof(double) * (size_t)np * np, g_st));
    CU(cudaMemsetAsync(gp->info.p, 0, sizeof(int), g_st));
    // right-looking blocked Cholesky, panel width 64.  B200BO_POTRF=legacy selects the first
    // (unblocked) diagonal-block kernel, B200BO_POTRF=serial the blocked kernel without look-ahead, for A/B
    // measurements.
    // B200BO_GEMM=64 takes the serial loop too: the look-ahead needs the side store of A[j+2, j+1] that only the
    // 128-tile trailing update writes, and with 64-tile GEMMs the next diagonal block read a stale copy of it.
    const bool legacy_potrf = potrf_mode() == 2, serial_potrf = potrf_mode() == 1;
    if (legacy_potrf || serial_potrf || gemm_force64() || np <= 128) {
        for (int j0 = 0; j0 < np; j0 += 64) {
            if (legacy_potrf)
                potrf_diag_legacy_kernel<<<1, 256, kPotrfLegacySmemBytes, g_st>>>(L, np, j0, W + (size_t)j0 * np + j0, np,
                                                                            gp->info.as<int>());
            else
                potrf_diag_kernel<<<1, 256, kPotrfSmemBytes, g_st>>>(L, np, j0, W + (size_t)j0 * np + j0, np,
                                                               gp->info.as<int>(), nullptr, nullptr, 0);
            LAUNCHED();
            const int below = np - j0 - 64;
            if (below > 0) {
                double* panel = L + (size_t)(j0 + 64) * np + j0;
                // L_ij = A_ij * inv(L_jj)^T
                if ((rc = gemm<false, true>(below, 64, 64, 1.0, panel, np, 0, W + (size_t)j0 * np + j0, np, 0,
                                            0.0, panel, np, 0, 1, 0, 0)))
                    return rc;
                // trailing update (lower tiles only): A_ik -= L_ij L_kj^T
                if ((rc = gemm<false, true>(below, below, 64, -1.0, panel, np, 0, panel, np, 0, 1.0,
                                            L + (size_t)(j0 + 64) * np + j0 + 64, np, 0, 1, 1, 0)))
                    return rc;
            }
        }
    } else {
        // Look-ahead: the 64 diagonal blocks are a dependent chain of single-CTA kernels; everything else of a
        // step (panel solve, trailing update) is bulk work for the whole GPU.  The chain runs on the handle's
        // stream, the bulk on a second stream; the diagonal kernel of step j+1 resolves its dependence on
        // panel j itself (potrf_diag_kernel, look-ahead form) from a copy of A[j+1, j] taken before the bulk
        // panel solve, and the bulk trailing update leaves block (j+1, j+1) alone.  Every value is produced by
        // exactly one kernel: the result does not depend on how the two streams interleave.
        const cudaStream_t sb = gp->bulk_stream;
        // A[j+1, j] as it is BEFORE the bulk panel solve of panel j overwrites it in place: produced by the trailing
        // update of panel j-1 (its epilogue stores that block a second time, densely), double-buffered by step parity
        double* Pside[2] = {gp->pside.as<double>(), gp->pside.as<double>() + 64 * 64};
        CU(cudaEventRecord(gp->ev_chain, g_st));
        CU(cudaStreamWaitEvent(sb, gp->ev_chain, 0));  // K build / copies issued so far
        copy_block64_kernel<<<1, 256, 0, sb>>>(L + (size_t)64 * np, np, Pside[1]);  // A[1, 0]: no earlier panel touches it
        LAUNCHED();
        CU(cudaEventRecord(gp->ev_bulk, sb));
        potrf_diag_kernel<<<1, 256, kPotrfSmemBytes, g_st>>>(L, np, 0, W, np, gp->info.as<int>(), nullptr, nullptr, 0);
        LAUNCHED();
        CU(cudaEventRecord(gp->ev_chain, g_st));
        for (int j0 = 0, j = 0; j0 + 64 < np; j0 += 64, ++j) {
            const int below = np - j0 - 64;
            double* panel = L + (size_t)(j0 + 64) * np + j0;  // rows below the diagonal block, columns of panel j
            const double* Dj = W + (size_t)j0 * np + j0;
            // chain: diagonal block j+1.  Its inputs: Pside[(j+1)&1] (written by the trailing update of panel j-1, or the
            // initial copy) and A[j+1, j+1] with the updates of panels < j - both complete when ev_bulk (recorded after
            // that trailing update) has fired; inv(L_jj) comes from the previous kernel of this stream.
            CU(cudaStreamWaitEvent(g_st, gp->ev_bulk, 0));
            potrf_diag_kernel<<<1, 256, kPotrfSmemBytes, g_st>>>(L, np, j0 + 64, W + (size_t)(j0 + 64) * np + j0 + 64, np,
                                                           gp->info.as<int>(), Pside[(j + 1) & 1], Dj, np);
            LAUNCHED();
            // bulk: panel solve (needs inv(L_jj): ev_chain of the PREVIOUS chain kernel), then the trailing update of
            // panel j on everything but block (j+1, j+1); it also leaves A[j+2, j+1] in Pside[j&1] for the next step
            CU(cudaStreamWaitEvent(sb, gp->ev_chain, 0));
            CU(cudaEventRecord(gp->ev_chain, g_st));  // re-recorded AFTER the wait above was enqueued: now marks step j+1
            if ((rc = gemm<false, true>(below, 64, 64, 1.0, panel, np, 0, Dj, np, 0, 0.0, panel, np, 0, 1, 0, 0, 0, &sb)))
                return rc;
            if (below >= 1024 && !gemm_force64() && trail_kernel() == 1) {  // large updates only: measured no gain below
                dim3 grid((below + 127) / 128, below / 64);
                trailing_update64_kernel<<<grid, 256, kTrailSmemBytes, sb>>>(below, panel, np, L + (size_t)(j0 + 64) * np + j0 + 64,
                                                                            np, 64, Pside[j & 1]);
                LAUNCHED();
                CU(cudaGetLastError());
            } else if ((rc = gemm<false, true>(below, below, 64, -1.0, panel, np, 0, panel, np, 0, 1.0,
                                               L + (size_t)(j0 + 64) * np + j0 + 64, np, 0, 1, 1, 0, 64, &sb, Pside[j & 1])))
                return rc;
            CU(cudaEventRecord(gp->ev_bulk, sb));
        }
        CU(cudaEventRecord(gp->ev_bulk, sb));
        CU(cudaStreamWaitEvent(g_st, gp->ev_bulk, 0));
    }
    {
        dim3 blk(32, 8), grd((np + 31) / 32, (np + 7) / 8);
        zero_upper_kernel<<<grd, blk, 0, g_st>>>(L, np);
        LAUNCHED();
    }
    // W = L^-1 by recursive doubling over diagonal blocks:
    //   inv([[A,0],[C,B]]) = [[A^-1,0],[-B^-1 C A^-1, B^-1]]
    for (int s = 64; s < np; s *= 2) {
        const int full = np / (2 * s);
        const int rem = np % (2 * s);
        const long long stride = (long long)2 * s * ((long long)np + 1);
        if (full > 0) {
            // T = C * A^-1      (A^-1 lower-triangular: k >= n0)
            if ((rc = gemm<false, false>(s, s, s, 1.0, L + (size_t)s * np, np, stride, W, np, stride, 0.0,
                                         T + (size_t)s * np, np, stride, full, 0, 2)))
                return rc;
            // W21 = -B^-1 * T   (B^-1 lower-triangular: k < m0 + 64)
            if ((rc = gemm<false, false>(s, s, s, -1.0, W + (size_t)s * np + s, np, stride,
                                         T + (size_t)s * np, np, stride, 0.0, W + (size_t)s * np, np,
                                         stride, full, 0, 1)))
                return rc;
        }
        if (rem > s) {
            const int m2 = rem - s;
            const size_t o = (size_t)full * 2 * s;
            const double* C = L + (o + s) * np + o;
            double* Tt = T + (o + s) * np + o;
            if ((rc = gemm<false, false>(m2, s, s, 1.0, C, np, 0, W + o * np + o, np, 0, 0.0, Tt, np, 0, 1,
                                         0, 2)))
                return rc;
            if ((rc = gemm<false, false>(m2, s, m2, -1.0, W + (o + s) * np + o + s, np, 0, Tt, np, 0, 0.0,
                                         W + (o + s) * np + o, np, 0, 1, 0, 1)))
                return rc;
        }
    }
    CU(cudaGetLastError());
    if ((rc = transpose_W(gp))) return rc;
    return solve_alpha(gp);
}


// One LML evaluation is ~350 dependent launches and ~250 event operations: issued one by one the HOST is the
// bottleneck (2-3 us per call, the kernels of a 64-wide step are shorter than that).  The sequence has the same
// arguments whatever theta is, so it is captured ONCE per handle and training-set size into a CUDA graph (both
// streams of the look-ahead join the capture) and replayed with one call.  B200BO_GRAPH=0 issues it directly.
static int run_factor(b200bo_gp* gp) {
    int rc;
    if ((rc = ensure_bulk_stream(gp))) return rc;
    if ((rc = gp->pside.reserve(sizeof(double) * 2 * 64 * 64))) return rc;
    // graphs pay off where the launch-by-launch host cost matters (measured: N=4096 5.70 vs 5.92 ms; N=1024 no gain) and
    // cost a capture + instantiation per handle and size: used from np >= 2048 (B200BO_GRAPH=0 never, =1 always)
    const char* ge = getenv("B200BO_GRAPH");
    if ((ge && ge[0] == '0') || (!(ge && ge[0] == '1') && gp->np < 2048)) return factor_body(gp);
    const unsigned long long key[] = {(unsigned long long)gp->np, (unsigned long long)gp->K.p, (unsigned long long)gp->L.p,
                                      (unsigned long long)gp->W.p, (unsigned long long)gp->WT.p, (unsigned long long)gp->T.p,
                                      (unsigned long long)gp->alphav.p, (unsigned long long)gp->y.p, (unsigned long long)gp->v1.p,
                                      (unsigned long long)gp->v2.p, (unsigned long long)gp->info.p, (unsigned long long)gp->pside.p,
                                      (unsigned long long)(potrf_mode() * 4 + trail_kernel() * 2 + (gemm_force64() ? 1 : 0))};
    constexpr int NKEY = sizeof(key) / sizeof(key[0]);
    if (!gp->fgraph_exec || memcmp(key, gp->fgraph_key, sizeof(key)) != 0) {
        if (gp->fgraph_exec) {
            cudaGraphExecDestroy(gp->fgraph_exec);
            gp->fgraph_exec = nullptr;
        }
        if (!gp->cap_stream) CU(cudaStreamCreateWithFlags(&gp->cap_stream, cudaStreamNonBlocking));
        const long long before = g_launches.load();
        cudaStream_t saved = g_st;
        g_st = gp->cap_stream;
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamBeginCapture(gp->cap_stream, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            rc = factor_body(gp);
            e = cudaStreamEndCapture(gp->cap_stream, &graph);
            if (rc == B200BO_OK && e == cudaSuccess) e = cudaGraphInstantiate(&gp->fgraph_exec, graph, 0);
            if (graph) cudaGraphDestroy(graph);
        }
        g_st = saved;
        gp->fgraph_nodes = g_launches.load() - before;
        g_launches.store(before);  // nothing ran during the capture
        if (rc != B200BO_OK || e != cudaSuccess || !gp->fgraph_exec) {
            cudaGetLastError();
            gp->fgraph_exec = nullptr;
            static bool warned = false;
            if (!warned) {
                warned = true;
                fprintf(stderr, "b200bo: CUDA-graph capture of the factorisation failed (%s); issuing the launches directly\n",
                        e != cudaSuccess ? cudaGetErrorString(e) : g_err);
            }
            return factor_body(gp);
        }
        static_assert(NKEY <= 16, "key");
        memcpy(gp->fgraph_key, key, sizeof(key));
    }
    CU(cudaGraphLaunch(gp->fgraph_exec, g_st));
    g_launches.fetch_add(gp->fgraph_nodes, std::memory_order_relaxed);
    return B200BO_OK;
}

// K build + Cholesky + explicit triangular inverse + alpha_.  On return L holds the clean lower factor,
// W = L^-1 (lower), WT its transpose.  *info_out = 0 or the failing pivot (1-based).
static int factorize(b200bo_gp* gp, const b200bo_kernel* kern, double jitter, int* info_out) {
    const int n = (int)gp->n, np = gp->np, d = gp->d;
    double ls[B200BO_MAX_DIM];
    for (int j = 0; j < d; ++j) ls[j] = kern->length_scale[kern->n_length_scale == 1 ? 0 : j];
    int rc;
    if ((rc = h2d(gp->ls.p, ls, sizeof(double) * d))) return rc;
    const int* xf = gp->xform.empty() ? nullptr : gp->xf.as<int>();
    {
        const long long tot = (long long)np * d;
        scale_x_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, g_st>>>(gp->X.as<double>(), gp->ls.as<double>(), xf,
                                                               gp->Xs.as<double>(), n, np, d);
        LAUNCHED();
    }
    {
        dim3 blk(32, 8), grd(np / 32, np / 32);
        double* Kp = gp->K.as<double>();
        const double* Xsp = gp->Xs.as<double>();
        switch (cov_code(kern->family, kern->nu)) {
            case 0: kbuild_kernel<0><<<grd, blk, 0, g_st>>>(Xsp, Kp, n, np, d, kern->const_value, jitter); break;
            case 1: kbuild_kernel<1><<<grd, blk, 0, g_st>>>(Xsp, Kp, n, np, d, kern->const_value, jitter); break;
            case 2: kbuild_kernel<2><<<grd, blk, 0, g_st>>>(Xsp, Kp, n, np, d, kern->const_value, jitter); break;
            default: kbuild_kernel<3><<<grd, blk, 0, g_st>>>(Xsp, Kp, n, np, d, kern->const_value, jitter); break;
        }
        LAUNCHED();
    }
    CU(cudaGetLastError());
    if ((rc = run_factor(gp))) return rc;
    int info = 0;
    if ((rc = d2h(&info, gp->info.p, sizeof(int)))) return rc;
    *info_out = info;
    return B200BO_OK;
}

static int transpose_W(b200bo_gp* gp) {
    const int np = gp->np;
    dim3 blk(32, 8), grd(np / 32, np / 32);
    transpose_kernel<<<grd, blk, 0, g_st>>>(gp->W.as<double>(), gp->WT.as<double>(), np);
    LAUNCHED();
    CU(cudaGetLastError());
    return B200BO_OK;
}

// a = K^-1 y via the explicit inverse factors + one step of iterative refinement.  y, a: np entries (y zero
// padded); v1, v2: np-entry scratch.  alpha_ (solve_alpha) and the per-path solves of b200bo_paths_create.
static int solve_spd(b200bo_gp* gp, const double* y, double* a, double* v1, double* v2) {
    const int np = gp->np;
    const int wpb = 8;  // warps per block
    dim3 blk(32 * wpb), grd((np + wpb - 1) / wpb);
    // z = W y ; a = W^T z
    gemv_rows_kernel<<<grd, blk, 0, g_st>>>(gp->W.as<double>(), np, y, v1, np, np, 1);
    gemv_rows_kernel<<<grd, blk, 0, g_st>>>(gp->WT.as<double>(), np, v1, a, np, np, 2);
    // r = y - K a ; a += W^T W r
    gemv_rows_kernel<<<grd, blk, 0, g_st>>>(gp->K.as<double>(), np, a, v1, np, np, 0);
    residual_kernel<<<(np + 255) / 256, 256, 0, g_st>>>(y, v1, np);
    gemv_rows_kernel<<<grd, blk, 0, g_st>>>(gp->W.as<double>(), np, v1, v2, np, np, 1);
    gemv_rows_kernel<<<grd, blk, 0, g_st>>>(gp->WT.as<double>(), np, v2, v1, np, np, 2);
    axpy1_kernel<<<(np + 255) / 256, 256, 0, g_st>>>(a, v1, np);
    for (int i = 0; i < 7; ++i) LAUNCHED();
    CU(cudaGetLastError());
    return B200BO_OK;
}

// alpha_ = K^-1 y
static int solve_alpha(b200bo_gp* gp) {
    return solve_spd(gp, gp->y.as<double>(), gp->alphav.as<double>(), gp->v1.as<double>(), gp->v2.as<double>());
}

extern "C" int b200bo_gp_fit(b200bo_gp* gp, const double* X, const double* y, int64_t n, int d,
                             const b200bo_kernel* kern, double alpha, int normalize_y, int64_t* info) {
    int rc;
    if ((rc = b200bo_gp_set_data(gp, X, y, n, d, normalize_y))) return rc;
    if ((rc = check_kernel(gp, kern))) return rc;
    StreamScope scope(gp);
    NvtxRange nvtx_range("b200bo:fit");
    if (info) *info = 0;
    int finfo = 0;
    if ((rc = factorize(gp, kern, alpha + kern->noise_level, &finfo))) return rc;
    if (finfo != 0) {
        if (info) *info = finfo;
        return set_err(B200BO_ERR_NOT_PD, "%d-th leading minor of the array is not positive definite", finfo);
    }
    if ((rc = sync_fit_stream())) return rc;
    gp->family = kern->family;
    gp->nu = kern->family == B200BO_KERNEL_RBF ? B200BO_NU_INF : kern->nu;
    gp->constv = kern->const_value;
    gp->jitter = alpha + kern->noise_level;
    gp->noise = kern->noise_level;
    gp->fitted = true;
    return B200BO_OK;
}

// NEI fantasies (include/b200bo.h, DESIGN.md 4.13): per sample s one product with L0 and the solves with K and K0 on
// the device; the O(n) combinations on the host, in double, in the order of the definition.
extern "C" int b200bo_gp_set_fantasies(b200bo_gp* nl, const b200bo_gp* ny, const double* z, const double* e, int S,
                                       const uint8_t* incumbent, double* f_out, double* best_out) {
    if (!nl || !ny || !z || !e || !incumbent) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (S < 1 || S > B200BO_MAX_PATHS) return set_err(B200BO_ERR_ARG, "S=%d out of range [1,%d]", S, B200BO_MAX_PATHS);
    if (!nl->fitted || !ny->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (nl->replica || ny->replica) return set_err(B200BO_ERR_STATE, "handle is a predict-only replica");
    if (nl->device != ny->device) return set_err(B200BO_ERR_ARG, "the two handles live on different devices");
    if (nl->n != ny->n || nl->d != ny->d || nl->np != ny->np)
        return set_err(B200BO_ERR_ARG, "the two handles hold different training sets (n, d or capacity)");
    if (nl->y_mean != ny->y_mean || nl->y_std != ny->y_std)
        return set_err(B200BO_ERR_ARG, "the two handles have different y statistics");
    if (nl->noise != 0.0) return set_err(B200BO_ERR_ARG, "the noiseless handle has a WhiteKernel term");
    const double tau = nl->jitter, s2 = ny->jitter;
    if (!(s2 >= tau))
        return set_err(B200BO_ERR_ARG, "noise variance %.17g of the fitted GP is below tau = %.17g", s2, tau);
    const int n = (int)nl->n, np = nl->np;
    bool any = false;
    for (int i = 0; i < n; ++i) any = any || incumbent[i] != 0;
    if (!any) return set_err(B200BO_ERR_ARG, "the incumbent mask is empty");
    for (long long i = 0; i < (long long)n * S; ++i)
        if (!std::isfinite(z[i]) || !std::isfinite(e[i])) return set_err(B200BO_ERR_ARG, "non-finite draw at %lld", i);
    CU(cudaSetDevice(nl->device));
    StreamScope scope(nl);
    NvtxRange nvtx_range("b200bo:set_fantasies");
    nl->fant_best.clear();
    int rc;
    DevBuf in, out, v1, v2;
    for (DevBuf* b : {&in, &out, &v1, &v2})
        if ((rc = b->reserve(sizeof(double) * np))) return rc;
    b200bo_gp* noisy = const_cast<b200bo_gp*>(ny);
    const double sq = std::sqrt(s2 - tau), ds = s2 - tau;
    const std::vector<double>& y = nl->y_norm;
    std::vector<double> col(np, 0.0), fp(n), kr(n), F((size_t)n * S), A((size_t)np * S, 0.0), a(n);
    // the state pending rows need (b200bo_gp_condition_fantasies): F, Z and W = K^-1 R per sample.  With
    // sigma_n^2 = tau, k^T K0^-1 (y_n - L0 Z) + l^T Z = k^T K0^-1 y_n for a new row [l^T, r] of L0, so Z is kept as
    // zeros and W as alpha_ = K0^-1 y_n: the same values without a solve.
    for (DevBuf* b : {&nl->fant_f, &nl->fant_z})
        if ((rc = b->reserve(sizeof(double) * np * S))) return rc;
    if ((rc = nl->fant_w.reserve(sizeof(double) * n * S))) return rc;
    if (ds == 0.0) CU(cudaMemsetAsync(nl->fant_z.p, 0, sizeof(double) * np * S, g_st));
    nl->fant_nreg = n;
    const int wpb = 8;
    const dim3 blk(32 * wpb), grd((np + wpb - 1) / wpb);
    for (int s = 0; s < S; ++s) {
        double* fz = nl->fant_z.as<double>() + (size_t)s * np;
        double* fw = nl->fant_w.as<double>() + (size_t)s * n;
        for (int i = 0; i < n; ++i) col[i] = z[(size_t)i * S + s];
        if ((rc = h2d(in.p, col.data(), sizeof(double) * np))) return rc;
        if (ds > 0.0) CU(cudaMemcpyAsync(fz, in.p, sizeof(double) * np, cudaMemcpyDeviceToDevice, g_st));
        gemv_rows_kernel<<<grd, blk, 0, g_st>>>(nl->L.as<double>(), np, in.as<double>(), out.as<double>(), np, np, 1);
        LAUNCHED();
        CU(cudaGetLastError());
        if ((rc = d2h(fp.data(), out.p, sizeof(double) * n))) return rc;  // F_prior = L0 z
        if (ds > 0.0) {
            for (int i = 0; i < n; ++i) col[i] = (y[i] - fp[i]) - sq * e[(size_t)i * S + s];  // R
            if ((rc = h2d(in.p, col.data(), sizeof(double) * np))) return rc;
            if ((rc = solve_spd(noisy, in.as<double>(), out.as<double>(), v1.as<double>(), v2.as<double>()))) return rc;
            CU(cudaMemcpyAsync(fw, out.p, sizeof(double) * n, cudaMemcpyDeviceToDevice, g_st));
            if ((rc = d2h(kr.data(), out.p, sizeof(double) * n))) return rc;  // K^-1 R
            for (int i = 0; i < n; ++i) col[i] = (y[i] - sq * e[(size_t)i * S + s]) - ds * kr[i];
        } else {
            CU(cudaMemcpyAsync(fw, nl->alphav.p, sizeof(double) * n, cudaMemcpyDeviceToDevice, g_st));
            for (int i = 0; i < n; ++i) col[i] = y[i];  // sigma_n^2 = tau: F = y_n exactly
        }
        for (int i = 0; i < n; ++i) F[(size_t)i * S + s] = col[i];
        if ((rc = h2d(in.p, col.data(), sizeof(double) * np))) return rc;
        CU(cudaMemcpyAsync(nl->fant_f.as<double>() + (size_t)s * np, in.p, sizeof(double) * np,
                           cudaMemcpyDeviceToDevice, g_st));
        if ((rc = solve_spd(nl, in.as<double>(), out.as<double>(), v1.as<double>(), v2.as<double>()))) return rc;
        if ((rc = d2h(a.data(), out.p, sizeof(double) * n))) return rc;  // a_s = K0^-1 f_s
        for (int i = 0; i < n; ++i) A[(size_t)i * S + s] = a[i];
    }
    std::vector<double> best(S, -std::numeric_limits<double>::infinity());
    for (int s = 0; s < S; ++s)
        for (int i = 0; i < n; ++i)
            if (incumbent[i]) best[s] = std::fmax(best[s], nl->y_std * F[(size_t)i * S + s] + nl->y_mean);
    A.insert(A.end(), best.begin(), best.end());  // the kernels read best_s behind A
    if ((rc = nl->fant_a.reserve(sizeof(double) * A.size()))) return rc;
    if ((rc = h2d(nl->fant_a.p, A.data(), sizeof(double) * A.size()))) return rc;
    if ((rc = sync_fit_stream())) return rc;
    for (size_t i = 0; i < F.size(); ++i)  // A's first n * S entries are the rows of F
        if (!std::isfinite(F[i]) || !std::isfinite(A[i]))
            return set_err(B200BO_ERR_NOT_PD, "the fantasies are not finite: K0 = c k(X, X) + tau I is too "
                                              "ill-conditioned (raise jitter)");
    if (f_out)
        for (size_t i = 0; i < F.size(); ++i) f_out[i] = nl->y_std * F[i] + nl->y_mean;
    if (best_out)
        for (int s = 0; s < S; ++s) best_out[s] = best[s];
    nl->fant_best = best;
    return B200BO_OK;
}

// Per-sample incumbents of CNEI (include/b200bo.h, DESIGN.md 4.15): best_s from the fantasies F the handle keeps
// ([S][np], normalised), in data units as b200bo_gp_set_fantasies forms them, with the empty-sample floor.
extern "C" int b200bo_gp_set_fantasy_incumbent(b200bo_gp* nl, const uint8_t* eligible, double* best_out) {
    if (!nl || !eligible) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!nl->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (nl->replica) return set_err(B200BO_ERR_STATE, "handle is a predict-only replica");
    if (nl->fant_best.empty())
        return set_err(B200BO_ERR_STATE, "the handle holds no fantasies (b200bo_gp_set_fantasies)");
    if (nl->fant_nreg != nl->n)
        return set_err(B200BO_ERR_STATE, "the fantasies are conditioned on pending rows");
    const int n = (int)nl->n, np = nl->np, S = (int)nl->fant_best.size();
    CU(cudaSetDevice(nl->device));
    StreamScope scope(nl);
    int rc;
    std::vector<double> F((size_t)S * np);
    if ((rc = d2h(F.data(), nl->fant_f.p, sizeof(double) * F.size()))) return rc;
    std::vector<double> best(S);
    for (int s = 0; s < S; ++s) {
        double hi = -std::numeric_limits<double>::infinity(), lo = std::numeric_limits<double>::infinity();
        bool any = false;
        for (int i = 0; i < n; ++i) {
            const double v = nl->y_std * F[(size_t)s * np + i] + nl->y_mean;
            lo = std::fmin(lo, v);
            if (eligible[(size_t)i * S + s]) {
                hi = std::fmax(hi, v);
                any = true;
            }
        }
        best[s] = any ? hi : lo;
    }
    if ((rc = h2d(nl->fant_a.as<double>() + (size_t)np * S, best.data(), sizeof(double) * S))) return rc;
    if ((rc = sync_fit_stream())) return rc;
    nl->fant_best = best;
    if (best_out)
        for (int s = 0; s < S; ++s) best_out[s] = best[s];
    return B200BO_OK;
}

// CNEI's incumbents on the device (include/b200bo.h, DESIGN.md 4.16): eligibility and best_s from the F of the target and
// constraint handles, over registered and pending rows alike; only the S incumbents come back to the host.
extern "C" int b200bo_gp_set_constrained_incumbent(b200bo_gp* target, b200bo_gp* const* constraints, int n_constraints,
                                                   const double* lb, const double* ub, const uint8_t* in_bounds,
                                                   double* best_out) {
    if (!target || !in_bounds || (n_constraints > 0 && (!constraints || !lb || !ub)))
        return set_err(B200BO_ERR_ARG, "NULL argument");
    if (n_constraints < 0 || n_constraints > B200BO_MAX_GPS - 1)
        return set_err(B200BO_ERR_ARG, "n_constraints=%d out of range [0,%d]", n_constraints, B200BO_MAX_GPS - 1);
    IncumbentGPs G{};
    G.n_gps = n_constraints + 1;
    for (int g = 0; g < G.n_gps; ++g) {
        const b200bo_gp* h = g == 0 ? target : constraints[g - 1];
        if (!h) return set_err(B200BO_ERR_ARG, "NULL argument");
        if (!h->fitted) return set_err(B200BO_ERR_STATE, "GP handle %d is not fitted", g);
        if (h->replica) return set_err(B200BO_ERR_STATE, "handle %d is a predict-only replica", g);
        if (h->fant_best.empty())
            return set_err(B200BO_ERR_STATE, "handle %d holds no fantasies (b200bo_gp_set_fantasies)", g);
        if (h->device != target->device || h->n != target->n || h->np != target->np ||
            h->fant_best.size() != target->fant_best.size())
            return set_err(B200BO_ERR_ARG, "handle %d differs from the target in device, n, np or S", g);
        if (g > 0 && !(lb[g - 1] < ub[g - 1]))
            return set_err(B200BO_ERR_ARG, "constraint %d: lb=%.17g is not below ub=%.17g", g - 1, lb[g - 1], ub[g - 1]);
        G.f[g] = h->fant_f.as<double>();
        G.y_std[g] = h->y_std;
        G.y_mean[g] = h->y_mean;
        G.lb[g] = g > 0 ? lb[g - 1] : 0.0;
        G.ub[g] = g > 0 ? ub[g - 1] : 0.0;
    }
    const int n = (int)target->n, np = target->np, S = (int)target->fant_best.size();
    CU(cudaSetDevice(target->device));
    StreamScope scope(target);
    NvtxRange nvtx_range("b200bo:set_constrained_incumbent");
    int rc;
    if ((rc = target->fant_mask.reserve(n))) return rc;
    if ((rc = h2d(target->fant_mask.p, in_bounds, n))) return rc;
    double* best = target->fant_a.as<double>() + (size_t)np * S;  // the kernels read best_s behind A
    fantasy_incumbent_kernel<<<1, 32 * S, 0, g_st>>>(G, target->fant_mask.as<uint8_t>(), n, np, best);
    LAUNCHED();
    CU(cudaGetLastError());
    std::vector<double> bst(S);
    if ((rc = d2h(bst.data(), best, sizeof(double) * S))) return rc;
    target->fant_best = bst;
    if (best_out)
        for (int s = 0; s < S; ++s) best_out[s] = bst[s];
    return B200BO_OK;
}

// Row n of the O(N^2) factor update at the hyper-parameters of the last fit, shared by b200bo_gp_append and
// b200bo_gp_condition: row n of X / Xs, row and column n of K, row n of L (pivot checked) and of L^-1 (W and WT).
// tvec: n-entry device scratch.  believer (nullable, device): receives k(x, X) . alpha_ in normalised units, computed
// from the new K row right after it is built - before anything writes tvec, which may be alpha_ itself.
// *finfo = 0, or the failing pivot (1-based) and rows n of K / L are garbage.  gp->n is the caller's to advance.
static int append_factor_row(b200bo_gp* gp, const double* x_new, double* tvec, double* believer, int* finfo) {
    const int n = (int)gp->n, np = gp->np, d = gp->d;
    int rc;
    if ((rc = gp->xc.reserve(sizeof(double) * B200BO_MAX_DIM))) return rc;
    CU(cudaMemcpy(gp->xc.p, x_new, sizeof(double) * d, cudaMemcpyHostToDevice));
    CU(cudaMemset(gp->info.p, 0, sizeof(int)));
    const int* xf = gp->xform.empty() ? nullptr : gp->xf.as<int>();
    double* kvec = gp->v1.as<double>();
    double* lvec = gp->v2.as<double>();
    if (n > 0) {
        append_krow_kernel<<<(n + 127) / 128, 128>>>(gp->xc.as<double>(), gp->ls.as<double>(), xf, gp->Xs.as<double>(),
                                                     gp->X.as<double>(), kvec, n, d, gp->family, gp->nu, gp->constv);
        if (believer) {  // mu_norm(x) = k^T alpha_: one warp, fixed-order reduction
            gemv_rows_kernel<<<1, 32>>>(kvec, np, gp->alphav.as<double>(), believer, 1, n, 0);
            LAUNCHED();
        }
        const int wpb = 8;
        dim3 blk(32 * wpb), grd((n + wpb - 1) / wpb);
        gemv_rows_kernel<<<grd, blk>>>(gp->W.as<double>(), np, kvec, lvec, n, n, 1);   // l = W k
        append_rows_kernel<<<1, 256>>>(gp->K.as<double>(), gp->L.as<double>(), kvec, lvec, n, np,
                                       gp->constv + gp->jitter, gp->info.as<int>(), gp->part.as<double>());
        gemv_rows_kernel<<<grd, blk>>>(gp->WT.as<double>(), np, lvec, tvec, n, n, 2);  // t = W^T l
        for (int i = 0; i < 4; ++i) LAUNCHED();
    }
    *finfo = 0;
    CU(cudaMemcpy(finfo, gp->info.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (*finfo != 0) return B200BO_OK;
    append_winv_kernel<<<(n + 1 + 127) / 128, 128>>>(gp->W.as<double>(), gp->WT.as<double>(), tvec,
                                                     gp->part.as<double>(), n, np);
    LAUNCHED();
    return B200BO_OK;
}

// Append one training point at the hyper-parameters of the last fit, O(N^2) (SURVEY.md 8f rank 3).
// Falls outside the padded capacity (n == np) -> B200BO_ERR_STATE: the caller refits from scratch.
extern "C" int b200bo_gp_append(b200bo_gp* gp, const double* x_new, double y_new, int64_t* info) {
    if (!gp || !x_new) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (gp->replica) return set_err(B200BO_ERR_STATE, "handle is a predict-only replica: append to the source and replicate again");
    if (gp->n >= gp->np) return set_err(B200BO_ERR_STATE, "no padding slack left (n == np): refit");
    CU(cudaSetDevice(gp->device));
    const int n = (int)gp->n;
    if (info) *info = 0;
    gp->fant_best.clear();
    int rc;
    int finfo = 0;
    // alpha_ is recomputed below; reuse it as scratch
    if ((rc = append_factor_row(gp, x_new, gp->alphav.as<double>(), nullptr, &finfo))) return rc;
    if (finfo != 0) {
        gp->fitted = false;  // row n of K/L is garbage now
        if (info) *info = finfo;
        return set_err(B200BO_ERR_NOT_PD, "%d-th leading minor of the array is not positive definite", finfo);
    }
    // targets: new normalisation statistics, alpha_ = K^-1 y
    gp->y_raw.push_back(y_new);
    const int64_t nn = n + 1;
    normalize_targets(gp);
    CU(cudaMemcpy(gp->y.p, gp->y_norm.data(), sizeof(double) * nn, cudaMemcpyHostToDevice));
    gp->n = nn;
    gp->tc_valid = false;
    gp->pad_valid = false;
    gp->gram_valid = false;
    if ((rc = solve_alpha(gp))) return rc;
    CU(cudaDeviceSynchronize());
    return B200BO_OK;
}

// Row n of b200bo_gp_condition: the factor row update, the believer target mu_norm(x) in y's padding slot n and as
// row n of the host targets, alpha_ = [alpha_; 0].  *mu (nullable) receives the target in data units.  A non-positive
// pivot leaves the handle unfitted.  gp->tscratch holds np entries.
static int condition_row(b200bo_gp* gp, const double* x, double* mu) {
    const int n = (int)gp->n;
    double* yn = gp->y.as<double>() + n;
    int finfo = 0, rc;
    if ((rc = append_factor_row(gp, x, gp->tscratch.as<double>(), yn, &finfo))) return rc;
    if (finfo != 0) {
        gp->fitted = false;  // row n of K/L is garbage now
        return set_err(B200BO_ERR_NOT_PD, "%d-th leading minor of the array is not positive definite", finfo);
    }
    double mu_norm = 0.0;
    CU(cudaMemcpy(&mu_norm, yn, sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemset(gp->alphav.as<double>() + n, 0, sizeof(double)));  // alpha_ = [alpha_; 0]
    const double m = gp->y_std * mu_norm + gp->y_mean;  // data units, as the predict kernels form the mean
    gp->y_norm.push_back(mu_norm);
    gp->y_raw.push_back(m);
    if (mu) *mu = m;
    gp->n = n + 1;
    gp->tc_valid = false;
    gp->pad_valid = false;
    gp->gram_valid = false;
    return B200BO_OK;
}

// Kriging believer (DESIGN.md 4.11): row n gets the target mu_norm(x) = k(x, X)^T alpha_, so K' [alpha_; 0] =
// [y; mu_norm(x)] and alpha_ extends by a zero - no solve, the mean is unchanged everywhere, only K, L, L^-1 grow.
extern "C" int b200bo_gp_condition(b200bo_gp* gp, const double* Xp, int64_t p, double* mu_out) {
    if (!gp || (p > 0 && !Xp)) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (p < 0) return set_err(B200BO_ERR_ARG, "p=%lld must be >= 0", (long long)p);
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (gp->replica)
        return set_err(B200BO_ERR_STATE, "handle is a predict-only replica: condition the source or a fork of it");
    if (p > gp->np - gp->n)
        return set_err(B200BO_ERR_STATE, "no padding slack for %lld rows (n=%lld, np=%d): fork with extra_rows",
                       (long long)p, gp->n, gp->np);
    const int d = gp->d;
    for (int64_t i = 0; i < p * d; ++i)
        if (!std::isfinite(Xp[i])) return set_err(B200BO_ERR_ARG, "Input X contains NaN or infinity.");
    CU(cudaSetDevice(gp->device));
    NvtxRange nvtx_range("b200bo:condition");
    gp->fant_best.clear();
    int rc;
    if ((rc = gp->tscratch.reserve(sizeof(double) * gp->np))) return rc;
    for (int64_t r = 0; r < p; ++r)
        if ((rc = condition_row(gp, Xp + r * d, mu_out ? mu_out + r : nullptr))) return rc;
    CU(cudaDeviceSynchronize());
    return B200BO_OK;
}

// The work of b200bo_gp_condition_fantasies after its checks; on an error the caller drops the fantasies.
static int extend_fantasies(b200bo_gp* gp, const double* Xp, int64_t p, const double* zp, double* f_out,
                            double* best_out) {
    const int d = gp->d, S = (int)gp->fant_best.size();
    const int np = gp->np, n0 = (int)gp->n;
    int rc;
    if ((rc = gp->tscratch.reserve(sizeof(double) * np))) return rc;
    if ((rc = gp->fant_tmp.reserve(sizeof(double) * ((size_t)np * S + S)))) return rc;
    double* acol = gp->fant_tmp.as<double>();
    double* zrow = acol + (size_t)np * S;
    double* best = gp->fant_a.as<double>() + (size_t)np * S;
    for (int64_t r = 0; r < p; ++r) {
        const int n = (int)gp->n;
        if ((rc = condition_row(gp, Xp + r * d, nullptr))) return rc;
        CU(cudaMemcpy(zrow, zp + r * S, sizeof(double) * S, cudaMemcpyHostToDevice));
        fantasy_row_kernel<<<1, 32 * S>>>(gp->K.as<double>(), gp->L.as<double>(), np, n, gp->fant_nreg,
                                          gp->fant_w.as<double>(), zrow, gp->fant_z.as<double>(),
                                          gp->fant_f.as<double>(), best, gp->y_std, gp->y_mean);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    const int n = (int)gp->n;
    for (int s = 0; s < S && p > 0; ++s)
        if ((rc = solve_spd(gp, gp->fant_f.as<double>() + (size_t)s * np, acol + (size_t)s * np, gp->v1.as<double>(),
                            gp->v2.as<double>())))
            return rc;
    if (p > 0) {
        fantasy_pack_kernel<<<(np * S + 255) / 256, 256>>>(acol, np, n, S, gp->fant_a.as<double>());
        LAUNCHED();
        CU(cudaGetLastError());
    }
    std::vector<double> F((size_t)S * np), A((size_t)np * S), bst(S);
    CU(cudaMemcpy(F.data(), gp->fant_f.p, sizeof(double) * F.size(), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(A.data(), gp->fant_a.p, sizeof(double) * A.size(), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(bst.data(), best, sizeof(double) * S, cudaMemcpyDeviceToHost));
    for (int s = 0; s < S; ++s)
        for (int i = 0; i < n; ++i)
            if (!std::isfinite(F[(size_t)s * np + i]) || !std::isfinite(A[(size_t)i * S + s]))
                return set_err(B200BO_ERR_NOT_PD, "the fantasies are not finite: K0 = c k(X, X) + tau I is too "
                                                  "ill-conditioned (raise jitter)");
    gp->fant_best = bst;
    if (f_out)
        for (int64_t r = 0; r < p; ++r)
            for (int s = 0; s < S; ++s) f_out[r * S + s] = gp->y_std * F[(size_t)s * np + n0 + r] + gp->y_mean;
    if (best_out)
        for (int s = 0; s < S; ++s) best_out[s] = bst[s];
    return B200BO_OK;
}

// NEI fantasies at pending rows (include/b200bo.h, DESIGN.md 4.14): per row the believer row update of
// b200bo_gp_condition, then fantasy_row_kernel forms the S values F_js on the device; after the last row
// A' = K0'^-1 F' per sample with solve_spd, as b200bo_gp_set_fantasies solves.
extern "C" int b200bo_gp_condition_fantasies(b200bo_gp* gp, const double* Xp, int64_t p, const double* zp,
                                             double* f_out, double* best_out) {
    if (!gp || (p > 0 && (!Xp || !zp))) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (p < 0) return set_err(B200BO_ERR_ARG, "p=%lld must be >= 0", (long long)p);
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (gp->replica)
        return set_err(B200BO_ERR_STATE, "handle is a predict-only replica: condition the source or a fork of it");
    if (p > gp->np - gp->n)
        return set_err(B200BO_ERR_STATE, "no padding slack for %lld rows (n=%lld, np=%d): fork with extra_rows",
                       (long long)p, gp->n, gp->np);
    if (gp->fant_best.empty())
        return set_err(B200BO_ERR_STATE, "the handle holds no fantasies (b200bo_gp_set_fantasies)");
    const int d = gp->d, S = (int)gp->fant_best.size();
    for (int64_t i = 0; i < p * d; ++i)
        if (!std::isfinite(Xp[i])) return set_err(B200BO_ERR_ARG, "Input X contains NaN or infinity.");
    for (int64_t i = 0; i < p * S; ++i)
        if (!std::isfinite(zp[i])) return set_err(B200BO_ERR_ARG, "non-finite draw at %lld", (long long)i);
    CU(cudaSetDevice(gp->device));
    NvtxRange nvtx_range("b200bo:condition_fantasies");
    const int rc = extend_fantasies(gp, Xp, p, zp, f_out, best_out);
    if (rc != B200BO_OK) gp->fant_best.clear();  // A no longer matches the factor and F
    return rc;
}

// the fitted model's shape, hyper-parameters and target statistics: what a fork and a replica both take from the source
static void copy_model_state(const b200bo_gp* src, b200bo_gp* dst) {
    dst->n = src->n;
    dst->d = src->d;
    dst->family = src->family;
    dst->nu = src->nu;
    dst->constv = src->constv;
    dst->jitter = src->jitter;
    dst->noise = src->noise;
    dst->y_mean = src->y_mean;
    dst->y_std = src->y_std;
    dst->normalize = src->normalize;
    dst->xform = src->xform;
    dst->precision = src->precision;
}

static int fork_into(const b200bo_gp* src, int64_t extra_rows, b200bo_gp* dst) {
    copy_model_state(src, dst);
    dst->np = round_up(src->n + extra_rows, kPad);
    dst->y_norm = src->y_norm;
    dst->y_raw = src->y_raw;
    dst->ystar = src->ystar;
    const size_t n = src->n, d = src->d, np0 = src->np, np = dst->np;
    int rc;
    DevBuf* vecs[] = {&dst->X, &dst->Xs, &dst->y, &dst->alphav, &dst->v1, &dst->v2};
    const size_t vec_len[] = {np * d, np * d, np, np, np, np};
    for (int i = 0; i < 6; ++i) {
        if ((rc = vecs[i]->reserve(sizeof(double) * vec_len[i]))) return rc;
        CU(cudaMemset(vecs[i]->p, 0, sizeof(double) * vec_len[i]));
    }
    if ((rc = dst->ls.reserve(sizeof(double) * B200BO_MAX_DIM))) return rc;
    if ((rc = dst->xf.reserve(sizeof(int) * B200BO_MAX_DIM))) return rc;
    if ((rc = dst->info.reserve(sizeof(int)))) return rc;
    if ((rc = dst->part.reserve(sizeof(double) * 64))) return rc;
    CU(cudaMemcpy(dst->X.p, src->X.p, sizeof(double) * n * d, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(dst->Xs.p, src->Xs.p, sizeof(double) * n * d, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(dst->y.p, src->y.p, sizeof(double) * n, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(dst->alphav.p, src->alphav.p, sizeof(double) * n, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(dst->ls.p, src->ls.p, sizeof(double) * B200BO_MAX_DIM, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(dst->xf.p, src->xf.p, sizeof(int) * B200BO_MAX_DIM, cudaMemcpyDeviceToDevice));
    struct Mat {
        DevBuf* to;
        const DevBuf* from;
    } mats[] = {{&dst->K, &src->K}, {&dst->L, &src->L}, {&dst->W, &src->W}, {&dst->WT, &src->WT}};
    const dim3 blk(32, 8), grd((unsigned)(np / 32), (unsigned)(np / 32));
    for (const Mat& m : mats) {
        if ((rc = m.to->reserve(sizeof(double) * np * np))) return rc;
        repitch_identity_kernel<<<grd, blk>>>(m.from->as<double>(), (int)np0, m.to->as<double>(), (int)np);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    if (!src->fant_best.empty()) {  // NEI fantasies: A ([np'][S], best_s behind it), F and Z ([S][np']), W as it is
        const size_t S = src->fant_best.size(), nreg = src->fant_nreg;
        if ((rc = dst->fant_a.reserve(sizeof(double) * (np * S + S)))) return rc;
        CU(cudaMemset(dst->fant_a.p, 0, sizeof(double) * np * S));
        CU(cudaMemcpy(dst->fant_a.p, src->fant_a.p, sizeof(double) * n * S, cudaMemcpyDeviceToDevice));
        CU(cudaMemcpy(dst->fant_a.as<double>() + np * S, src->fant_a.as<double>() + np0 * S, sizeof(double) * S,
                      cudaMemcpyDeviceToDevice));
        for (const Mat& m : {Mat{&dst->fant_f, &src->fant_f}, Mat{&dst->fant_z, &src->fant_z}}) {
            if ((rc = m.to->reserve(sizeof(double) * np * S))) return rc;
            CU(cudaMemset(m.to->p, 0, sizeof(double) * np * S));
            CU(cudaMemcpy2D(m.to->p, sizeof(double) * np, m.from->p, sizeof(double) * np0, sizeof(double) * n, S,
                            cudaMemcpyDeviceToDevice));
        }
        if ((rc = dst->fant_w.reserve(sizeof(double) * nreg * S))) return rc;
        CU(cudaMemcpy(dst->fant_w.p, src->fant_w.p, sizeof(double) * nreg * S, cudaMemcpyDeviceToDevice));
        dst->fant_nreg = src->fant_nreg;
        dst->fant_best = src->fant_best;
    }
    CU(cudaDeviceSynchronize());
    dst->fitted = true;
    return B200BO_OK;
}

// A full, appendable copy of a fitted handle with capacity for extra_rows more rows (DESIGN.md 4.11).
extern "C" int b200bo_gp_fork(const b200bo_gp* src, int64_t extra_rows, b200bo_gp** out) {
    if (!src || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (extra_rows < 0) return set_err(B200BO_ERR_ARG, "extra_rows=%lld must be >= 0", (long long)extra_rows);
    if (!src->fitted) return set_err(B200BO_ERR_STATE, "source GP handle is not fitted");
    if (src->replica)
        return set_err(B200BO_ERR_STATE, "a predict-only replica holds no K / L: fork the source handle");
    if (src->n + extra_rows > 38000)
        return set_err(B200BO_ERR_ARG, "n + extra_rows = %lld too large (<= 38000)", (long long)(src->n + extra_rows));
    b200bo_gp* dst = nullptr;
    int rc;
    if ((rc = b200bo_gp_create(&dst, src->device))) return rc;
    NvtxRange nvtx_range("b200bo:fork");
    if ((rc = fork_into(src, extra_rows, dst))) {
        cudaGetLastError();  // an out-of-memory cudaMalloc leaves its error behind
        b200bo_gp_destroy(dst);
        return rc;
    }
    *out = dst;
    return B200BO_OK;
}

extern "C" int b200bo_gp_lml(b200bo_gp* gp, const b200bo_kernel* kern, double alpha, int has_const,
                             double* lml, double* grad) {
    if (!gp || !lml) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!gp->has_data) return set_err(B200BO_ERR_STATE, "no training data: call b200bo_gp_set_data");
    int rc;
    if ((rc = check_kernel(gp, kern))) return rc;
    CU(cudaSetDevice(gp->device));
    StreamScope scope(gp);
    NvtxRange nvtx_range("b200bo:lml");
    gp->fitted = false;  // buffers are being overwritten
    gp->tc_valid = false;
    gp->pad_valid = false;
    gp->gram_valid = false;
    const int n = (int)gp->n, np = gp->np, d = gp->d;
    const int aniso = kern->n_length_scale > 1;
    const int want_noise = (has_const & 2) ? 1 : 0;
    has_const &= 1;
    const int ntheta_k = (has_const ? 1 : 0) + kern->n_length_scale;  // produced by the pair kernel
    const int ntheta = ntheta_k + want_noise;
    int finfo = 0;
    if ((rc = factorize(gp, kern, alpha + kern->noise_level, &finfo))) return rc;
    if (finfo != 0) {  // SK/_gpr.py:590-593
        *lml = -std::numeric_limits<double>::infinity();
        if (grad)
            for (int p = 0; p < ntheta; ++p) grad[p] = 0.0;
        return B200BO_OK;
    }
    diag_kernel<<<(n + 255) / 256, 256, 0, g_st>>>(gp->L.as<double>(), np, gp->v1.as<double>(), n);
    LAUNCHED();
    std::vector<double> a(n), dg(n);
    if ((rc = d2h(a.data(), gp->alphav.p, sizeof(double) * n))) return rc;
    if ((rc = d2h(dg.data(), gp->v1.p, sizeof(double) * n))) return rc;
    long double ya = 0.0L, ld = 0.0L;
    for (int i = 0; i < n; ++i) {
        ya += (long double)gp->y_norm[i] * a[i];
        ld += logl((long double)dg[i]);
    }
    *lml = (double)(-0.5L * ya - ld - (long double)n / 2.0L * logl(2.0L * 3.14159265358979323846264338327950288L));
    if (grad) {
        // Kinv = W^T W  (W lower: k >= max(m0, n0)); lower tiles only - the gradient kernel uses symmetry
        if ((rc = gemm<true, false>(np, np, np, 1.0, gp->W.as<double>(), np, 0, gp->W.as<double>(), np, 0,
                                    0.0, gp->T.as<double>(), np, 0, 1, 1, 3)))
            return rc;
        size_t nblk;
        const int cov = cov_code(kern->family, kern->nu);
        if (d <= LG_DMAX) {
            // 64x64 patches on or below the diagonal, covariance and iso/aniso as template parameters
            const int nb64 = (n + 63) / 64;
            dim3 grd(nb64, nb64);
            nblk = (size_t)nb64 * (nb64 + 1) / 2;
            if ((rc = gp->part.reserve(sizeof(double) * nblk * ntheta_k))) return rc;
            const double* Xsp = gp->Xs.as<double>();
            const double* Ki = gp->T.as<double>();
            const double* al = gp->alphav.as<double>();
            double* pt = gp->part.as<double>();
#define B200BO_LG(COV)                                                                                              \
    if (aniso)                                                                                                      \
        lml_grad_tile_kernel<COV, true><<<grd, 256, 0, g_st>>>(Xsp, Ki, np, al, n, d, kern->const_value, has_const, pt, ntheta_k); \
    else                                                                                                            \
        lml_grad_tile_kernel<COV, false><<<grd, 256, 0, g_st>>>(Xsp, Ki, np, al, n, d, kern->const_value, has_const, pt, ntheta_k);
            switch (cov) {
                case 0: B200BO_LG(0) break;
                case 1: B200BO_LG(1) break;
                case 2: B200BO_LG(2) break;
                default: B200BO_LG(3) break;
            }
#undef B200BO_LG
        } else {
            dim3 grd((n + 15) / 16, (n + 15) / 16);
            nblk = (size_t)grd.x * grd.y;
            if ((rc = gp->part.reserve(sizeof(double) * nblk * ntheta_k))) return rc;
            lml_grad_kernel<<<grd, 256, 0, g_st>>>(gp->Xs.as<double>(), gp->T.as<double>(), np, gp->alphav.as<double>(),
                                                   n, d, kern->family,
                                                   kern->family == B200BO_KERNEL_RBF ? B200BO_NU_INF : kern->nu,
                                                   kern->const_value, has_const, aniso, gp->part.as<double>(), ntheta_k);
        }
        LAUNCHED();
        CU(cudaGetLastError());
        std::vector<double> part(nblk * ntheta_k);
        if ((rc = d2h(part.data(), gp->part.p, sizeof(double) * nblk * ntheta_k))) return rc;
        for (int p = 0; p < ntheta_k; ++p) {
            long double s = 0.0L;
            for (size_t b = 0; b < nblk; ++b) s += part[b * ntheta_k + p];
            grad[p] = (double)s;
        }
        if (want_noise) {
            // dK/dlog(noise_level) = noise_level * I (SK/gaussian_process/kernels.py:1311-1322):
            // grad = 0.5 * noise_level * sum_i (alpha_i^2 - (K^-1)_ii)
            diag_kernel<<<(n + 255) / 256, 256, 0, g_st>>>(gp->T.as<double>(), np, gp->v2.as<double>(), n);
            LAUNCHED();
            std::vector<double> kd(n);
            if ((rc = d2h(kd.data(), gp->v2.p, sizeof(double) * n))) return rc;
            long double sn = 0.0L;
            for (int i = 0; i < n; ++i) sn += (long double)a[i] * a[i] - (long double)kd[i];
            grad[ntheta_k] = (double)(0.5L * (long double)kern->noise_level * sn);
        }
    }
    return B200BO_OK;
}

extern "C" int b200bo_gp_get(b200bo_gp* gp, int what, double* out, int64_t len) {
    if (!gp || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    CU(cudaSetDevice(gp->device));
    const size_t n = gp->n, np = gp->np;
    const void* src = nullptr;
    if (gp->replica && (what == B200BO_GET_L || what == B200BO_GET_K))
        return set_err(B200BO_ERR_STATE, "a predict-only replica holds no K / L: read them from the source handle");
    switch (what) {
        case B200BO_GET_L: src = gp->L.p; break;
        case B200BO_GET_K: src = gp->K.p; break;
        case B200BO_GET_LINV: src = gp->W.p; break;
        case B200BO_GET_ALPHA:
            if (len != (int64_t)n) return set_err(B200BO_ERR_ARG, "len must be n");
            CU(cudaMemcpy(out, gp->alphav.p, sizeof(double) * n, cudaMemcpyDeviceToHost));
            return B200BO_OK;
        case B200BO_GET_YSTATS:
            if (len != 2) return set_err(B200BO_ERR_ARG, "len must be 2");
            out[0] = gp->y_mean;
            out[1] = gp->y_std;
            return B200BO_OK;
        default: return set_err(B200BO_ERR_ARG, "unknown selector %d", what);
    }
    if (len != (int64_t)(n * n)) return set_err(B200BO_ERR_ARG, "len must be n*n");
    CU(cudaMemcpy2D(out, sizeof(double) * n, src, sizeof(double) * np, sizeof(double) * n, n,
                    cudaMemcpyDeviceToHost));
    return B200BO_OK;
}

// ---------------------------------------------------------------------------------------
// predict / acquisition
// ---------------------------------------------------------------------------------------
// work units of the small path's triangular products: row block i covers k in [0, 64 (i + 1)) of L^-1 v, or
// [64 i, np) of L^-T v (upper), in SKCH chunks; rbs[i] = (first unit of row block i, its number of units)
static void small_units(int np, bool upper, std::vector<int2>& units, std::vector<int2>& rbs) {
    for (int i = 0; i < np / SROWS; ++i) {
        const int nk = upper ? np - i * SROWS : (i + 1) * SROWS;
        const int nj = (nk + SKCH - 1) / SKCH;
        rbs.push_back(make_int2((int)units.size(), nj));
        for (int j = 0; j < nj; ++j) units.push_back(make_int2(i, j));
    }
}

// gradient calls: the work units of u = L^-T v + their scratch for one GP
static int ensure_small_grad(b200bo_gp* gp) {
    const int np = gp->np, d = gp->d;
    if (gp->s_grad_np == np && gp->s_grad_d == d) return B200BO_OK;
    std::vector<int2> units, rbs;
    small_units(np, true, units, rbs);
    int rc;
    if ((rc = gp->s_unit_u.reserve(sizeof(int2) * units.size()))) return rc;
    if ((rc = gp->s_rb_u.reserve(sizeof(int2) * rbs.size()))) return rc;
    if ((rc = gp->s_vsum.reserve(sizeof(double) * (size_t)SMAXP * np * SMC))) return rc;
    if ((rc = gp->s_usum.reserve(sizeof(double) * (size_t)SMAXP * np * SMC))) return rc;
    if ((rc = gp->s_partial_u.reserve(sizeof(double) * (size_t)SMAXP * units.size() * SROWS * SMC))) return rc;
    if ((rc = gp->s_gpart.reserve(sizeof(double) * (size_t)SMAXP * (np / 128) * 2 * d * SMC))) return rc;
    CU(cudaMemcpy(gp->s_unit_u.p, units.data(), sizeof(int2) * units.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(gp->s_rb_u.p, rbs.data(), sizeof(int2) * rbs.size(), cudaMemcpyHostToDevice));
    gp->s_grad_np = np;
    gp->s_grad_d = d;
    gp->s_nunits_u = (int)units.size();
    return B200BO_OK;
}

// small-batch path: work-unit tables + scratch for one GP
static int ensure_small(b200bo_gp* gp, bool grad = false) {
    if (grad) {
        const int rc = ensure_small_grad(gp);
        if (rc) return rc;
    }
    const int np = gp->np;
    if (gp->s_np == np) return B200BO_OK;
    std::vector<int2> units, rbs;
    small_units(np, false, units, rbs);
    int rc;
    if ((rc = gp->s_unit.reserve(sizeof(int2) * units.size()))) return rc;
    if ((rc = gp->s_rb.reserve(sizeof(int2) * rbs.size()))) return rc;
    if ((rc = gp->s_ksm.reserve(sizeof(double) * (size_t)SMAXP * np * SMC))) return rc;
    if ((rc = gp->s_partial.reserve(sizeof(double) * (size_t)SMAXP * units.size() * SROWS * SMC))) return rc;
    if ((rc = gp->s_mupart.reserve(sizeof(double) * (size_t)SMAXP * (np / 128) * SMC))) return rc;
    if ((rc = gp->s_colsq.reserve(sizeof(double) * (size_t)SMAXP * (np / SROWS) * SMC))) return rc;
    CU(cudaMemcpy(gp->s_unit.p, units.data(), sizeof(int2) * units.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(gp->s_rb.p, rbs.data(), sizeof(int2) * rbs.size(), cudaMemcpyHostToDevice));
    gp->s_np = np;
    gp->s_nunits = (int)units.size();
    return B200BO_OK;
}

// Cost model (microseconds, orders of magnitude) choosing between the tiled
// persistent kernel and the small-batch path.  B200BO_SMALL_PATH=0/1 forces one of them.
// B200BO_PATH_STABLE: the decision is taken for a nominal batch of one pass (SMC rows) whatever m is,
// so an optimiser's f(x) and its finite-difference stencil always run through the same kernels.
static bool use_small_path(long long m, int np_max, int n_gps, int sm_count, int path) {
    const char* e = getenv("B200BO_SMALL_PATH");
    if (e && (e[0] == '0' || e[0] == '1')) return e[0] == '1';
    if (m <= 0) return false;
    if (path == B200BO_PATH_STABLE) m = SMC;
    const double x = (np_max / 4096.0) * (np_max / 4096.0);
    const double passes = (double)((m + SMC - 1) / SMC);
    const double tiles = (double)((m + PBN - 1) / PBN);
    const double t_small = passes * (15.0 + 60.0 * x) * n_gps;
    const double t_big = std::ceil(tiles / sm_count) * (10.0 + 9000.0 * x) * n_gps;
    return t_small < t_big;
}

// GEMM inner-loop variant of the fused predict kernel: "dmma" (mma.sync f64, default; shape: predict_mma) or
// "dfma" (8x8 register tiles).  Both are exact fp64 with fixed-order reductions; the environment
// variable B200BO_PREDICT_IMPL selects one for A/B measurements.
static int predict_impl(int precision) {
    const char* e = getenv("B200BO_PREDICT_IMPL");
    if (e && (e[0] == 'd' || e[0] == 'D') && (e[1] == 'f' || e[1] == 'F')) return PREDICT_IMPL_DFMA;
    if (e && (e[0] == 't' || e[0] == 'T')) return PREDICT_IMPL_TF32;  // "tf32": fp32 mode on wgmma
    if (e && (e[0] == 'd' || e[0] == 'D')) return PREDICT_IMPL_DMMA;
    return precision == B200BO_PRECISION_FP32 ? PREDICT_IMPL_TF32 : PREDICT_IMPL_DMMA;
}

// 8-warp (predict_acq_kernel) or 16-warp (predict_acq16_kernel) version of the fp64 kernel;
// B200BO_PREDICT_WARPS=8|16 overrides the default for A/B measurements
static int predict_warps() {
    const char* e = getenv("B200BO_PREDICT_WARPS");
    if (e && e[0] == '1' && e[1] == '6') return 16;
    if (e && e[0] == '8') return 8;
    return kDefaultPredictWarps;
}

// MMA shape of phase B of predict_acq16_kernel: 1684 (mma.sync m16n8k4 f64, sm_90, default) or, with
// B200BO_PREDICT_MMA=884, the sm_80 shape m8n8k4 for A/B measurements
static int predict_mma() {
    const char* e = getenv("B200BO_PREDICT_MMA");
    return (e && strcmp(e, "884") == 0) ? 884 : 1684;
}

// phase B data path of predict_acq16_kernel (m16n8k4 only; m8n8k4 keeps cp.async): B200BO_PREDICT_PIPE=bulk (bulk
// copies on an mbarrier ring, L^-1 multicast across CTA pairs), bulk_nomc (the same without clusters) or cpasync
// (per-thread cp.async under CTA barriers) overrides the default for A/B measurements
static int predict_pipe() {
    const char* e = getenv("B200BO_PREDICT_PIPE");
    if (e && strcmp(e, "bulk") == 0) return PIPE_BULK_MC;
    if (e && strcmp(e, "bulk_nomc") == 0) return PIPE_BULK;
    if (e && strcmp(e, "cpasync") == 0) return PIPE_CPASYNC;
    return kDefaultPredictPipe;
}

// launch configuration of predict_acq16_kernel, in 2-CTA clusters when pair (attr: the storage cfg points to)
static void predict16_config(int grid, cudaStream_t stream, bool pair, cudaLaunchConfig_t& cfg,
                             cudaLaunchAttribute& attr) {
    cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(P16_NT);
    cfg.dynamicSmemBytes = kPredictSmemBytesDmma;
    cfg.stream = stream;
    if (pair) {
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = 2;
        attr.val.clusterDim.y = 1;
        attr.val.clusterDim.z = 1;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
    }
}

template <int MMA, int PIPE>
static int launch_predict16(bool dreg, int grid, cudaStream_t stream, const PredictParams& P) {
    auto fn = dreg ? predict_acq16_kernel<true, MMA, PIPE> : predict_acq16_kernel<false, MMA, PIPE>;
    if constexpr (PIPE != PIPE_CPASYNC) {  // NEI / LogNEI, CNEI / LogCNEI: bulk-copy pipes only (DESIGN.md 4.13, 4.15)
        if (acq_is_nei(P.acq_kind))
            fn = dreg ? predict_acq16_kernel<true, MMA, PIPE, true> : predict_acq16_kernel<false, MMA, PIPE, true>;
        else if (acq_is_cnei(P.acq_kind))
            fn = dreg ? predict_acq16_kernel<true, MMA, PIPE, false, true>
                      : predict_acq16_kernel<false, MMA, PIPE, false, true>;
    }
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr;
    predict16_config(grid, stream, PIPE == PIPE_BULK_MC, cfg, attr);
    CU(cudaLaunchKernelEx(&cfg, fn, P));
    return B200BO_OK;
}

// grid of the clustered launch: two CTAs per cluster that can be resident at once, never more than one per SM
static int predict_pair_grid(b200bo_gp* g0) {
    if (g0->pair_grid > 0) return B200BO_OK;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr;
    predict16_config(2, nullptr, true, cfg, attr);
    int clusters = 0;
    CU(cudaOccupancyMaxActiveClusters(&clusters, predict_acq16_kernel<true, 1684, PIPE_BULK_MC>, &cfg));
    int nodreg = 0;
    CU(cudaOccupancyMaxActiveClusters(&nodreg, predict_acq16_kernel<false, 1684, PIPE_BULK_MC>, &cfg));
    clusters = nodreg < clusters ? nodreg : clusters;
    if (clusters < 1) return set_err(B200BO_ERR_CUDA, "predict_acq16_kernel: no CTA pair fits on the device");
    g0->pair_grid = 2 * clusters < g0->sm_count ? 2 * clusters : g0->sm_count & ~1;
    return B200BO_OK;
}

// predict_acq16_kernel's bulk-copy phase B and the Gram bound pass flag an mbarrier wait that ran out of its budget (a
// protocol error)
static int check_pipe_timeout(b200bo_gp* g0) {
    if (!g0->pipe_armed) return B200BO_OK;
    unsigned long long f = 0;
    CU(cudaSetDevice(g0->device));
    CU(cudaMemcpyFromSymbol(&f, g_pipe_timeout, sizeof(f)));
    if (f != 0) return set_err(B200BO_ERR_CUDA, "a bulk-copy pipeline wait (phase B or the Gram bound pass) timed out");
    return B200BO_OK;
}

// evict_last fraction of predict_acq16_kernel's L^-1 loads; B200BO_PREDICT_L2=<fraction in (0,1]> or "none"
// (evict_normal) overrides the measured default for A/B measurements
static float predict_linv_l2_last() {
    const char* e = getenv("B200BO_PREDICT_L2");
    if (e && strcmp(e, "none") == 0) return 0.f;
    if (e && *e) {
        const float f = strtof(e, nullptr);
        if (f > 0.f && f <= 1.f) return f;
    }
    return kDefaultLinvL2Last;
}

// selection-only pruning (DESIGN.md 4.9) of selection-only calls of the 16-warp fp64 kernel; B200BO_PRUNE=0 turns it
// off (read per call) for A/B measurements
static bool prune_enabled() {
    const char* e = getenv("B200BO_PRUNE");
    return !(e && e[0] == '0');
}

// Leading row blocks of the refine stages of pruning (DESIGN.md 4.9), or 0 when the launch keeps to the tile kernel:
// B200BO_PRUNE_REFINE=0 (read per call, for A/B measurements), fewer than 8 row blocks of L^-1 (the refined bound
// would cost a sizeable part of the exact value) or too few tiles for a lead stage.  B200BO_PRUNE_REFINE_BLOCKS (default
// 4) is clamped to an eighth of the row blocks.
static int prune_refine_blocks(int np, long long ntiles) {
    const char* e = getenv("B200BO_PRUNE_REFINE");
    const int nb = np / PBM;
    if ((e && e[0] == '0') || nb < 8 || ntiles < 4 * kLeadTiles) return 0;
    const char* eb = getenv("B200BO_PRUNE_REFINE_BLOCKS");
    int b = eb && *eb ? atoi(eb) : 4;
    b = b < 1 ? 1 : b;
    return b < nb / 8 ? b : nb / 8;
}

// survivors of the level in key order (sorted slots pos): their local indices and carried prefixes
__global__ void level_gather_kernel(const unsigned long long* __restrict__ ctl, int n_word, const int* __restrict__ pos,
                                    const int* __restrict__ idx, const double* __restrict__ pre, int* __restrict__ idx_out,
                                    double* __restrict__ pre_out) {
    const long long n = (long long)ctl[n_word] * 32;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long sl = i >> 5;
        const int q = (int)(i & 31), p = pos[sl];
        if (q == 0) idx_out[sl] = idx[p];
        pre_out[i] = pre[(size_t)p * 32 + q];
    }
}

// control words of a launch with refine stages: the tile kernel starts behind the lead tiles, and the lead stage sees
// the k-th key carried into the launch
__global__ void prune_ctl_refine_kernel(unsigned long long* ctl) {
    ctl[kCtlTile] = ctl[kCtlRefTile] = kLeadTiles;
    ctl[kCtlSurv] = ctl[kCtlUnit] = ctl[kCtlLevel] = 0ull;
    ctl[kCtlKthLead] = ctl[kCtlKth];
}

// Whether the final rounds can run (final_rounds_kernel, a cooperative launch): the device supports cooperative
// launches and `grid` CTAs of 512 threads with the phase B shared memory are co-resident (one per SM).  Checked once
// per handle; without it a call takes no refine stages.
static bool final_rounds_coop(b200bo_gp* g0, bool dreg, int grid) {
    int& ok = g0->coop_final[dreg ? 1 : 0];
    if (ok < 0) {
        int dev = 0, coop = 0, per_sm = 0;
        ok = cudaGetDevice(&dev) == cudaSuccess &&
             cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) == cudaSuccess && coop &&
             cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                 &per_sm, dreg ? final_rounds_kernel<true> : final_rounds_kernel<false>, P16_NT,
                 kPredictSmemBytesDmma) == cudaSuccess &&
             per_sm * g0->sm_count >= grid;
        cudaGetLastError();
    }
    return ok == 1;
}

// The lead, refine, level and final stages of a pruned launch (predict16.cuh), between prune_prepare and the tile
// kernel.  ks_build_kernel builds the K* of a stage's or round's tiles once, before its units.  The refine stage
// stores every survivor's prefix, the level carries it on over row blocks [b, 2b) and passes its survivors on, and
// the final stage starts from row block 2b in rounds over those survivors sorted by key, skipping the tiles above the
// key, in one cooperative launch (the caller has checked final_rounds_coop).  The k-th key is merged after the lead
// stage and after every final round.
static int prune_refine_stages(b200bo_gp* g0, const PredictParams& P, bool dreg, int blocks, bool resume,
                               cudaStream_t stream) {
    const int nb = P.gp[0].np / PBM, grid = g0->sm_count;
    const int nsurv = kRefineMaxTiles * PBN;
    int rc;
    if ((rc = g0->prune_surv.reserve(sizeof(int) * 4 * (size_t)nsurv))) return rc;
    if ((rc = g0->prune_surv_key.reserve(sizeof(unsigned long long) * 3 * (size_t)nsurv))) return rc;
    if ((rc = g0->prune_prefix.reserve(sizeof(double) * 2 * 32 * (size_t)nsurv))) return rc;
    if ((rc = g0->prune_part.reserve(sizeof(double) * (size_t)kUnitSlots * nb * 32 * PBN))) return rc;
    if ((rc = g0->prune_mu_unit.reserve(sizeof(double) * (size_t)kUnitSlots * PBN))) return rc;
    if ((rc = g0->prune_arrive.reserve(sizeof(unsigned) * kUnitSlots))) return rc;
    unsigned long long* skey = g0->prune_surv_key.as<unsigned long long>();
    int* sidx = g0->prune_surv.as<int>();
    // lists A (the refine stage's survivors) and B (the level's), the level's slots and the second key and slot buffers
    // of their sort; the sorted survivors are gathered back into list A
    unsigned long long* lkey[2] = {skey, skey + nsurv};
    int* lidx[2] = {sidx, sidx + nsurv};
    int* spos = sidx + 2 * nsurv;
    double* lpre[2] = {g0->prune_prefix.as<double>(), g0->prune_prefix.as<double>() + (size_t)32 * nsurv};
    cub::DoubleBuffer<unsigned long long> lk(lkey[1], skey + 2 * nsurv);
    cub::DoubleBuffer<int> lp(spos, sidx + 3 * nsurv);
    size_t tmp = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp, lk, lp, nsurv, 0, 64, stream));
    if ((rc = g0->prune_tmp.reserve(tmp))) return rc;
    unsigned long long* ctl = g0->prune_ctl.as<unsigned long long>();
    if (!resume) CU(cudaMemsetAsync(ctl + kCtlRefined, 0, sizeof(unsigned long long), stream));
    CU(cudaMemsetAsync(g0->prune_arrive.p, 0, sizeof(unsigned) * kUnitSlots, stream));
    prune_ctl_refine_kernel<<<1, 1, 0, stream>>>(ctl);
    LAUNCHED();
    RefineParams R = {};
    R.mu = g0->prune_mu.as<double2>();
    R.mu_unit = g0->prune_mu_unit.as<double>();
    R.surv = sidx;
    R.surv_key = skey;
    R.prefix = nullptr;
    R.part = g0->prune_part.as<double>();
    R.arrive = g0->prune_arrive.as<unsigned>();
    R.blocks = blocks;
    R.groups_max = nb / 2 < 32 ? nb / 2 : 32;
    R.final_stage = kStageLead;
    R.b0 = 0;
    R.b1 = nb;
    R.n_word = kCtlSurv;
    R.t0 = 0;
    R.t1 = kRefineMaxTiles;
    auto build = dreg ? ks_build_kernel<true> : ks_build_kernel<false>;
    const SelList* lists = g0->sel_cta.as<SelList>();
    build<<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(P, R);
    LAUNCHED();
    predict_units_kernel<<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(P, R);
    LAUNCHED();
    merge_kth_kernel<<<1, 32, 0, stream>>>(lists, grid, P.sel_k, ctl);
    LAUNCHED();
    CU(cudaEventRecord(g0->ev_stage[2], stream));
    PredictParams Q = P;  // the lead stage has begun the per-CTA lists
    Q.sel_resume = 1;
    R.prefix = lpre[0];
    if (dreg)
        predict_refine_kernel<true><<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(Q, R);
    else
        predict_refine_kernel<false><<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(Q, R);
    LAUNCHED();
    CU(cudaEventRecord(g0->ev_stage[3], stream));
    // The level: the survivors of list A, counted in kCtlSurv, over row blocks [b, 2b) into list B.  It always exists:
    // prune_refine_blocks clamps b to nb / 8 with nb >= 8, so 2b <= nb / 4 < nb.  One level is enough: at C3 (DESIGN.md
    // 4.9) it leaves 1.6 tiles of the refine stage's 12.1, and a further level cannot shorten the final round, whose
    // latency is that of its last row block.
    R.final_stage = kStageLevel;
    R.b0 = blocks;
    R.b1 = 2 * blocks;
    R.surv_out = lidx[1];
    R.surv_key_out = lkey[1];
    R.prefix_out = lpre[1];
    R.pos_out = spos;
    R.out_word = kCtlLevel;
    CU(cudaMemsetAsync(lkey[1], 0xFF, sizeof(unsigned long long) * nsurv, stream));  // unused slots sort last
    for (int t0 = 0; t0 < kRefineMaxTiles; t0 = R.t1) {
        R.t0 = t0;
        R.t1 = t0 + grid < kRefineMaxTiles ? t0 + grid : kRefineMaxTiles;
        CU(cudaMemsetAsync(ctl + kCtlUnit, 0, sizeof(unsigned long long), stream));
        build<<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(Q, R);
        LAUNCHED();
        predict_units_kernel<<<grid, P16_NT, kPredictSmemBytesDmma, stream>>>(Q, R);
        LAUNCHED();
    }
    CU(cudaEventRecord(g0->ev_stage[5], stream));
    // the level's survivors ascending by key (the sentinels of the unused slots last), sorted with their slots, then
    // their indices and prefixes gathered into list A in that order
    CU(cub::DeviceRadixSort::SortPairs(g0->prune_tmp.p, tmp, lk, lp, nsurv, 0, 64, stream));
    LAUNCHED();
    level_gather_kernel<<<2 * grid, 256, 0, stream>>>(ctl, kCtlLevel, lp.Current(), lidx[1], lpre[1], lidx[0],
                                                       lpre[0]);
    LAUNCHED();
    R.final_stage = kStageFinal;
    R.b0 = 2 * blocks;
    R.b1 = nb;
    R.n_word = kCtlLevel;
    R.surv = lidx[0];
    R.surv_key = lk.Current();
    R.prefix = lpre[0];
    CU(cudaMemsetAsync(ctl + kCtlUnit, 0, sizeof(unsigned long long), stream));
    void* args[] = {(void*)&Q, (void*)&R};
    CU(cudaLaunchCooperativeKernel(dreg ? (const void*)final_rounds_kernel<true> : (const void*)final_rounds_kernel<false>,
                                   dim3(grid), dim3(P16_NT), args, kPredictSmemBytesDmma, stream));
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaEventRecord(g0->ev_stage[4], stream));
    return B200BO_OK;
}

// Gram bound pass operand of pruning (once per fit): [np][stride] doubles, A1, Ymax, then np floats (alpha_) and np
// float pairs (the margin weights of predict_bound_gram_reg_kernel).  A1 is read back (one synchronisation per fit) for
// the choice of pass.
static int ensure_gram(b200bo_gp* gp, cudaStream_t stream) {
    if (gp->gram_valid) return B200BO_OK;
    const int np = gp->np, d = gp->d;
    int rc;
    if ((rc = gp->gram.reserve(sizeof(double) * ((size_t)np * gram_stride(d) + 2) + 3 * sizeof(float) * np)))
        return rc;
    double* img = gp->gram.as<double>();
    gram_operand_kernel<<<(np + 255) / 256, 256, 0, stream>>>(gp->Xs.as<double>(), gp->alphav.as<double>(),
                                                              (int)gp->n, np, d, cov_code(gp->family, gp->nu), img);
    LAUNCHED();
    gram_stats_kernel<<<1, 1024, 0, stream>>>(gp->alphav.as<double>(), (int)gp->n, d, img,
                                              img + (size_t)np * gram_stride(d));
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&gp->gram_a1, img + (size_t)np * gram_stride(d), sizeof(double), cudaMemcpyDeviceToHost,
                       stream));
    CU(cudaStreamSynchronize(stream));
    gp->gram_valid = true;
    return B200BO_OK;
}

// The bound passes of pruning (DESIGN.md 4.9)
enum { kBoundDirect = 0, kBoundGram64 = 1, kBoundGram32 = 2 };

// The fp32 Gram pass widens mu by about A1 constv 2^-24 times a few tens (the covariance's rounding, summed with the
// weights |alpha_i|); the fp64 Gram pass by about A1 constv 2^-53 (DESIGN.md 4.9).  Above A1 constv 2^-24 = 1e-3
// (normalised units) the fp32 interval starts to let candidates through that the fp64 one prunes, so such GPs (large
// alpha_ on an ill-conditioned K) keep the fp64 pass.  B200BO_PRUNE_BOUND=f64 / f32 (read per call) forces one of the
// Gram passes for A/B measurements; Matern-0.5 always runs the direct pass.  Needs ensure_gram.
constexpr double kPruneF32MaxMargin = 1e-3;
static int bound_pass_choice(const b200bo_gp* g0, const GpDev& G) {
    if (cov_code(G.family, G.nu) == 0) return kBoundDirect;
    const char* e = getenv("B200BO_PRUNE_BOUND");
    if (e && !strcmp(e, "f64")) return kBoundGram64;
    if (e && !strcmp(e, "f32")) return kBoundGram32;
    return g0->gram_a1 * G.constv * 0x1p-24 <= kPruneF32MaxMargin ? kBoundGram32 : kBoundGram64;
}

// The fp32 Gram pass at d <= kGramRegMaxDim runs predict_bound_gram_reg_kernel (candidate fragments in registers, the
// default) unless B200BO_PRUNE_GRAM_KERNEL=ring (read per call, for A/B measurements) picks predict_bound_gram_kernel,
// which every other d, and the fp64 Gram pass, runs.
static bool gram_reg_kernel(int d) {
    if (d > kGramRegMaxDim) return false;
    const char* e = getenv("B200BO_PRUNE_GRAM_KERNEL");
    return !(e && !strcmp(e, "ring"));
}

template <int COV>
static void launch_bound_gram_reg(const PredictParams& P, unsigned ntiles, unsigned long long* keys, int* idx,
                                  double* kmax, double2* mu, cudaStream_t stream) {
    const size_t smem = gram_reg_bound_smem(P.d);
    switch ((P.d + 2 + 3) / 4) {
        case 1: predict_bound_gram_reg_kernel<COV, 1><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        case 2: predict_bound_gram_reg_kernel<COV, 2><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        case 3: predict_bound_gram_reg_kernel<COV, 3><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        case 4: predict_bound_gram_reg_kernel<COV, 4><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        default: predict_bound_gram_reg_kernel<COV, 5><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
    }
}

template <bool F32>
static void launch_bound_gram(const PredictParams& P, unsigned long long* keys, int* idx, double* kmax, double2* mu,
                              cudaStream_t stream) {
    const unsigned ntiles = (unsigned)((P.m + kGramTile - 1) / kGramTile);
    if (F32 && gram_reg_kernel(P.d)) {
        switch (cov_code(P.gp[0].family, P.gp[0].nu)) {
            case 1: launch_bound_gram_reg<1>(P, ntiles, keys, idx, kmax, mu, stream); break;
            case 2: launch_bound_gram_reg<2>(P, ntiles, keys, idx, kmax, mu, stream); break;
            default: launch_bound_gram_reg<3>(P, ntiles, keys, idx, kmax, mu, stream); break;
        }
        return;
    }
    const size_t smem = gram_bound_smem(P.d);
    switch (cov_code(P.gp[0].family, P.gp[0].nu)) {
        case 1: predict_bound_gram_kernel<1, F32><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        case 2: predict_bound_gram_kernel<2, F32><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
        default: predict_bound_gram_kernel<3, F32><<<ntiles, kGramNT, smem, stream>>>(P, keys, idx, kmax, mu); break;
    }
}

// The bound pass of a pruned launch (kBound*; -1: bound_pass_choice): a Gram pass (distances on the fp64 tensor pipe)
// for every covariance whose dk/d(r^2) is bounded, the direct pass for Matern-0.5 (DESIGN.md 4.9).  mu: [m] interval
// (mu_lo, mu_hi); idx, kmax may be nullptr.  resume: a later launch of a chunked batch, which keeps the timeout flag.
static int launch_bound_pass(b200bo_gp* g0, PredictParams& P, int pass, unsigned long long* keys, int* idx,
                             double* kmax, double2* mu, bool resume, cudaStream_t stream) {
    if (cov_code(P.gp[0].family, P.gp[0].nu) == 0) pass = kBoundDirect;
    if (pass != kBoundDirect) {
        int rc;
        if ((rc = ensure_gram(g0, stream))) return rc;
        if (pass < 0) pass = bound_pass_choice(g0, P.gp[0]);
        P.gp[0].gram = g0->gram.as<double>();
        if (!resume) {  // the operand ring's timeout flag, read by check_pipe_timeout
            void* flag = nullptr;
            CU(cudaGetSymbolAddress(&flag, g_pipe_timeout));
            CU(cudaMemsetAsync(flag, 0, sizeof(unsigned long long), stream));
            g0->pipe_armed = true;
        }
        if (pass == kBoundGram32)
            launch_bound_gram<true>(P, keys, idx, kmax, mu, stream);
        else
            launch_bound_gram<false>(P, keys, idx, kmax, mu, stream);
    } else {
        const unsigned ntiles = (unsigned)((P.m + PBN - 1) / PBN);
        const size_t smem = sizeof(double) * ((size_t)(PBN + 2 * PA_CHUNK) * P.d + 2 * PA_CHUNK);
        if (P.d <= kPredictMaxDimRegs)
            predict_bound_kernel<true><<<ntiles, P16_NT, smem, stream>>>(P, keys, idx, kmax, mu);
        else
            predict_bound_kernel<false><<<ntiles, P16_NT, smem, stream>>>(P, keys, idx, kmax, mu);
    }
    LAUNCHED();
    CU(cudaGetLastError());
    return B200BO_OK;
}

// Bound pass + radix sort of (bound key, local index): fills P.perm / P.perm_key / P.prune_ctl for predict_acq16_kernel.
// The k-th key word and the evaluated count carry over from launch to launch of a chunked batch (resume).
static int prune_prepare(b200bo_gp* g0, PredictParams& P, bool resume, cudaStream_t stream) {
    const long long m = P.m;
    int rc;
    if ((rc = g0->prune_key.reserve(sizeof(unsigned long long) * 2 * (size_t)m))) return rc;
    if ((rc = g0->prune_idx.reserve(sizeof(int) * 2 * (size_t)m))) return rc;
    if ((rc = g0->prune_ctl.reserve(sizeof(unsigned long long) * kCtlWords))) return rc;
    if ((rc = g0->prune_mu.reserve(sizeof(double2) * (size_t)m))) return rc;
    unsigned long long* keys = g0->prune_key.as<unsigned long long>();
    int* idx = g0->prune_idx.as<int>();
    unsigned long long* ctl = g0->prune_ctl.as<unsigned long long>();
    const bool gram = cov_code(P.gp[0].family, P.gp[0].nu) != 0;
    if (gram && !g0->gram_valid) {
        if ((rc = ensure_gram(g0, stream))) return rc;
        CU(cudaEventRecord(g0->ev0, stream));  // exclude the one-off operand build from the kernel time
    }
    if ((rc = launch_bound_pass(g0, P, -1, keys, idx, nullptr, g0->prune_mu.as<double2>(), resume, stream))) return rc;
    CU(cudaEventRecord(g0->ev_stage[0], stream));
    cub::DoubleBuffer<unsigned long long> kb(keys, keys + m);
    cub::DoubleBuffer<int> ib(idx, idx + m);
    size_t tmp = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp, kb, ib, (int)m, 0, 64, stream));
    if ((rc = g0->prune_tmp.reserve(tmp))) return rc;
    CU(cub::DeviceRadixSort::SortPairs(g0->prune_tmp.p, tmp, kb, ib, (int)m, 0, 64, stream));
    LAUNCHED();
    CU(cudaMemsetAsync(ctl + kCtlTile, 0, sizeof(unsigned long long), stream));
    if (!resume) {
        CU(cudaMemsetAsync(ctl + kCtlKth, 0xFF, sizeof(unsigned long long), stream));
        CU(cudaMemsetAsync(ctl + kCtlEval, 0, sizeof(unsigned long long), stream));
    }
    CU(cudaEventRecord(g0->ev_stage[1], stream));
    P.perm = ib.Current();
    P.perm_key = kb.Current();
    P.prune_ctl = ctl;
    return B200BO_OK;
}

// padded stage images of L^-1 for the bulk-copy phase B of the fp64 kernel (once per fit)
static int ensure_pad(b200bo_gp* gp, cudaStream_t stream) {
    if (gp->pad_valid) return B200BO_OK;
    const int np = gp->np;
    int rc;
    if ((rc = gp->pad_linv.reserve(sizeof(double) * pad_linv_doubles(np)))) return rc;
    dim3 grid(np / PBK_DMMA, np / PBM);
    pad_linv_stages_kernel<<<grid, 256, 0, stream>>>(gp->WT.as<double>(), np, gp->pad_linv.as<double>());
    LAUNCHED();
    CU(cudaGetLastError());
    gp->pad_valid = true;
    return B200BO_OK;
}

// fp32 mode operand images of L^-1 (once per fit)
static int ensure_tc(b200bo_gp* gp, cudaStream_t stream) {
    if (gp->tc_valid) return B200BO_OK;
    const int np = gp->np;
    int rc;
    if ((rc = gp->tc_linv.reserve((size_t)(np / PBM) * (np / tc::kTcK) * 2 * tc::kTcImgBytes))) return rc;
    dim3 grid(np / tc::kTcK, np / PBM);
    pretile_linv_tc_kernel<<<grid, 256, 0, stream>>>(gp->W.as<double>(), np, gp->tc_linv.as<uint8_t>());
    LAUNCHED();
    CU(cudaGetLastError());
    gp->tc_valid = true;
    return B200BO_OK;
}

// B200BO_ACQ_MEAN: T = 2 B + 1 with B = |y_mean| + y_std const_value A1 of gps[0] (include/b200bo.h).  A1 = sum |alpha_|
// comes with the Gram operand of pruning (once per fit; the first call after a fit synchronises `stream`).
static int mean_merit_T(b200bo_gp* g0, cudaStream_t stream, double& T) {
    const int rc = ensure_gram(g0, stream);
    if (rc) return rc;
    T = 2.0 * (fabs(g0->y_mean) + g0->y_std * g0->constv * g0->gram_a1) + 1.0;
    return B200BO_OK;
}

// dynamic shared memory of predict_mean_kernel: phase A's staged candidates, training rows and alpha_
static size_t mean_smem_bytes(int d) { return sizeof(double) * ((size_t)(PBN + 2 * PA_CHUNK) * d + 2 * PA_CHUNK); }

static int check_spec(const b200bo_acq* spec) {
    if (!spec) return set_err(B200BO_ERR_ARG, "spec is NULL");
    if (spec->n_gps < 1 || spec->n_gps > B200BO_MAX_GPS)
        return set_err(B200BO_ERR_ARG, "n_gps=%d out of range [1,%d]", spec->n_gps, B200BO_MAX_GPS);
    if (!acq_kind_valid(spec->kind))
        return set_err(B200BO_ERR_ARG, "unknown acquisition kind %d", spec->kind);
    if (spec->path != B200BO_PATH_AUTO && spec->path != B200BO_PATH_STABLE)
        return set_err(B200BO_ERR_ARG, "unknown path policy %d", spec->path);
    for (int g = 0; g < spec->n_gps; ++g) {
        const b200bo_gp* gp = spec->gps[g];
        if (!gp) return set_err(B200BO_ERR_ARG, "gps[%d] is NULL", g);
        if (!gp->fitted) return set_err(B200BO_ERR_STATE, "gps[%d] is not fitted", g);
        if (gp->d != spec->gps[0]->d) return set_err(B200BO_ERR_ARG, "gps[%d] has a different dimension", g);
        if (gp->device != spec->gps[0]->device)
            return set_err(B200BO_ERR_ARG, "gps[%d] lives on a different device", g);
        if (g >= 1 && !(spec->lb[g] < spec->ub[g]))
            return set_err(B200BO_ERR_ARG, "constraint %d: lb must be < ub", g);
    }
    if (spec->kind == B200BO_ACQ_MES && spec->gps[0]->ystar.empty())
        return set_err(B200BO_ERR_STATE, "MES: gps[0] holds no samples of the maximum (b200bo_gp_set_max_values)");
    if (acq_is_nei(spec->kind) && spec->gps[0]->fant_best.empty())
        return set_err(B200BO_ERR_STATE, "NEI: gps[0] holds no fantasies (b200bo_gp_set_fantasies)");
    if (acq_is_cnei(spec->kind)) {  // every GP a noiseless handle with fantasies of the same S and n
        const b200bo_gp* g0 = spec->gps[0];
        for (int g = 0; g < spec->n_gps; ++g) {
            const b200bo_gp* gp = spec->gps[g];
            if (gp->fant_best.empty())
                return set_err(B200BO_ERR_STATE, "CNEI: gps[%d] holds no fantasies (b200bo_gp_set_fantasies)", g);
            if (gp->fant_best.size() != g0->fant_best.size())
                return set_err(B200BO_ERR_ARG, "CNEI: gps[%d] holds %d fantasies, gps[0] %d", g,
                               (int)gp->fant_best.size(), (int)g0->fant_best.size());
            if (gp->n != g0->n || gp->np != g0->np)
                return set_err(B200BO_ERR_ARG, "CNEI: gps[%d] has a different training set size", g);
        }
    }
    return B200BO_OK;
}

// Where a launch's candidates come from: a device matrix (parity mode: the reference's host MT19937 stream,
// uploaded) or the in-kernel Philox generator (throughput mode).
struct CandSrc {
    const double* d_Xc = nullptr;
    bool philox = false;
    uint64_t seed = 0;
    const double* lo = nullptr;  // host, d entries
    const double* hi = nullptr;
};

// resume != 0: the per-CTA selection lists of the previous launch on this handle are continued instead of
// re-initialised (chunked batches: one merge after the last chunk); finish == 0 skips the merge.
struct SelMode {
    int resume = 0;
    int finish = 1;
};

// Philox bounds of the throughput mode as the kernels read them: pb = (lo_j, hi_j - lo_j), 2 d entries
static int pack_pbounds(const double* lo, const double* hi, int d, double* pb) {
    for (int j = 0; j < d; ++j) {
        if (!(lo[j] <= hi[j])) return set_err(B200BO_ERR_ARG, "Philox bounds: lo > hi in column %d", j);
        pb[j] = lo[j];
        pb[d + j] = hi[j] - lo[j];
    }
    return B200BO_OK;
}

// launch parameters of the predict kernels for spec over the candidates of src (everything but outputs and scratch);
// np_max: the largest padded training size of the spec's GPs
static int fill_params(const b200bo_acq* spec, const CandSrc& src, int64_t m, int64_t index_base, cudaStream_t stream,
                       PredictParams& P, int& np_max) {
    int rc;
    b200bo_gp* g0 = spec->gps[0];
    memset(&P, 0, sizeof(P));
    np_max = 0;
    for (int g = 0; g < spec->n_gps; ++g) {
        b200bo_gp* gp = spec->gps[g];
        GpDev& G = P.gp[g];
        G.Xs = gp->Xs.as<double>();
        G.linvT = gp->WT.as<double>();
        G.alphav = gp->alphav.as<double>();
        G.ls = gp->ls.as<double>();
        G.xform = gp->xform.empty() ? nullptr : gp->xf.as<int>();
        G.linv_tc = nullptr;
        G.n = (int)gp->n;
        G.np = gp->np;
        G.family = gp->family;
        G.nu = gp->nu;
        G.constv = gp->constv;
        G.prior = gp->constv + gp->noise;
        G.kdiag = gp->constv + gp->jitter;
        G.y_mean = gp->y_mean;
        G.y_std = gp->y_std;
        G.lb = spec->lb[g];
        G.ub = spec->ub[g];
        np_max = gp->np > np_max ? gp->np : np_max;
    }
    P.n_gps = spec->n_gps;
    P.d = g0->d;
    P.acq_kind = spec->kind;
    P.kappa = spec->kappa;
    P.xi = spec->xi;
    P.y_max = spec->y_max;
    if (spec->kind == B200BO_ACQ_MES) {
        P.n_ystar = (int)g0->ystar.size();
        for (int k = 0; k < P.n_ystar; ++k) P.ystar[k] = g0->ystar[k];
    } else if (acq_uses_fantasies(spec->kind)) {  // A and best_s on the device
        P.n_ystar = (int)g0->fant_best.size();
        P.fant_a = g0->fant_a.as<double>();
        if (acq_is_cnei(spec->kind))
            for (int g = 0; g < spec->n_gps; ++g) P.fant_a_gp[g] = spec->gps[g]->fant_a.as<double>();
    }
    P.Xc = src.philox ? nullptr : src.d_Xc;
    P.index_base = index_base;
    if (src.philox) {
        double pb[2 * B200BO_MAX_DIM];
        if ((rc = pack_pbounds(src.lo, src.hi, P.d, pb))) return rc;
        if ((rc = g0->pbounds.reserve(sizeof(double) * 2 * B200BO_MAX_DIM))) return rc;
        CU(cudaMemcpyAsync(g0->pbounds.p, pb, sizeof(double) * 2 * P.d, cudaMemcpyHostToDevice, stream));
        P.pbounds = g0->pbounds.as<double>();
        P.seed = src.seed;
    }
    P.m = m;
    return B200BO_OK;
}

// The small-batch kernels over the m candidates of S.P (predict_kernels.cuh).  Per launch group of up to SMAXP passes
// and per GP: K*, v = L^-1 k* and its sums; grad adds u = L^-T v and the gradient partials into S.grad_out.  Then one
// finish for every GP.
static int small_launch(const b200bo_acq* spec, SmallParams& S, int64_t m, bool grad, cudaStream_t stream) {
    b200bo_gp* g0 = spec->gps[0];
    const bool nei = acq_is_nei(spec->kind), cnei = acq_is_cnei(spec->kind), mean = spec->kind == B200BO_ACQ_MEAN;
    int rc;
    for (int g = 0; g < spec->n_gps; ++g) {
        b200bo_gp* gp = spec->gps[g];
        if ((rc = ensure_small(gp, grad))) return rc;
        SmallGp& Q = S.sg[g];
        Q.W = gp->W.as<double>();
        Q.ksm = gp->s_ksm.as<double>();
        Q.partial = gp->s_partial.as<double>();
        Q.mu_part = gp->s_mupart.as<double>();
        Q.colsq_rb = gp->s_colsq.as<double>();
        Q.unit_tab = gp->s_unit.as<int2>();
        Q.rb_tab = gp->s_rb.as<int2>();
        S.nunits[g] = gp->s_nunits;
        // S mean lists + the u list per block (small_grad_kernel<true>): gps[0] of NEI, every GP of CNEI
        if (grad && ((g == 0 && nei) || cnei)) {
            const size_t lists = g0->fant_best.size() + 1;
            if ((rc = gp->s_gpart.reserve(sizeof(double) * (size_t)SMAXP * (gp->np / 128) * lists * gp->d * SMC)))
                return rc;
        }
        if (grad) {
            Q.vsum = gp->s_vsum.as<double>();
            Q.usum = gp->s_usum.as<double>();
            Q.partial_u = gp->s_partial_u.as<double>();
            Q.gpart = gp->s_gpart.as<double>();
            Q.unit_tab_u = gp->s_unit_u.as<int2>();
            Q.rb_tab_u = gp->s_rb_u.as<int2>();
            S.nunits_u[g] = gp->s_nunits_u;
        }
    }
    S.m_end = m;
    CU(cudaEventRecord(g0->ev0, stream));
    for (long long c0 = 0; c0 < m; c0 += (long long)SMAXP * SMC) {
        S.c0 = c0;
        const long long left = m - c0;
        const int npass = (int)((left + SMC - 1) / SMC < SMAXP ? (left + SMC - 1) / SMC : SMAXP);
        const int ngrp = (npass + STPG - 1) / STPG;
        for (int g = 0; g < spec->n_gps; ++g) {
            const b200bo_gp* gp = spec->gps[g];
            small_kstar_kernel<<<dim3(gp->np / 128, npass), 256, 0, stream>>>(S, g);
            LAUNCHED();
            if (mean) {  // K* alpha_ only: no triangular product, no sums of squares
                if (grad) {
                    small_grad_kernel<false, false, true><<<dim3(gp->np / 128, npass), 256, 0, stream>>>(S, g);
                    LAUNCHED();
                }
                continue;
            }
            small_trsv_kernel<false><<<dim3(gp->s_nunits, ngrp), 256, kSmallTrsvSmemBytes, stream>>>(S, g, npass);
            if (grad) {
                small_reduce_kernel<1><<<dim3(gp->np / SROWS, npass), 256, 0, stream>>>(S, g);
                small_trsv_kernel<true><<<dim3(gp->s_nunits_u, ngrp), 256, kSmallTrsvSmemBytes, stream>>>(S, g, npass);
                small_reduce_kernel<2><<<dim3(gp->np / SROWS, npass), 256, 0, stream>>>(S, g);
                if (cnei)
                    small_grad_kernel<true, true><<<dim3(gp->np / 128, npass, (unsigned)g0->fant_best.size()), 256,
                                                    0, stream>>>(S, g);
                else if (nei && g == 0)
                    small_grad_kernel<true><<<dim3(gp->np / 128, npass, (unsigned)g0->fant_best.size()), 256, 0,
                                              stream>>>(S, g);
                else
                    small_grad_kernel<false><<<dim3(gp->np / 128, npass), 256, 0, stream>>>(S, g);
            } else {
                small_reduce_kernel<0><<<dim3(gp->np / SROWS, npass), 256, 0, stream>>>(S, g);
            }
            for (int i = 0; i < (grad ? 5 : 2); ++i) LAUNCHED();
        }
        if (mean)
            (grad ? small_finish_mean_kernel<true> : small_finish_mean_kernel<false>)<<<npass, 256, 0, stream>>>(S);
        else if (grad && cnei)
            small_finish_grad_cnei_kernel<<<npass, 256, 0, stream>>>(S);
        else if (grad)
            (nei ? small_finish_grad_kernel<true> : small_finish_grad_kernel<false>)<<<npass, 256, 0, stream>>>(S);
        else if (nei)
            small_finish_kernel<true><<<npass, 256, 0, stream>>>(S);
        else if (cnei)
            small_finish_kernel<false, true><<<npass, 256, 0, stream>>>(S);
        else
            small_finish_kernel<false><<<npass, 256, 0, stream>>>(S);
        LAUNCHED();
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(g0->ev1, stream));
    g_last_timed = g0;
    return B200BO_OK;
}

// Pruned selection batches are cut into launches of at most this many candidates: the bound keys, indices and sort
// buffers take 24 bytes per candidate (about 100 MB here), whatever the size of a Philox batch.
constexpr long long kPruneMaxBatch = 1ll << 22;

static int eval_launch(const b200bo_acq* spec, const CandSrc& src, int64_t m, double* d_acq_neg, double* d_mu,
                       double* d_sd, int k, void* d_sel, int64_t index_base, cudaStream_t stream, SelMode sm);

static int eval_core(const b200bo_acq* spec, const CandSrc& src, int64_t m, double* d_acq_neg, double* d_mu,
                     double* d_sd, int k, void* d_sel, int64_t index_base, cudaStream_t stream,
                     SelMode sm = SelMode()) {
    const bool split = k > 0 && !d_acq_neg && !d_mu && !d_sd && m > kPruneMaxBatch && prune_enabled() && spec &&
                       spec->gps[0] && spec->kind != B200BO_ACQ_MEAN;
    if (!split) return eval_launch(spec, src, m, d_acq_neg, d_mu, d_sd, k, d_sel, index_base, stream, sm);
    // consecutive launches continue the per-CTA selection lists (and the pruning's k-th key), one merge at the end
    for (long long c0 = 0; c0 < m; c0 += kPruneMaxBatch) {
        const long long mc = m - c0 < kPruneMaxBatch ? m - c0 : kPruneMaxBatch;
        CandSrc s = src;
        if (!s.philox && s.d_Xc) s.d_Xc += (size_t)c0 * spec->gps[0]->d;
        SelMode part;
        part.resume = sm.resume || c0 > 0;
        part.finish = sm.finish && c0 + mc >= m;
        const int rc = eval_launch(spec, s, mc, nullptr, nullptr, nullptr, k, d_sel, index_base + c0, stream, part);
        if (rc) return rc;
    }
    return B200BO_OK;
}

static int eval_launch(const b200bo_acq* spec, const CandSrc& src, int64_t m, double* d_acq_neg, double* d_mu,
                       double* d_sd, int k, void* d_sel, int64_t index_base, cudaStream_t stream, SelMode sm) {
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (m < 0 || (m > 0 && !src.philox && !src.d_Xc)) return set_err(B200BO_ERR_ARG, "bad candidates");
    if (src.philox && (!src.lo || !src.hi)) return set_err(B200BO_ERR_ARG, "Philox mode needs lo/hi");
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (k > 0 && !d_sel) return set_err(B200BO_ERR_ARG, "d_sel is NULL");
    b200bo_gp* g0 = spec->gps[0];
    // NEI / LogNEI, CNEI / LogCNEI: no single mean to report; always fp64 (the 16-warp kernel or the small-batch
    // kernels)
    const bool nei = acq_uses_fantasies(spec->kind);
    if (nei && (d_mu || d_sd))
        return set_err(B200BO_ERR_ARG, "NEI averages over fantasies and has no single posterior mean: mu / sd outputs "
                                       "are not available");
    const bool mean = spec->kind == B200BO_ACQ_MEAN;
    if (mean && d_sd)
        return set_err(B200BO_ERR_ARG, "the posterior-mean merit needs no sigma and does not form it: the sd output is "
                                       "not available");
    const int precision = nei ? B200BO_PRECISION_FP64 : g0->precision;
    CU(cudaSetDevice(g0->device));
    NvtxRange nvtx_range("b200bo:predict_acq");
    PredictParams P;
    int np_max = 0;
    if ((rc = fill_params(spec, src, m, index_base, stream, P, np_max))) return rc;
    if (mean && spec->n_gps > 1 && (rc = mean_merit_T(g0, stream, P.mean_T))) return rc;
    P.acq_out = d_acq_neg;
    P.mu_out = d_mu;
    P.sd_out = d_sd;
    if ((rc = g0->clamp.reserve(2 * sizeof(unsigned long long)))) return rc;
    P.clamp_count = g0->clamp.as<unsigned long long>();
    if (!sm.resume) CU(cudaMemsetAsync(g0->clamp.p, 0, 2 * sizeof(unsigned long long), stream));
    const long long ntiles = (m + PBN - 1) / PBN;
    int grid = (int)(ntiles < g0->sm_count ? ntiles : g0->sm_count);
    if (sm.resume || !sm.finish) grid = g0->sm_count;  // chunked batches keep one list per SM across launches
    const bool small = grid > 0 && !sm.resume && sm.finish &&
                       use_small_path(m, np_max, spec->n_gps, g0->sm_count, spec->path);
    bool fused_sel = false, prune = false;
    if (small) {
        if (k > 0 && !P.acq_out) {  // the small path selects from the materialised values
            if ((rc = g0->out_acq.reserve(sizeof(double) * (size_t)(m > 0 ? m : 1)))) return rc;
            P.acq_out = g0->out_acq.as<double>();
        }
        SmallParams S;
        memset(&S, 0, sizeof(S));
        S.P = P;
        if ((rc = small_launch(spec, S, m, false, stream))) return rc;
    } else if (grid > 0 && mean) {
        // fp64 whatever the handle's precision, never pruned; chunked batches keep one list per CTA across launches
        const bool dreg = P.d <= kPredictMaxDimRegs;
        const size_t smem = mean_smem_bytes(P.d);
        int per_sm = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
            &per_sm, dreg ? predict_mean_kernel<true> : predict_mean_kernel<false>, P16_NT, smem));
        const int full = g0->sm_count * (per_sm > 0 ? per_sm : 1);
        grid = (sm.resume || !sm.finish || ntiles >= full) ? full : (int)ntiles;
        if (k > 0) {
            if ((rc = g0->sel_cta.reserve(sizeof(SelList) * (size_t)full))) return rc;
            P.sel_cta = g0->sel_cta.as<SelList>();
            P.sel_k = k;
            P.sel_resume = sm.resume;
            fused_sel = true;
        }
        CU(cudaEventRecord(g0->ev0, stream));
        (dreg ? predict_mean_kernel<true> : predict_mean_kernel<false>)<<<grid, P16_NT, smem, stream>>>(P);
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaEventRecord(g0->ev1, stream));
        g_last_timed = g0;
    } else if (grid > 0) {
        if (k > 0) {  // selection fused into the epilogue: no acq[M] needed
            if ((rc = g0->sel_cta.reserve(sizeof(SelList) * (size_t)g0->sm_count))) return rc;
            P.sel_cta = g0->sel_cta.as<SelList>();
            P.sel_k = k;
            P.sel_resume = sm.resume;
            fused_sel = true;
        }
        // phase B path of the 16-warp fp64 kernel; the bulk-copy paths read K* in the padded stage layout
        const bool fp64_16 = predict_impl(precision) == PREDICT_IMPL_DMMA && predict_warps() == 16;
        if (nei && !fp64_16)
            return set_err(B200BO_ERR_UNSUPPORTED, "NEI runs on the 16-warp fp64 kernel only (B200BO_PREDICT_IMPL / "
                                                   "B200BO_PREDICT_WARPS select a kernel without it)");
        const int pipe = fp64_16 && predict_mma() != 884 ? predict_pipe() : PIPE_CPASYNC;
        if (nei && (pipe == PIPE_CPASYNC || predict_mma() == 884))
            return set_err(B200BO_ERR_UNSUPPORTED, "NEI runs on the bulk-copy phase-B pipes only (B200BO_PREDICT_PIPE="
                                                   "cpasync / B200BO_PREDICT_MMA=884 select a pipe without it)");
        P.scratch_stride = (long long)np_max * (pipe == PIPE_CPASYNC ? PBN : PSTR_DMMA);
        if (acq_is_cnei(spec->kind)) {  // the per-sample carry of CNEI behind K*, one column per candidate
            P.carry_off = P.scratch_stride;
            P.scratch_stride += (long long)P.n_ystar * PSTR_DMMA;
        }
        if ((rc = g0->pscratch.reserve(sizeof(double) * (size_t)P.scratch_stride * g0->sm_count))) return rc;
        P.scratch = g0->pscratch.as<double>();
        CU(cudaEventRecord(g0->ev0, stream));
        const bool dreg = P.d <= kPredictMaxDimRegs;
        if (predict_impl(precision) == PREDICT_IMPL_TF32) {
            for (int g = 0; g < spec->n_gps; ++g) {
                if ((rc = ensure_tc(spec->gps[g], stream))) return rc;
                P.gp[g].linv_tc = spec->gps[g]->tc_linv.as<uint8_t>();
            }
            CU(cudaEventRecord(g0->ev0, stream));  // exclude the one-off tiling from the kernel time
            if (dreg) {
                predict_acq_tc_kernel<true><<<grid, PNT, kPredictSmemBytesTc, stream>>>(P);
            } else {
                predict_acq_tc_kernel<false><<<grid, PNT, kPredictSmemBytesTc, stream>>>(P);
            }
        } else if (fp64_16) {
            P.linv_l2_last = predict_linv_l2_last();
            if (pipe != PIPE_CPASYNC) {
                for (int g = 0; g < spec->n_gps; ++g) {
                    if ((rc = ensure_pad(spec->gps[g], stream))) return rc;
                    P.gp[g].linv_pad = spec->gps[g]->pad_linv.as<double>();
                }
                if (!sm.resume) {
                    void* flag = nullptr;
                    CU(cudaGetSymbolAddress(&flag, g_pipe_timeout));
                    CU(cudaMemsetAsync(flag, 0, sizeof(unsigned long long), stream));
                    g0->pipe_armed = true;
                }
                CU(cudaEventRecord(g0->ev0, stream));  // exclude the one-off staging from the kernel time
            }
            prune = fused_sel && !P.acq_out && !P.mu_out && !P.sd_out && P.n_gps == 1 && pipe != PIPE_BULK_MC &&
                    acq_prunable(spec->kind) && m <= std::numeric_limits<int>::max() && prune_enabled();
            if (prune && (rc = prune_prepare(g0, P, sm.resume, stream))) return rc;
            const int refine = prune && predict_mma() == 1684 && final_rounds_coop(g0, dreg, g0->sm_count)
                                   ? prune_refine_blocks(P.gp[0].np, ntiles)
                                   : 0;
            g0->stage_refined = refine > 0;
            if (refine) {
                // every SM keeps a list, begun by the lead stage and continued by the final stage and the tile kernel
                grid = g0->sm_count;
                if ((rc = prune_refine_stages(g0, P, dreg, refine, sm.resume, stream))) return rc;
                P.sel_resume = 1;
            }
            if (predict_mma() == 884) {
                rc = launch_predict16<884, PIPE_CPASYNC>(dreg, grid, stream, P);
            } else if (pipe == PIPE_BULK_MC) {
                // whole CTA pairs, each pair running the same number of tiles (see predict_acq16_kernel)
                if ((rc = predict_pair_grid(g0))) return rc;
                const long long pairs = (ntiles + 1) / 2;
                grid = (sm.resume || !sm.finish || pairs >= g0->pair_grid / 2) ? g0->pair_grid : (int)(2 * pairs);
                rc = launch_predict16<1684, PIPE_BULK_MC>(dreg, grid, stream, P);
            } else if (pipe == PIPE_BULK) {
                rc = launch_predict16<1684, PIPE_BULK>(dreg, grid, stream, P);
            } else {
                rc = launch_predict16<1684, PIPE_CPASYNC>(dreg, grid, stream, P);
            }
            if (rc) return rc;
        } else if (predict_impl(precision) == PREDICT_IMPL_DMMA) {
            if (dreg)
                predict_acq_kernel<PREDICT_IMPL_DMMA, true><<<grid, PNT, kPredictSmemBytesDmma, stream>>>(P);
            else
                predict_acq_kernel<PREDICT_IMPL_DMMA, false><<<grid, PNT, kPredictSmemBytesDmma, stream>>>(P);
        } else {
            if (dreg)
                predict_acq_kernel<PREDICT_IMPL_DFMA, true><<<grid, PNT, kPredictSmemBytesDfma, stream>>>(P);
            else
                predict_acq_kernel<PREDICT_IMPL_DFMA, false><<<grid, PNT, kPredictSmemBytesDfma, stream>>>(P);
        }
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaEventRecord(g0->ev1, stream));
        g_last_timed = g0;
    }
    if (!sm.resume) {
        g0->stat_total = g0->stat_direct = 0;
        g0->prune_counted = false;
    }
    g0->stat_total += m;
    g0->stage_timed = prune;
    if (prune)
        g0->prune_counted = true;
    else
        g0->stat_direct += m;
    if (k > 0 && sm.finish) {
        NvtxRange nvtx_sel("b200bo:select");
        if (fused_sel) {
            merge_sel_kernel<<<1, 256, 0, stream>>>(g0->sel_cta.as<SelList>(), grid, k,
                                                    reinterpret_cast<SelRecord*>(d_sel));
        } else if (m > 0) {
            select_kernel<<<1, 1024, 0, stream>>>(P.acq_out, m, k, reinterpret_cast<SelRecord*>(d_sel), index_base);
        } else {
            CU(cudaMemsetAsync(d_sel, 0xFF, sizeof(SelRecord) * (k + 1), stream));  // empty: index -1, value NaN
        }
        LAUNCHED();
        CU(cudaGetLastError());
    }
    return B200BO_OK;
}

extern "C" int b200bo_acq_eval_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m,
                                   double* d_acq_neg, double* d_mu, double* d_sd, int k, void* d_sel,
                                   int64_t index_base, void* stream_) {
    CandSrc src;
    src.d_Xc = d_Xc;
    return eval_core(spec, src, m, d_acq_neg, d_mu, d_sd, k, d_sel, index_base, (cudaStream_t)stream_);
}

// the bound pass alone (kBound*); d_mu (Gram only): [m][2] (mu_lo, mu_hi)
static int prune_bound_entry(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key, double* d_kmax,
                             double* d_mu, int pass, void* stream_) {
    const bool gram = pass != kBoundDirect;
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (spec->n_gps != 1 || !acq_prunable(spec->kind))
        return set_err(B200BO_ERR_ARG, "the pruning bound covers EI, UCB, PoI, LogEI and LogPoI on one GP");
    if (m <= 0 || m > std::numeric_limits<int>::max() || !d_Xc || !d_key)
        return set_err(B200BO_ERR_ARG, "bad candidates or key buffer");
    b200bo_gp* g0 = spec->gps[0];
    if (gram && cov_code(g0->family, g0->nu) == 0)
        return set_err(B200BO_ERR_UNSUPPORTED, "Matern-0.5 has no Gram bound (dk/d(r^2) is unbounded at r = 0)");
    CU(cudaSetDevice(g0->device));
    const cudaStream_t stream = (cudaStream_t)stream_;
    CandSrc src;
    src.d_Xc = d_Xc;
    PredictParams P;
    int np_max = 0;
    if ((rc = fill_params(spec, src, m, 0, stream, P, np_max))) return rc;
    return launch_bound_pass(g0, P, pass, reinterpret_cast<unsigned long long*>(d_key), nullptr, d_kmax,
                             reinterpret_cast<double2*>(d_mu), false, stream);
}

extern "C" int b200bo_acq_prune_bound_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key,
                                          double* d_kmax, void* stream_) {
    return prune_bound_entry(spec, d_Xc, m, d_key, d_kmax, nullptr, kBoundDirect, stream_);
}

extern "C" int b200bo_acq_prune_bound_gram_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key,
                                               double* d_mu, double* d_kmax_lb, void* stream_) {
    return prune_bound_entry(spec, d_Xc, m, d_key, d_kmax_lb, d_mu, kBoundGram64, stream_);
}

extern "C" int b200bo_acq_prune_bound_gram32_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m,
                                                 uint64_t* d_key, double* d_mu, double* d_kmax_lb, void* stream_) {
    return prune_bound_entry(spec, d_Xc, m, d_key, d_kmax_lb, d_mu, kBoundGram32, stream_);
}

extern "C" int b200bo_acq_prune_bound_pass(const b200bo_acq* spec, int* pass, void* stream_) {
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (spec->n_gps != 1 || !pass) return set_err(B200BO_ERR_ARG, "one GP and a result pointer");
    b200bo_gp* g0 = spec->gps[0];
    CU(cudaSetDevice(g0->device));
    if (cov_code(g0->family, g0->nu) != 0 && (rc = ensure_gram(g0, (cudaStream_t)stream_))) return rc;
    GpDev G;
    G.family = g0->family;
    G.nu = g0->nu;
    G.constv = g0->constv;
    *pass = bound_pass_choice(g0, G);
    return B200BO_OK;
}

// the fp32 covariance of the fp32 Gram pass on n fp32 arguments (tests)
template <int COV>
__global__ void cov_f32_kernel(const float* __restrict__ s, int64_t n, float* __restrict__ k, float* __restrict__ z) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float zi;
        k[i] = cov_f32<COV>((double)s[i], zi);
        if (z) z[i] = zi;
    }
}

extern "C" int b200bo_cov_f32_dev(int family, int nu, const float* d_s, int64_t n, float* d_k, float* d_z,
                                  void* stream_) {
    const int cov = cov_code(family, nu);
    if (cov == 0) return set_err(B200BO_ERR_UNSUPPORTED, "Matern-0.5 has no fp32 Gram pass");
    if (n <= 0 || !d_s || !d_k) return set_err(B200BO_ERR_ARG, "bad arguments");
    const cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
    if (cov == 1) cov_f32_kernel<1><<<grid, 256, 0, stream>>>(d_s, n, d_k, d_z);
    else if (cov == 2) cov_f32_kernel<2><<<grid, 256, 0, stream>>>(d_s, n, d_k, d_z);
    else cov_f32_kernel<3><<<grid, 256, 0, stream>>>(d_s, n, d_k, d_z);
    LAUNCHED();
    CU(cudaGetLastError());
    return B200BO_OK;
}

extern "C" int b200bo_acq_select_philox_dev(const b200bo_acq* spec, uint64_t seed, const double* lo,
                                            const double* hi, int64_t m, int64_t index_base, int k, void* d_sel,
                                            void* stream_) {
    if (k <= 0) return set_err(B200BO_ERR_ARG, "k must be > 0");
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    CandSrc src;
    src.philox = true;
    src.seed = seed;
    src.lo = lo;
    src.hi = hi;
    return eval_core(spec, src, m, nullptr, nullptr, nullptr, k, d_sel, index_base, (cudaStream_t)stream_);
}

extern "C" int b200bo_last_kernel_ms(float* ms) {
    if (!ms) return set_err(B200BO_ERR_ARG, "ms is NULL");
    if (!g_last_timed) return set_err(B200BO_ERR_STATE, "no timed kernel on this thread");
    CU(cudaSetDevice(g_last_timed->device));
    CU(cudaEventSynchronize(g_last_timed->ev1));
    CU(cudaEventElapsedTime(ms, g_last_timed->ev0, g_last_timed->ev1));
    return check_pipe_timeout(g_last_timed);
}

extern "C" int b200bo_last_prune_stats(int64_t* evaluated, int64_t* total) {
    if (!evaluated || !total) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!g_last_timed) return set_err(B200BO_ERR_STATE, "no timed kernel on this thread");
    b200bo_gp* g0 = g_last_timed;
    CU(cudaSetDevice(g0->device));
    CU(cudaEventSynchronize(g0->ev1));
    unsigned long long pruned_eval = 0;
    if (g0->prune_counted) CU(cudaMemcpy(&pruned_eval, g0->prune_ctl.as<unsigned long long>() + kCtlEval, sizeof(pruned_eval),
                                         cudaMemcpyDeviceToHost));
    *evaluated = g0->stat_direct + (int64_t)pruned_eval;
    *total = g0->stat_total;
    return B200BO_OK;
}

extern "C" int b200bo_last_prune_stage_ms(float* ms, int64_t* refined) {
    if (!ms || !refined) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!g_last_timed) return set_err(B200BO_ERR_STATE, "no timed kernel on this thread");
    b200bo_gp* g0 = g_last_timed;
    if (!g0->stage_timed) return set_err(B200BO_ERR_STATE, "the last launch on this thread was not pruned");
    CU(cudaSetDevice(g0->device));
    CU(cudaEventSynchronize(g0->ev1));
    for (int i = 0; i < 6; ++i) ms[i] = 0.f;
    *refined = 0;
    CU(cudaEventElapsedTime(&ms[0], g0->ev0, g0->ev_stage[0]));
    CU(cudaEventElapsedTime(&ms[1], g0->ev_stage[0], g0->ev_stage[1]));
    cudaEvent_t last = g0->ev_stage[1];
    if (g0->stage_refined) {  // the refine levels are counted with the refine stage
        CU(cudaEventElapsedTime(&ms[2], g0->ev_stage[1], g0->ev_stage[2]));
        CU(cudaEventElapsedTime(&ms[3], g0->ev_stage[2], g0->ev_stage[5]));
        CU(cudaEventElapsedTime(&ms[4], g0->ev_stage[5], g0->ev_stage[4]));
        last = g0->ev_stage[4];
        unsigned long long n = 0;
        CU(cudaMemcpy(&n, g0->prune_ctl.as<unsigned long long>() + kCtlRefined, sizeof(n), cudaMemcpyDeviceToHost));
        *refined = (int64_t)n;
    }
    CU(cudaEventElapsedTime(&ms[5], last, g0->ev1));
    return B200BO_OK;
}

extern "C" int b200bo_last_prune_levels(float* ms, int64_t* passed, int* levels) {
    if (!ms || !passed || !levels) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!g_last_timed) return set_err(B200BO_ERR_STATE, "no timed kernel on this thread");
    b200bo_gp* g0 = g_last_timed;
    if (!g0->stage_timed) return set_err(B200BO_ERR_STATE, "the last launch on this thread was not pruned");
    CU(cudaSetDevice(g0->device));
    CU(cudaEventSynchronize(g0->ev1));
    *ms = 0.f;
    *levels = g0->stage_refined ? 1 : 0;
    for (int l = 0; l < 5; ++l) passed[l] = 0;
    if (!g0->stage_refined) return B200BO_OK;
    CU(cudaEventElapsedTime(ms, g0->ev_stage[3], g0->ev_stage[5]));
    unsigned long long w[kCtlWords];
    CU(cudaMemcpy(w, g0->prune_ctl.as<unsigned long long>(), sizeof(w), cudaMemcpyDeviceToHost));
    passed[0] = (int64_t)w[kCtlSurv];
    passed[1] = (int64_t)w[kCtlLevel];
    return B200BO_OK;
}

// Host-buffer front end shared by predict / acq_eval / argmin_topk.  Large selection-only batches are
// streamed: the candidate matrix goes up in chunks of a whole number of tiles per SM on a copy stream while
// the previous chunk is evaluated (double-buffered device chunks), the per-CTA selection lists carry over
// from launch to launch and are merged once - the H2D copy disappears behind the kernel.
constexpr long long kChunkTilesPerSm = 8;

int ChunkedUpload::ensure() {
    if (!copy) {
        CU(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
        CU(cudaStreamCreateWithFlags(&exec, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CU(cudaEventCreateWithFlags(&up[i], cudaEventDisableTiming));
            CU(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
        }
    }
    return B200BO_OK;
}

template <class Launch>
int ChunkedUpload::run(const double* Xc, long long m, int d, long long chunk, double* const buf[2], Launch launch) {
    int rc, i = 0;
    for (long long c0 = 0; c0 < m; c0 += chunk, ++i) {
        const long long mc = (m - c0) < chunk ? (m - c0) : chunk;
        const int b = i & 1;
        if (i >= 2) CU(cudaStreamWaitEvent(copy, done[b], 0));  // buffer b consumed
        CU(cudaMemcpyAsync(buf[b], Xc + (size_t)c0 * d, sizeof(double) * (size_t)mc * d, cudaMemcpyHostToDevice, copy));
        CU(cudaEventRecord(up[b], copy));
        CU(cudaStreamWaitEvent(exec, up[b], 0));
        if ((rc = launch(buf[b], mc, c0, i, c0 + chunk >= m))) return rc;
        CU(cudaEventRecord(done[b], exec));
    }
    return B200BO_OK;
}

// sklearn's validate_data rejects NaN / inf in X; the kernels count them while loading the candidates
static int check_nonfinite(b200bo_gp* g0) {
    unsigned long long c[2] = {0, 0};
    CU(cudaMemcpy(c, g0->clamp.p, sizeof(c), cudaMemcpyDeviceToHost));
    if (c[1] != 0) return set_err(B200BO_ERR_ARG, "Input X contains NaN or infinity.");
    return check_pipe_timeout(g0);
}

static int run_host_chunked(const b200bo_acq* spec, const double* Xc, int64_t m, int k, SelRecord* sel_host) {
    b200bo_gp* g0 = spec->gps[0];
    int rc;
    ChunkedUpload& U = g0->upload;
    if ((rc = U.ensure())) return rc;
    const int d = g0->d;
    const long long chunk = kChunkTilesPerSm * PBN * g0->sm_count;
    if ((rc = g0->xc.reserve(sizeof(double) * (size_t)2 * chunk * d))) return rc;
    if ((rc = g0->sel.reserve(sizeof(SelRecord) * (B200BO_MAX_TOPK + 1)))) return rc;
    double* const buf[2] = {g0->xc.as<double>(), g0->xc.as<double>() + (size_t)chunk * d};
    rc = U.run(Xc, m, d, chunk, buf, [&](const double* dx, long long mc, long long c0, int i, bool last) {
        CandSrc src;
        src.d_Xc = dx;
        SelMode sm;
        sm.resume = i > 0;
        sm.finish = last;
        return eval_core(spec, src, mc, nullptr, nullptr, nullptr, k, g0->sel.p, c0, U.exec, sm);
    });
    if (rc) return rc;
    CU(cudaStreamSynchronize(U.exec));
    CU(cudaMemcpy(sel_host, g0->sel.p, sizeof(SelRecord) * (k + 1), cudaMemcpyDeviceToHost));
    return check_nonfinite(g0);
}

static int run_host(const b200bo_acq* spec, const double* Xc, int64_t m, double* acq_neg, double* mu,
                    double* sd, int k, SelRecord* sel_host, int64_t* n_clamped, int64_t index_base = 0) {
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (m < 0 || (m > 0 && !Xc)) return set_err(B200BO_ERR_ARG, "bad candidates");
    b200bo_gp* g0 = spec->gps[0];
    CU(cudaSetDevice(g0->device));
    {
        int np_max = 0;
        for (int g = 0; g < spec->n_gps; ++g) np_max = spec->gps[g]->np > np_max ? spec->gps[g]->np : np_max;
        const long long chunk = kChunkTilesPerSm * PBN * g0->sm_count;
        const char* e = getenv("B200BO_CHUNKED");
        const bool allow = !(e && e[0] == '0');
        if (allow && k > 0 && sel_host && !acq_neg && !mu && !sd && !n_clamped && index_base == 0 && m >= 2 * chunk &&
            !use_small_path(m, np_max, spec->n_gps, g0->sm_count, spec->path))
            return run_host_chunked(spec, Xc, m, k, sel_host);
    }
    const size_t mm = (size_t)(m > 0 ? m : 1);
    if ((rc = g0->xc.reserve(sizeof(double) * mm * g0->d))) return rc;
    if (acq_neg && (rc = g0->out_acq.reserve(sizeof(double) * mm))) return rc;
    if (mu && (rc = g0->out_mu.reserve(sizeof(double) * mm))) return rc;
    if (sd && (rc = g0->out_sd.reserve(sizeof(double) * mm))) return rc;
    if ((rc = g0->sel.reserve(sizeof(SelRecord) * (B200BO_MAX_TOPK + 1)))) return rc;
    if (m > 0) CU(cudaMemcpy(g0->xc.p, Xc, sizeof(double) * (size_t)m * g0->d, cudaMemcpyHostToDevice));
    CandSrc src;
    src.d_Xc = g0->xc.as<double>();
    if ((rc = eval_core(spec, src, m, acq_neg ? g0->out_acq.as<double>() : nullptr,
                        mu ? g0->out_mu.as<double>() : nullptr, sd ? g0->out_sd.as<double>() : nullptr, k,
                        g0->sel.p, index_base, nullptr)))
        return rc;
    CU(cudaDeviceSynchronize());
    if (m > 0) {
        if (acq_neg) CU(cudaMemcpy(acq_neg, g0->out_acq.p, sizeof(double) * m, cudaMemcpyDeviceToHost));
        if (mu) CU(cudaMemcpy(mu, g0->out_mu.p, sizeof(double) * m, cudaMemcpyDeviceToHost));
        if (sd) CU(cudaMemcpy(sd, g0->out_sd.p, sizeof(double) * m, cudaMemcpyDeviceToHost));
    }
    if (k > 0 && sel_host)
        CU(cudaMemcpy(sel_host, g0->sel.p, sizeof(SelRecord) * (k + 1), cudaMemcpyDeviceToHost));
    if (n_clamped) {
        unsigned long long c = 0;
        CU(cudaMemcpy(&c, g0->clamp.p, sizeof(c), cudaMemcpyDeviceToHost));
        *n_clamped = (int64_t)c;
    }
    return m > 0 ? check_nonfinite(g0) : B200BO_OK;
}

extern "C" int b200bo_gp_predict(b200bo_gp* gp, const double* Xc, int64_t m, double* mu, double* sd,
                                 int64_t* n_clamped) {
    if (!gp || !mu) return set_err(B200BO_ERR_ARG, "NULL argument");
    b200bo_acq spec;
    memset(&spec, 0, sizeof(spec));
    spec.kind = B200BO_ACQ_NONE;
    spec.n_gps = 1;
    spec.gps[0] = gp;
    return run_host(&spec, Xc, m, nullptr, mu, sd, 0, nullptr, n_clamped);
}

extern "C" int b200bo_gp_predict_cov(b200bo_gp* gp, const double* Xc, int64_t m, double* mu, double* cov) {
    if (!gp || !Xc || !mu || !cov) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (m <= 0 || m > 16384) return set_err(B200BO_ERR_ARG, "return_cov supports 1 <= m <= 16384 (m=%lld)", (long long)m);
    CU(cudaSetDevice(gp->device));
    StreamScope scope(nullptr);  // legacy default stream
    const int n = (int)gp->n, np = gp->np, d = gp->d, mi = (int)m, mp = round_up(m, 128);
    int rc;
    if ((rc = gp->cov_xc.reserve(sizeof(double) * (size_t)mp * d))) return rc;
    if ((rc = gp->cov_kst.reserve(sizeof(double) * (size_t)np * mp))) return rc;
    if ((rc = gp->cov_v.reserve(sizeof(double) * (size_t)np * mp))) return rc;
    if ((rc = gp->cov_c.reserve(sizeof(double) * (size_t)mp * mp))) return rc;
    if ((rc = gp->cov_out.reserve(sizeof(double) * (size_t)mi * mi))) return rc;
    if ((rc = gp->cov_mu.reserve(sizeof(double) * (size_t)mp))) return rc;
    if ((rc = gp->xc.reserve(sizeof(double) * (size_t)mi * d))) return rc;
    CU(cudaMemcpy(gp->xc.p, Xc, sizeof(double) * (size_t)mi * d, cudaMemcpyHostToDevice));
    const int* xf = gp->xform.empty() ? nullptr : gp->xf.as<int>();
    {
        const long long tot = (long long)mp * d;
        scale_xc_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(gp->xc.as<double>(), gp->ls.as<double>(), xf,
                                                                gp->cov_xc.as<double>(), mi, mp, d);
        dim3 blk(32, 8), grd((mp + 31) / 32, (np + 7) / 8);
        kcross_kernel<<<grd, blk>>>(gp->Xs.as<double>(), gp->cov_xc.as<double>(), gp->cov_kst.as<double>(), n, np,
                                    mi, mp, d, gp->family, gp->nu, gp->constv);
        cross_mean_kernel<<<(mi + 127) / 128, 128>>>(gp->cov_kst.as<double>(), gp->alphav.as<double>(),
                                                     gp->cov_mu.as<double>(), np, mi, mp, gp->y_mean, gp->y_std);
        LAUNCHED();
        LAUNCHED();
        LAUNCHED();
    }
    // V = L^-1 K*^T  (np x mp) ; VtV = V^T V (mp x mp)
    if ((rc = gemm<false, false>(np, mp, np, 1.0, gp->W.as<double>(), np, 0, gp->cov_kst.as<double>(), mp, 0, 0.0,
                                 gp->cov_v.as<double>(), mp, 0, 1, 0, 1)))
        return rc;
    if ((rc = gemm<true, false>(mp, mp, np, 1.0, gp->cov_v.as<double>(), mp, 0, gp->cov_v.as<double>(), mp, 0, 0.0,
                                gp->cov_c.as<double>(), mp, 0, 1, 0, 0)))
        return rc;
    {
        dim3 blk(32, 8), grd((mi + 31) / 32, (mi + 7) / 8);
        cov_finish_kernel<<<grd, blk>>>(gp->cov_xc.as<double>(), gp->cov_c.as<double>(), mp, gp->cov_out.as<double>(),
                                        mi, d, gp->family, gp->nu, gp->constv, gp->y_std, gp->noise);
        LAUNCHED();
    }
    CU(cudaGetLastError());
    CU(cudaMemcpy(mu, gp->cov_mu.p, sizeof(double) * (size_t)mi, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(cov, gp->cov_out.p, sizeof(double) * (size_t)mi * mi, cudaMemcpyDeviceToHost));
    return B200BO_OK;
}

extern "C" int b200bo_acq_eval(const b200bo_acq* spec, const double* Xc, int64_t m, double* acq_neg) {
    if (!acq_neg && m > 0) return set_err(B200BO_ERR_ARG, "acq_neg is NULL");
    if (spec && spec->kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    return run_host(spec, Xc, m, acq_neg, nullptr, nullptr, 0, nullptr, nullptr);
}

// Value and input gradient of the closure on the small-batch kernels (small_launch with grad: v = L^-1 k* and its sums
// exactly those of the value path).
extern "C" int b200bo_acq_value_grad(const b200bo_acq* spec, const double* Xc, int64_t m, double* val, double* grad) {
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (spec->kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    if (m < 0 || (m > 0 && (!Xc || !val || !grad))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    b200bo_gp* g0 = spec->gps[0];
    const int d = g0->d;
    CU(cudaSetDevice(g0->device));
    NvtxRange nvtx_range("b200bo:acq_value_grad");
    if ((rc = g0->xc.reserve(sizeof(double) * (size_t)m * d))) return rc;
    if ((rc = g0->out_acq.reserve(sizeof(double) * (size_t)m))) return rc;
    if ((rc = g0->out_grad.reserve(sizeof(double) * (size_t)m * d))) return rc;
    CU(cudaMemcpy(g0->xc.p, Xc, sizeof(double) * (size_t)m * d, cudaMemcpyHostToDevice));
    CandSrc src;
    src.d_Xc = g0->xc.as<double>();
    SmallParams S;
    memset(&S, 0, sizeof(S));
    int np_max = 0;
    cudaStream_t stream = nullptr;
    if ((rc = fill_params(spec, src, m, 0, stream, S.P, np_max))) return rc;
    if (spec->kind == B200BO_ACQ_MEAN && spec->n_gps > 1 && (rc = mean_merit_T(g0, stream, S.P.mean_T))) return rc;
    S.P.acq_out = g0->out_acq.as<double>();
    if ((rc = g0->clamp.reserve(2 * sizeof(unsigned long long)))) return rc;
    S.P.clamp_count = g0->clamp.as<unsigned long long>();
    CU(cudaMemsetAsync(g0->clamp.p, 0, 2 * sizeof(unsigned long long), stream));
    S.grad_out = g0->out_grad.as<double>();
    if ((rc = small_launch(spec, S, m, true, stream))) return rc;
    g0->stat_total = g0->stat_direct = m;
    g0->prune_counted = false;
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(val, g0->out_acq.p, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(grad, g0->out_grad.p, sizeof(double) * (size_t)m * d, cudaMemcpyDeviceToHost));
    return check_nonfinite(g0);
}

// q sets of (kk+1) records, kk = max(k, 1) (k = 0 still runs one round for the argmin record): set p's argmin into
// best_*[p], its top k into topk_*[p k, p k + k); every output nullable
static void unpack_records(const SelRecord* sel, int q, int k, double* best_val, int64_t* best_idx, double* topk_val,
                           int64_t* topk_idx) {
    const int kk = k > 0 ? k : 1;
    for (int p = 0; p < q; ++p) {
        const SelRecord* s = sel + (size_t)p * (kk + 1);
        if (best_val) best_val[p] = s[0].value;
        if (best_idx) best_idx[p] = s[0].index;
        for (int i = 0; i < k; ++i) {
            if (topk_val) topk_val[(size_t)p * k + i] = s[1 + i].value;
            if (topk_idx) topk_idx[(size_t)p * k + i] = s[1 + i].index;
        }
    }
}

// the q sets of records of a finished selection at d_sel, read back and unpacked
static int read_records(const void* d_sel, int q, int k, double* best_val, int64_t* best_idx, double* topk_val,
                        int64_t* topk_idx) {
    std::vector<SelRecord> rec((size_t)q * ((k > 0 ? k : 1) + 1));
    CU(cudaMemcpy(rec.data(), d_sel, sizeof(SelRecord) * rec.size(), cudaMemcpyDeviceToHost));
    unpack_records(rec.data(), q, k, best_val, best_idx, topk_val, topk_idx);
    return B200BO_OK;
}

extern "C" int b200bo_acq_argmin_topk(const b200bo_acq* spec, const double* Xc, int64_t m, int k,
                                      double* best_val, int64_t* best_idx, double* topk_val,
                                      int64_t* topk_idx, double* acq_neg) {
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    if (spec && spec->kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    SelRecord sel[B200BO_MAX_TOPK + 1];
    // k = 0 still needs the argmin record: run the selection with one round
    int rc = run_host(spec, Xc, m, acq_neg, nullptr, nullptr, k > 0 ? k : 1, sel, nullptr);
    if (rc) return rc;
    unpack_records(sel, 1, k, best_val, best_idx, topk_val, topk_idx);
    return B200BO_OK;
}

// ---------------------------------------------------------------------------------------
// throughput mode (device Philox candidates)
// ---------------------------------------------------------------------------------------
// The Philox rows of q sets of (kk+1) merged records at d_rec (kk = max(k, 1)), regenerated on stream into prow from
// the device bounds pbounds: best_x (q,d), topk_x (q,k,d) host, either nullable
// tr: the trust-region source, pbounds [3][d] with the centre last, perturbation probability tr_p.
static int philox_winner_rows(DevBuf& prow, const DevBuf& pbounds, uint64_t seed, const SelRecord* d_rec, int q, int k,
                              int d, double* best_x, double* topk_x, cudaStream_t stream, bool tr = false,
                              double tr_p = 1.0) {
    if (!best_x && !(topk_x && k > 0)) return B200BO_OK;
    const int kk = k > 0 ? k : 1, nrec = q * (kk + 1);
    int rc;
    if ((rc = prow.reserve(sizeof(double) * (size_t)nrec * d))) return rc;
    if (tr)
        philox_tr_rows_kernel<<<nrec, 64, 0, stream>>>(seed, pbounds.as<double>(), tr_p, d, d_rec, nrec,
                                                       prow.as<double>());
    else
        philox_rows_kernel<<<nrec, 64, 0, stream>>>(seed, pbounds.as<double>(), d, d_rec, nrec, prow.as<double>());
    LAUNCHED();
    CU(cudaGetLastError());
    std::vector<double> rows((size_t)nrec * d);
    CU(cudaMemcpyAsync(rows.data(), prow.p, sizeof(double) * rows.size(), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    for (int p = 0; p < q; ++p) {
        const double* rp = rows.data() + (size_t)p * (kk + 1) * d;
        if (best_x) memcpy(best_x + (size_t)p * d, rp, sizeof(double) * d);
        if (topk_x && k > 0) memcpy(topk_x + (size_t)p * k * d, rp + d, sizeof(double) * (size_t)k * d);
    }
    return B200BO_OK;
}

extern "C" int b200bo_acq_argmin_topk_philox(const b200bo_acq* spec, uint64_t seed, const double* lo,
                                             const double* hi, int64_t m, int64_t index_base, int k,
                                             double* best_val, int64_t* best_idx, double* best_x, double* topk_val,
                                             int64_t* topk_idx, double* topk_x) {
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    int rc;
    if ((rc = check_spec(spec))) return rc;
    if (spec->kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    b200bo_gp* g0 = spec->gps[0];
    CU(cudaSetDevice(g0->device));
    if ((rc = g0->sel.reserve(sizeof(SelRecord) * (B200BO_MAX_TOPK + 1)))) return rc;
    const int kk = k > 0 ? k : 1;
    if ((rc = b200bo_acq_select_philox_dev(spec, seed, lo, hi, m, index_base, kk, g0->sel.p, nullptr))) return rc;
    if ((rc = read_records(g0->sel.p, 1, k, best_val, best_idx, topk_val, topk_idx))) return rc;
    return philox_winner_rows(g0->prow, g0->pbounds, seed, g0->sel.as<SelRecord>(), 1, k, g0->d, best_x, topk_x, nullptr);
}

extern "C" int b200bo_philox_rows(int device, uint64_t seed, const double* lo, const double* hi, int d,
                                  const int64_t* idx, int64_t n_idx, double* out) {
    if (!lo || !hi || !idx || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (d <= 0 || d > B200BO_MAX_DIM || n_idx < 0) return set_err(B200BO_ERR_ARG, "bad shape");
    if (n_idx == 0) return B200BO_OK;
    CU(cudaSetDevice(device));
    std::vector<SelRecord> rec((size_t)n_idx);
    std::vector<double> pb(2 * d);  // pack_pbounds' layout, unchecked: rows of any bounds, lo > hi included
    for (int j = 0; j < d; ++j) {
        pb[j] = lo[j];
        pb[d + j] = hi[j] - lo[j];
    }
    for (int64_t i = 0; i < n_idx; ++i) {
        rec[i].value = 0.0;
        rec[i].index = idx[i];
    }
    DevBuf d_rec, d_pb, d_out;
    int rc;
    if ((rc = d_rec.reserve(sizeof(SelRecord) * n_idx))) return rc;
    if ((rc = d_pb.reserve(sizeof(double) * 2 * d))) return rc;
    if ((rc = d_out.reserve(sizeof(double) * n_idx * d))) return rc;
    CU(cudaMemcpy(d_rec.p, rec.data(), sizeof(SelRecord) * n_idx, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_pb.p, pb.data(), sizeof(double) * 2 * d, cudaMemcpyHostToDevice));
    philox_rows_kernel<<<(unsigned)n_idx, 64>>>(seed, d_pb.as<double>(), d, d_rec.as<SelRecord>(), (int)n_idx,
                                                d_out.as<double>());
    LAUNCHED();
    cudaError_t e = cudaMemcpy(out, d_out.p, sizeof(double) * n_idx * d, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return set_err(B200BO_ERR_CUDA, "philox_rows: %s", cudaGetErrorString(e));
    return B200BO_OK;
}

// trust-region source (select.cuh philox_tr_coord): lo <= center <= hi, all finite, 0 <= p <= 1 -> pb [3][d]
static int pack_tr_bounds(const double* lo, const double* hi, const double* center, double p, int d, double* pb) {
    if (!lo || !hi || !center) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!(p >= 0.0 && p <= 1.0)) return set_err(B200BO_ERR_ARG, "trust region: p=%g out of [0,1]", p);
    for (int j = 0; j < d; ++j) {
        if (!(std::isfinite(lo[j]) && std::isfinite(hi[j]) && std::isfinite(center[j])))
            return set_err(B200BO_ERR_ARG, "trust region: non-finite bound or centre in column %d", j);
        if (!(lo[j] <= center[j] && center[j] <= hi[j]))
            return set_err(B200BO_ERR_ARG, "trust region: lo <= center <= hi fails in column %d", j);
        pb[j] = lo[j];
        pb[d + j] = hi[j] - lo[j];
        pb[2 * d + j] = center[j];
    }
    return B200BO_OK;
}

extern "C" int b200bo_philox_tr_rows(int device, uint64_t seed, const double* lo, const double* hi,
                                     const double* center, double p, int d, const int64_t* idx, int64_t n_idx,
                                     double* out) {
    if (!idx || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (d <= 0 || d > B200BO_MAX_DIM || n_idx < 0) return set_err(B200BO_ERR_ARG, "bad shape");
    std::vector<double> pb(3 * d);
    int rc;
    if ((rc = pack_tr_bounds(lo, hi, center, p, d, pb.data()))) return rc;
    if (n_idx == 0) return B200BO_OK;
    CU(cudaSetDevice(device));
    std::vector<SelRecord> rec((size_t)n_idx);
    for (int64_t i = 0; i < n_idx; ++i) {
        rec[i].value = 0.0;
        rec[i].index = idx[i];
    }
    DevBuf d_rec, d_pb, d_out;
    if ((rc = d_rec.reserve(sizeof(SelRecord) * n_idx))) return rc;
    if ((rc = d_pb.reserve(sizeof(double) * 3 * d))) return rc;
    if ((rc = d_out.reserve(sizeof(double) * n_idx * d))) return rc;
    CU(cudaMemcpy(d_rec.p, rec.data(), sizeof(SelRecord) * n_idx, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_pb.p, pb.data(), sizeof(double) * 3 * d, cudaMemcpyHostToDevice));
    philox_tr_rows_kernel<<<(unsigned)n_idx, 64>>>(seed, d_pb.as<double>(), p, d, d_rec.as<SelRecord>(), (int)n_idx,
                                                   d_out.as<double>());
    LAUNCHED();
    cudaError_t e = cudaMemcpy(out, d_out.p, sizeof(double) * n_idx * d, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return set_err(B200BO_ERR_CUDA, "philox_tr_rows: %s", cudaGetErrorString(e));
    return B200BO_OK;
}

// ---------------------------------------------------------------------------------------
// posterior sample paths (Thompson sampling): paths.cuh
// ---------------------------------------------------------------------------------------
// Everything a path evaluates is a copy owned by the path: a later fit, append or LML evaluation on the GP
// handle (which overwrite its factor buffers) does not change a path drawn earlier.
struct b200bo_paths {
    int device = 0, sm_count = 0, grid_cap = 0;
    int n = 0, np = 0, d = 0, q = 0, L = 0, Lp = 0, cov = 0;
    double constv = 1.0, feat_scale = 0.0, y_mean = 0.0, y_std = 1.0;
    bool has_xf = false;
    std::vector<double> bound;  // (q,) B_p >= |path_p(x)| everywhere (b200bo_paths_bound)
    DevBuf Xs, V, omega, bias, W, ls, xf, xc, out, sel_cta, sel, pbounds, prow, bad;
    DevBuf cvals, cmerit, craw;  // constrained calls with this handle as set 0: [G][chunk][q] values, outputs
    DevBuf pidx;                 // row-mode calls: (m,) path index per row
    DevBuf grad;                 // b200bo_paths_grad_rows: (m, d) gradients
    ChunkedUpload upload;
};

// register slots per thread for the q sums: 1, 4 or 16 (q = 1, 2..4, 5..16)
static int paths_qt(int q) { return q <= 1 ? 1 : (q <= 4 ? 4 : B200BO_MAX_PATHS); }

using PathsKernel = void (*)(const PathsParams);
static PathsKernel paths_kernel(int cov, int q) {
    static const PathsKernel tab[4][3] = {
        {paths_eval_kernel<0, 1>, paths_eval_kernel<0, 4>, paths_eval_kernel<0, B200BO_MAX_PATHS>},
        {paths_eval_kernel<1, 1>, paths_eval_kernel<1, 4>, paths_eval_kernel<1, B200BO_MAX_PATHS>},
        {paths_eval_kernel<2, 1>, paths_eval_kernel<2, 4>, paths_eval_kernel<2, B200BO_MAX_PATHS>},
        {paths_eval_kernel<3, 1>, paths_eval_kernel<3, 4>, paths_eval_kernel<3, B200BO_MAX_PATHS>},
    };
    const int qt = paths_qt(q);
    return tab[cov][qt == 1 ? 0 : (qt == 4 ? 1 : 2)];
}

// row mode (b200bo_paths_eval_rows): one sum per candidate whatever q
static PathsKernel paths_rows_kernel(int cov) {
    static const PathsKernel tab[4] = {paths_eval_kernel<0, 1, true>, paths_eval_kernel<1, 1, true>,
                                       paths_eval_kernel<2, 1, true>, paths_eval_kernel<3, 1, true>};
    return tab[cov];
}

static PathsParams paths_params(const b200bo_paths* ps) {
    PathsParams P;
    memset(&P, 0, sizeof(P));
    P.Xs = ps->Xs.as<double>();
    P.V = ps->V.as<double>();
    P.omega = ps->omega.as<double>();
    P.bias = ps->bias.as<double>();
    P.W = ps->W.as<double>();
    P.ls = ps->ls.as<double>();
    P.xform = ps->has_xf ? ps->xf.as<int>() : nullptr;
    P.n = ps->n;
    P.np = ps->np;
    P.d = ps->d;
    P.q = ps->q;
    P.Lp = ps->Lp;
    P.constv = ps->constv;
    P.feat_scale = ps->feat_scale;
    P.y_mean = ps->y_mean;
    P.y_std = ps->y_std;
    P.clamp_count = ps->bad.as<unsigned long long>();
    return P;
}

static int paths_grid(const b200bo_paths* ps, int64_t m) {
    const long long ntiles = (m + PBN - 1) / PBN;
    return (int)(ntiles < ps->grid_cap ? ntiles : ps->grid_cap);
}

static int paths_launch(const b200bo_paths* ps, const PathsParams& P, int grid, cudaStream_t st) {
    if (grid <= 0) return B200BO_OK;
    void* args[] = {(void*)&P};
    const PathsKernel fn = P.path_idx ? paths_rows_kernel(ps->cov) : paths_kernel(ps->cov, P.q);
    CU(cudaLaunchKernel((const void*)fn, dim3(grid), dim3(PT_NT), args,
                        paths_smem_bytes(P.d, P.q, P.sel_cta != nullptr), st));
    LAUNCHED();
    return B200BO_OK;
}

// one k-way merge per path: (k+1) records of path p at sel[p * (k+1)]
static int paths_merge(b200bo_paths* ps, int grid, int k, cudaStream_t st) {
    NvtxRange nvtx_sel("b200bo:select");
    for (int p = 0; p < ps->q; ++p) {
        merge_sel_kernel<<<1, 256, 0, st>>>(ps->sel_cta.as<SelList>() + (size_t)p * grid, grid, k,
                                            ps->sel.as<SelRecord>() + (size_t)p * (k + 1));
        LAUNCHED();
    }
    CU(cudaGetLastError());
    return B200BO_OK;
}

static int paths_check_nonfinite(b200bo_paths* ps) {
    unsigned long long c[2] = {0, 0};
    CU(cudaMemcpy(c, ps->bad.p, sizeof(c), cudaMemcpyDeviceToHost));
    if (c[1] != 0) return set_err(B200BO_ERR_ARG, "Input X contains NaN or infinity.");
    return B200BO_OK;
}

// copies of the GP's evaluation state, the draws, and V = K^-1 (y_norm - Phi(Xs) W - eps) column by column
static int paths_setup(b200bo_gp* gp, b200bo_paths* ps, const double* omega, const double* bv, const double* w,
                       const double* eps) {
    const int n = ps->n, np = ps->np, d = ps->d, q = ps->q, L = ps->L, Lp = ps->Lp;
    const void* fn = (const void*)paths_kernel(ps->cov, q);
    // One instantiation serves every (d, q) of its class and every path alive on the device: its opt-in limit is
    // the largest size any of them can need (d = B200BO_MAX_DIM, q = its QT: 230 784 B for QT = 16), so creating
    // a smaller path never lowers the limit below what a path drawn earlier launches with.
    CU(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)paths_smem_bytes(B200BO_MAX_DIM, paths_qt(q), true)));
    // the row-mode instantiation stages all q columns of V / W: its limit covers q = B200BO_MAX_PATHS
    CU(cudaFuncSetAttribute((const void*)paths_rows_kernel(ps->cov), cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)paths_smem_bytes(B200BO_MAX_DIM, B200BO_MAX_PATHS, false)));
    CU(cudaFuncSetAttribute(cpaths_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)cpaths_smem_bytes(B200BO_MAX_PATHS)));
    const size_t smem = paths_smem_bytes(d, q, true);
    int bps = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, fn, PT_NT, smem));
    ps->grid_cap = ps->sm_count * (bps < 1 ? 1 : (bps > 2 ? 2 : bps));
    int rc;
    if ((rc = ps->Xs.reserve(sizeof(double) * (size_t)np * d))) return rc;
    if ((rc = ps->V.reserve(sizeof(double) * (size_t)np * q))) return rc;
    if ((rc = ps->omega.reserve(sizeof(double) * (size_t)Lp * d))) return rc;
    if ((rc = ps->bias.reserve(sizeof(double) * (size_t)Lp))) return rc;
    if ((rc = ps->W.reserve(sizeof(double) * (size_t)Lp * q))) return rc;
    if ((rc = ps->ls.reserve(sizeof(double) * B200BO_MAX_DIM))) return rc;
    if ((rc = ps->xf.reserve(sizeof(int) * B200BO_MAX_DIM))) return rc;
    if ((rc = ps->bad.reserve(2 * sizeof(unsigned long long)))) return rc;
    if ((rc = ps->out.reserve(sizeof(double) * (size_t)n * q))) return rc;
    CU(cudaMemcpy(ps->Xs.p, gp->Xs.p, sizeof(double) * (size_t)np * d, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(ps->ls.p, gp->ls.p, sizeof(double) * d, cudaMemcpyDeviceToDevice));
    if (ps->has_xf) CU(cudaMemcpy(ps->xf.p, gp->xf.p, sizeof(int) * d, cudaMemcpyDeviceToDevice));
    {
        std::vector<double> om((size_t)Lp * d, 0.0), bb((size_t)Lp, 0.0), ww((size_t)Lp * q, 0.0);
        memcpy(om.data(), omega, sizeof(double) * (size_t)L * d);
        memcpy(bb.data(), bv, sizeof(double) * (size_t)L);
        memcpy(ww.data(), w, sizeof(double) * (size_t)L * q);
        CU(cudaMemcpy(ps->omega.p, om.data(), sizeof(double) * om.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(ps->bias.p, bb.data(), sizeof(double) * bb.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(ps->W.p, ww.data(), sizeof(double) * ww.size(), cudaMemcpyHostToDevice));
    }
    CU(cudaMemset(ps->V.p, 0, sizeof(double) * (size_t)np * q));
    CU(cudaMemset(ps->bad.p, 0, 2 * sizeof(unsigned long long)));
    // prior part at the training rows: the candidate kernel itself on the training inputs, with V = 0 and unit
    // output scaling, so r and every later candidate share one feature code
    PathsParams P = paths_params(ps);
    P.Xc = gp->X.as<double>();
    P.m = n;
    P.out = ps->out.as<double>();
    P.y_mean = 0.0;
    P.y_std = 1.0;
    if ((rc = paths_launch(ps, P, paths_grid(ps, n), nullptr))) return rc;
    std::vector<double> prior((size_t)n * q);
    CU(cudaMemcpy(prior.data(), ps->out.p, sizeof(double) * prior.size(), cudaMemcpyDeviceToHost));
    std::vector<double> R((size_t)q * np, 0.0);
    for (int i = 0; i < n; ++i)
        for (int p = 0; p < q; ++p)
            R[(size_t)p * np + i] = gp->y_norm[i] - prior[(size_t)i * q + p] - eps[(size_t)i * q + p];
    DevBuf r, x, t1, t2;
    if ((rc = r.reserve(sizeof(double) * R.size()))) return rc;
    if ((rc = x.reserve(sizeof(double) * R.size()))) return rc;
    if ((rc = t1.reserve(sizeof(double) * np))) return rc;
    if ((rc = t2.reserve(sizeof(double) * np))) return rc;
    CU(cudaMemcpy(r.p, R.data(), sizeof(double) * R.size(), cudaMemcpyHostToDevice));
    for (int p = 0; p < q; ++p)
        if ((rc = solve_spd(gp, r.as<double>() + (size_t)p * np, x.as<double>() + (size_t)p * np, t1.as<double>(),
                            t2.as<double>())))
            return rc;
    CU(cudaMemcpy(R.data(), x.p, sizeof(double) * R.size(), cudaMemcpyDeviceToHost));
    std::vector<double> Vrow((size_t)np * q, 0.0);
    for (int i = 0; i < n; ++i)
        for (int p = 0; p < q; ++p) Vrow[(size_t)i * q + p] = R[(size_t)p * np + i];
    CU(cudaMemcpy(ps->V.p, Vrow.data(), sizeof(double) * Vrow.size(), cudaMemcpyHostToDevice));
    // |cos| <= 1 and 0 <= c k <= c: B_p = |y_mean| + y_std (feat_scale sum_l |w_lp| + c sum_i |v_ip|) bounds |path_p|
    ps->bound.assign(q, 0.0);
    for (int p = 0; p < q; ++p) {
        double sw = 0.0, sv = 0.0;
        for (int l = 0; l < L; ++l) sw += std::fabs(w[(size_t)l * q + p]);
        for (int i = 0; i < n; ++i) sv += std::fabs(Vrow[(size_t)i * q + p]);
        ps->bound[p] = std::fabs(ps->y_mean) + ps->y_std * (ps->feat_scale * sw + ps->constv * sv);
    }
    return B200BO_OK;
}

extern "C" int b200bo_paths_create(b200bo_gp* gp, int q, int L, const double* omega, const double* b,
                                   const double* w, const double* eps, b200bo_paths** out) {
    if (!gp || !omega || !b || !w || !eps || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!gp->fitted) return set_err(B200BO_ERR_STATE, "GP handle is not fitted");
    if (gp->replica) return set_err(B200BO_ERR_STATE, "a predict-only replica holds no K: draw paths from the source handle");
    if (q < 1 || q > B200BO_MAX_PATHS) return set_err(B200BO_ERR_ARG, "q=%d out of range [1,%d]", q, B200BO_MAX_PATHS);
    if (L < 1 || L > (1 << 24)) return set_err(B200BO_ERR_ARG, "L=%d out of range [1,2^24]", L);
    CU(cudaSetDevice(gp->device));
    StreamScope scope(nullptr);  // legacy default stream
    NvtxRange nvtx_range("b200bo:paths_create");
    b200bo_paths* ps = new b200bo_paths();
    ps->device = gp->device;
    ps->sm_count = gp->sm_count;
    ps->n = (int)gp->n;
    ps->np = gp->np;
    ps->d = gp->d;
    ps->q = q;
    ps->L = L;
    ps->Lp = round_up(L, PT_CHUNK);
    ps->cov = cov_code(gp->family, gp->nu);
    ps->constv = gp->constv;
    ps->feat_scale = std::sqrt(2.0 * gp->constv / (double)L);
    ps->y_mean = gp->y_mean;
    ps->y_std = gp->y_std;
    ps->has_xf = !gp->xform.empty();
    const int rc = paths_setup(gp, ps, omega, b, w, eps);
    if (rc != B200BO_OK) {
        b200bo_paths_destroy(ps);
        return rc;
    }
    *out = ps;
    return B200BO_OK;
}

extern "C" void b200bo_paths_destroy(b200bo_paths* ps) {
    if (!ps) return;
    cudaSetDevice(ps->device);  // the buffers are freed by delete, on this device
    ps->upload.release();
    delete ps;
}

// path_idx (m,) host: every entry in [0, q), then copied into dst->pidx
static int paths_upload_rows(b200bo_paths* dst, int q, const int* path_idx, int64_t m) {
    for (int64_t i = 0; i < m; ++i)
        if (path_idx[i] < 0 || path_idx[i] >= q)
            return set_err(B200BO_ERR_ARG, "path_idx[%lld]=%d out of range [0,%d)", (long long)i, path_idx[i], q);
    int rc;
    if ((rc = dst->pidx.reserve(sizeof(int) * (size_t)m))) return rc;
    CU(cudaMemcpy(dst->pidx.p, path_idx, sizeof(int) * (size_t)m, cudaMemcpyHostToDevice));
    return B200BO_OK;
}

// The evaluation kernel over m host rows into ps->out: (m, q) values, or with path_idx (row mode) row i on path
// path_idx[i] only, (m,) values.  P: the parameters it ran with.
static int paths_eval_launch(b200bo_paths* ps, const double* Xc, const int* path_idx, int64_t m, PathsParams& P) {
    int rc;
    if (path_idx && (rc = paths_upload_rows(ps, ps->q, path_idx, m))) return rc;
    if ((rc = ps->xc.reserve(sizeof(double) * (size_t)m * ps->d))) return rc;
    if ((rc = ps->out.reserve(sizeof(double) * (size_t)m * (path_idx ? 1 : ps->q)))) return rc;
    CU(cudaMemcpy(ps->xc.p, Xc, sizeof(double) * (size_t)m * ps->d, cudaMemcpyHostToDevice));
    CU(cudaMemset(ps->bad.p, 0, 2 * sizeof(unsigned long long)));
    P = paths_params(ps);
    P.Xc = ps->xc.as<double>();
    P.m = m;
    P.out = ps->out.as<double>();
    if (path_idx) P.path_idx = ps->pidx.as<int>();
    return paths_launch(ps, P, paths_grid(ps, m), nullptr);
}

extern "C" int b200bo_paths_eval(b200bo_paths* ps, const double* Xc, int64_t m, double* out) {
    if (!ps || m < 0 || (m > 0 && (!Xc || !out))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_eval");
    PathsParams P;
    int rc;
    if ((rc = paths_eval_launch(ps, Xc, nullptr, m, P))) return rc;
    CU(cudaMemcpy(out, ps->out.p, sizeof(double) * (size_t)m * ps->q, cudaMemcpyDeviceToHost));
    return paths_check_nonfinite(ps);
}

extern "C" int b200bo_paths_eval_rows(b200bo_paths* ps, const double* Xc, const int* path_idx, int64_t m,
                                      double* out) {
    if (!ps || m < 0 || (m > 0 && (!Xc || !path_idx || !out))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_eval_rows");
    PathsParams P;
    int rc;
    if ((rc = paths_eval_launch(ps, Xc, path_idx, m, P))) return rc;
    CU(cudaMemcpy(out, ps->out.p, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost));
    return paths_check_nonfinite(ps);
}

// Value and input gradient of row i on path path_idx[i]: the value from the row-mode evaluation kernel (bit-equal
// to b200bo_paths_eval_rows), the gradient from paths_grad_kernel on the same device rows.
extern "C" int b200bo_paths_grad_rows(b200bo_paths* ps, const double* Xc, const int* path_idx, int64_t m, double* val,
                                      double* grad) {
    if (!ps || m < 0 || (m > 0 && (!Xc || !path_idx || !val || !grad))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    if (m > std::numeric_limits<int>::max()) return set_err(B200BO_ERR_ARG, "m=%lld too large", (long long)m);
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_grad_rows");
    const int d = ps->d;
    PathsParams P;
    int rc;
    if ((rc = paths_eval_launch(ps, Xc, path_idx, m, P))) return rc;
    if ((rc = ps->grad.reserve(sizeof(double) * (size_t)m * d))) return rc;
    double* dg = ps->grad.as<double>();
    switch (ps->cov) {
        case 0: paths_grad_kernel<0><<<(unsigned)m, PG_NT>>>(P, dg); break;
        case 1: paths_grad_kernel<1><<<(unsigned)m, PG_NT>>>(P, dg); break;
        case 2: paths_grad_kernel<2><<<(unsigned)m, PG_NT>>>(P, dg); break;
        default: paths_grad_kernel<3><<<(unsigned)m, PG_NT>>>(P, dg); break;
    }
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpy(val, ps->out.p, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(grad, ps->grad.p, sizeof(double) * (size_t)m * d, cudaMemcpyDeviceToHost));
    return paths_check_nonfinite(ps);
}

// Host batches of more than one chunk (kChunkTilesPerSm tiles per SM) are streamed as in run_host_chunked
// (ChunkedUpload): the per-CTA lists of every path carry over between launches and are merged once.
extern "C" int b200bo_paths_argmin_topk(b200bo_paths* ps, const double* Xc, int64_t m, int k, double* best_val,
                                        int64_t* best_idx, double* topk_val, int64_t* topk_idx) {
    if (!ps) return set_err(B200BO_ERR_ARG, "paths is NULL");
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0 || !Xc) return set_err(B200BO_ERR_ARG, "m must be > 0");
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_select");
    const int kk = k > 0 ? k : 1, d = ps->d, q = ps->q;
    const long long chunk = kChunkTilesPerSm * PBN * ps->sm_count;
    ChunkedUpload& U = ps->upload;
    int rc;
    if ((rc = U.ensure())) return rc;
    const bool one = m <= chunk;
    const long long cm = one ? m : chunk;
    const int grid = one ? paths_grid(ps, m) : ps->grid_cap;  // chunked: one list per CTA slot across launches
    if ((rc = ps->xc.reserve(sizeof(double) * (size_t)(one ? 1 : 2) * cm * d))) return rc;
    if ((rc = ps->sel_cta.reserve(sizeof(SelList) * (size_t)q * grid))) return rc;
    if ((rc = ps->sel.reserve(sizeof(SelRecord) * (size_t)q * (kk + 1)))) return rc;
    double* const buf[2] = {ps->xc.as<double>(), ps->xc.as<double>() + (one ? 0 : (size_t)cm * d)};
    CU(cudaMemsetAsync(ps->bad.p, 0, 2 * sizeof(unsigned long long), U.exec));
    PathsParams P = paths_params(ps);
    P.sel_cta = ps->sel_cta.as<SelList>();
    P.sel_k = kk;
    rc = U.run(Xc, m, d, cm, buf, [&](const double* dx, long long mc, long long c0, int i, bool) {
        P.Xc = dx;
        P.m = mc;
        P.index_base = c0;
        P.sel_resume = i > 0;
        return paths_launch(ps, P, grid, U.exec);
    });
    if (rc) return rc;
    if ((rc = paths_merge(ps, grid, kk, U.exec))) return rc;
    CU(cudaStreamSynchronize(U.exec));
    if ((rc = paths_check_nonfinite(ps))) return rc;
    return read_records(ps->sel.p, q, k, best_val, best_idx, topk_val, topk_idx);
}

// Philox bounds into ps->pbounds, in the order of `stream`: the kernels that read them run on it (a host-to-device copy
// from pageable memory returns once staged, so on the legacy stream alone it would not order a non-blocking stream)
static int paths_set_pbounds(b200bo_paths* ps, const double* lo, const double* hi, cudaStream_t stream = nullptr) {
    double pb[2 * B200BO_MAX_DIM];
    int rc;
    if ((rc = pack_pbounds(lo, hi, ps->d, pb))) return rc;
    if ((rc = ps->pbounds.reserve(sizeof(double) * 2 * B200BO_MAX_DIM))) return rc;
    CU(cudaMemcpyAsync(ps->pbounds.p, pb, sizeof(double) * 2 * ps->d, cudaMemcpyHostToDevice, stream));
    return B200BO_OK;
}

extern "C" int b200bo_paths_argmin_topk_philox(b200bo_paths* ps, uint64_t seed, const double* lo, const double* hi,
                                               int64_t m, int64_t index_base, int k, double* best_val,
                                               int64_t* best_idx, double* best_x, double* topk_val,
                                               int64_t* topk_idx, double* topk_x) {
    if (!ps || !lo || !hi) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_select");
    const int kk = k > 0 ? k : 1, q = ps->q;
    const int grid = paths_grid(ps, m);
    int rc;
    if ((rc = paths_set_pbounds(ps, lo, hi))) return rc;
    if ((rc = ps->sel_cta.reserve(sizeof(SelList) * (size_t)q * grid))) return rc;
    if ((rc = ps->sel.reserve(sizeof(SelRecord) * (size_t)q * (kk + 1)))) return rc;
    PathsParams P = paths_params(ps);
    P.pbounds = ps->pbounds.as<double>();
    P.seed = seed;
    P.index_base = index_base;
    P.m = m;
    P.sel_cta = ps->sel_cta.as<SelList>();
    P.sel_k = kk;
    if ((rc = paths_launch(ps, P, grid, nullptr))) return rc;
    if ((rc = paths_merge(ps, grid, kk, nullptr))) return rc;
    if ((rc = read_records(ps->sel.p, q, k, best_val, best_idx, topk_val, topk_idx))) return rc;
    return philox_winner_rows(ps->prow, ps->pbounds, seed, ps->sel.as<SelRecord>(), q, k, ps->d, best_x, topk_x, nullptr);
}

// trust-region bounds and centre into ps->pbounds ([3][d]), in the order of `stream` (as paths_set_pbounds)
static int paths_set_tr_bounds(b200bo_paths* ps, const double* lo, const double* hi, const double* center, double p,
                               cudaStream_t stream = nullptr) {
    double pb[3 * B200BO_MAX_DIM];
    int rc;
    if ((rc = pack_tr_bounds(lo, hi, center, p, ps->d, pb))) return rc;
    if ((rc = ps->pbounds.reserve(sizeof(double) * 3 * B200BO_MAX_DIM))) return rc;
    CU(cudaMemcpyAsync(ps->pbounds.p, pb, sizeof(double) * 3 * ps->d, cudaMemcpyHostToDevice, stream));
    return B200BO_OK;
}

extern "C" int b200bo_paths_argmin_topk_philox_tr(b200bo_paths* ps, uint64_t seed, const double* lo, const double* hi,
                                                  const double* center, double p, int64_t m, int64_t index_base, int k,
                                                  double* best_val, int64_t* best_idx, double* best_x,
                                                  double* topk_val, int64_t* topk_idx, double* topk_x) {
    if (!ps) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    CU(cudaSetDevice(ps->device));
    NvtxRange nvtx_range("b200bo:paths_select");
    int rc;
    if ((rc = paths_set_tr_bounds(ps, lo, hi, center, p))) return rc;
    const int kk = k > 0 ? k : 1, q = ps->q, d = ps->d;
    const int grid = paths_grid(ps, m);
    if ((rc = ps->sel_cta.reserve(sizeof(SelList) * (size_t)q * grid))) return rc;
    if ((rc = ps->sel.reserve(sizeof(SelRecord) * (size_t)q * (kk + 1)))) return rc;
    PathsParams P = paths_params(ps);
    P.pbounds = ps->pbounds.as<double>();
    P.tr_center = ps->pbounds.as<double>() + 2 * d;
    P.tr_p = p;
    P.seed = seed;
    P.index_base = index_base;
    P.m = m;
    P.sel_cta = ps->sel_cta.as<SelList>();
    P.sel_k = kk;
    if ((rc = paths_launch(ps, P, grid, nullptr))) return rc;
    if ((rc = paths_merge(ps, grid, kk, nullptr))) return rc;
    if ((rc = read_records(ps->sel.p, q, k, best_val, best_idx, topk_val, topk_idx))) return rc;
    return philox_winner_rows(ps->prow, ps->pbounds, seed, ps->sel.as<SelRecord>(), q, k, d, best_x, topk_x, nullptr,
                              true, p);
}

// ---------------------------------------------------------------------------------------
// constrained Thompson sampling: the target's and the constraint GPs' paths ranked jointly (paths.cuh,
// cpaths_select_kernel).  Per chunk of candidates every set's paths_eval_kernel writes its (chunk x q) values into
// set 0's [G][chunk][q] scratch, then cpaths_select_kernel combines them; one merge per path at the end.
// ---------------------------------------------------------------------------------------
extern "C" int b200bo_paths_bound(const b200bo_paths* ps, double* bound) {
    if (!ps || !bound) return set_err(B200BO_ERR_ARG, "NULL argument");
    memcpy(bound, ps->bound.data(), sizeof(double) * ps->q);
    return B200BO_OK;
}

static int cpaths_check(b200bo_paths* const* sets, int G, const double* lb, const double* ub, CPathsParams& C) {
    if (!sets || !lb || !ub) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (G < 2 || G > B200BO_MAX_GPS)
        return set_err(B200BO_ERR_ARG, "G=%d out of range [2,%d] (the target and 1..%d constraints)", G,
                       B200BO_MAX_GPS, B200BO_MAX_GPS - 1);
    for (int g = 0; g < G; ++g)
        if (!sets[g]) return set_err(B200BO_ERR_ARG, "sets[%d] is NULL", g);
    const b200bo_paths* s0 = sets[0];
    for (int g = 1; g < G; ++g) {
        if (sets[g]->device != s0->device) return set_err(B200BO_ERR_ARG, "sets[%d] lives on another device", g);
        if (sets[g]->d != s0->d) return set_err(B200BO_ERR_ARG, "sets[%d]: d=%d, target d=%d", g, sets[g]->d, s0->d);
        if (sets[g]->q != s0->q) return set_err(B200BO_ERR_ARG, "sets[%d]: q=%d, target q=%d", g, sets[g]->q, s0->q);
    }
    memset(&C, 0, sizeof(C));
    for (int j = 1; j < G; ++j) {
        if (!(lb[j - 1] <= ub[j - 1])) return set_err(B200BO_ERR_ARG, "constraint %d: lb > ub", j - 1);
        C.lb[j] = lb[j - 1];
        C.ub[j] = ub[j - 1];
    }
    for (int p = 0; p < s0->q; ++p) C.T[p] = 2.0 * s0->bound[p] + 1.0;
    C.G = G;
    C.q = s0->q;
    return B200BO_OK;
}

// Xc: host rows, streamed through set 0's ChunkedUpload; nullptr: the Philox source of set 0's pbounds and `seed`,
// generated chunk by chunk.  k > 0: -g folded into the per-path lists (merged into set 0's sel); merit / raw (host,
// nullable): the (m,q) merit and the (m,G,q) values.  pidx (device, (m,), nullable): row mode - merit is (m,), row i
// on path pidx[i] only (host rows, k = 0, no raw).  tr (Philox only): the trust-region source, set 0's pbounds [3][d]
// with the centre last, perturbation probability tr_p.  Returns with the work finished and the inputs checked.
static int cpaths_run(b200bo_paths* const* sets, CPathsParams& C, const double* Xc, uint64_t seed, int64_t m,
                      int64_t index_base, int k, double* merit, double* raw, const int* pidx = nullptr,
                      bool tr = false, double tr_p = 1.0) {
    b200bo_paths* s0 = sets[0];
    const int G = C.G, q = pidx ? 1 : C.q, d = s0->d;  // q: values per row
    const long long chunk = kChunkTilesPerSm * PBN * s0->sm_count;
    const bool one = m <= chunk;
    const long long cm = one ? m : chunk;
    const int sgrid = (int)std::min<long long>((cm + CP_NT - 1) / CP_NT, 2LL * s0->sm_count);
    ChunkedUpload& U = s0->upload;
    int rc;
    if ((rc = U.ensure())) return rc;
    if ((rc = s0->cvals.reserve(sizeof(double) * (size_t)G * cm * q))) return rc;
    if (merit && (rc = s0->cmerit.reserve(sizeof(double) * (size_t)cm * q))) return rc;
    if (raw && (rc = s0->craw.reserve(sizeof(double) * (size_t)cm * G * q))) return rc;
    if (k > 0) {
        if ((rc = s0->sel_cta.reserve(sizeof(SelList) * (size_t)q * sgrid))) return rc;
        if ((rc = s0->sel.reserve(sizeof(SelRecord) * (size_t)q * (k + 1)))) return rc;
    }
    CU(cudaMemsetAsync(s0->bad.p, 0, 2 * sizeof(unsigned long long), U.exec));
    C.vals = s0->cvals.as<double>();
    C.stride = cm;
    C.sel_k = k;
    C.merit = merit ? s0->cmerit.as<double>() : nullptr;
    C.raw = raw ? s0->craw.as<double>() : nullptr;
    C.sel_cta = k > 0 ? s0->sel_cta.as<SelList>() : nullptr;
    auto work = [&](const double* dx, long long mc, long long c0, int i) -> int {
        int r;
        for (int g = 0; g < G; ++g) {
            PathsParams P = paths_params(sets[g]);
            P.Xc = dx;
            P.pbounds = s0->pbounds.as<double>();
            if (tr) {
                P.tr_center = s0->pbounds.as<double>() + 2 * d;
                P.tr_p = tr_p;
            }
            P.seed = seed;
            P.index_base = index_base + c0;
            P.m = mc;
            P.clamp_count = s0->bad.as<unsigned long long>();
            P.out = s0->cvals.as<double>() + (size_t)g * cm * q;
            P.path_idx = pidx ? pidx + c0 : nullptr;
            if ((r = paths_launch(sets[g], P, paths_grid(sets[g], mc), U.exec))) return r;
        }
        C.m = mc;
        C.index_base = index_base + c0;
        C.sel_resume = i > 0;
        if (pidx) {
            C.path_idx = pidx + c0;
            cpaths_select_kernel<true><<<sgrid, CP_NT, 0, U.exec>>>(C);
        } else {
            cpaths_select_kernel<<<sgrid, CP_NT, cpaths_smem_bytes(k > 0 ? q : 0), U.exec>>>(C);
        }
        LAUNCHED();
        CU(cudaGetLastError());
        // pageable host memory: each copy returns once it is done, in stream order behind the kernels
        if (merit)
            CU(cudaMemcpyAsync(merit + (size_t)c0 * q, C.merit, sizeof(double) * (size_t)mc * q,
                               cudaMemcpyDeviceToHost, U.exec));
        if (raw)
            CU(cudaMemcpyAsync(raw + (size_t)c0 * G * q, C.raw, sizeof(double) * (size_t)mc * G * q,
                               cudaMemcpyDeviceToHost, U.exec));
        return B200BO_OK;
    };
    if (Xc) {
        if ((rc = s0->xc.reserve(sizeof(double) * (size_t)(one ? 1 : 2) * cm * d))) return rc;
        double* const buf[2] = {s0->xc.as<double>(), s0->xc.as<double>() + (one ? 0 : (size_t)cm * d)};
        rc = U.run(Xc, m, d, cm, buf, [&](const double* dx, long long mc, long long c0, int i, bool) {
            return work(dx, mc, c0, i);
        });
    } else {
        int i = 0;
        for (long long c0 = 0; c0 < m && rc == B200BO_OK; c0 += cm, ++i) rc = work(nullptr, std::min(cm, m - c0), c0, i);
    }
    if (rc) return rc;
    if (k > 0 && (rc = paths_merge(s0, sgrid, k, U.exec))) return rc;
    CU(cudaStreamSynchronize(U.exec));
    return Xc ? paths_check_nonfinite(s0) : B200BO_OK;
}

extern "C" int b200bo_cpaths_eval(b200bo_paths* const* sets, int G, const double* lb, const double* ub,
                                  const double* Xc, int64_t m, double* merit, double* raw) {
    CPathsParams C;
    int rc;
    if ((rc = cpaths_check(sets, G, lb, ub, C))) return rc;
    if (m < 0 || (m > 0 && (!Xc || !merit))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    CU(cudaSetDevice(sets[0]->device));
    NvtxRange nvtx_range("b200bo:cpaths_eval");
    return cpaths_run(sets, C, Xc, 0, m, 0, 0, merit, raw);
}

extern "C" int b200bo_cpaths_eval_rows(b200bo_paths* const* sets, int G, const double* lb, const double* ub,
                                       const double* Xc, const int* path_idx, int64_t m, double* merit) {
    CPathsParams C;
    int rc;
    if ((rc = cpaths_check(sets, G, lb, ub, C))) return rc;
    if (m < 0 || (m > 0 && (!Xc || !path_idx || !merit))) return set_err(B200BO_ERR_ARG, "bad arguments");
    if (m == 0) return B200BO_OK;
    CU(cudaSetDevice(sets[0]->device));
    NvtxRange nvtx_range("b200bo:cpaths_eval_rows");
    if ((rc = paths_upload_rows(sets[0], C.q, path_idx, m))) return rc;
    return cpaths_run(sets, C, Xc, 0, m, 0, 0, merit, nullptr, sets[0]->pidx.as<int>());
}

extern "C" int b200bo_cpaths_argmin_topk(b200bo_paths* const* sets, int G, const double* lb, const double* ub,
                                         const double* Xc, int64_t m, int k, double* best_val, int64_t* best_idx,
                                         double* topk_val, int64_t* topk_idx) {
    CPathsParams C;
    int rc;
    if ((rc = cpaths_check(sets, G, lb, ub, C))) return rc;
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0 || !Xc) return set_err(B200BO_ERR_ARG, "m must be > 0");
    b200bo_paths* s0 = sets[0];
    CU(cudaSetDevice(s0->device));
    NvtxRange nvtx_range("b200bo:cpaths_select");
    const int kk = k > 0 ? k : 1;
    if ((rc = cpaths_run(sets, C, Xc, 0, m, 0, kk, nullptr, nullptr))) return rc;
    return read_records(s0->sel.p, C.q, k, best_val, best_idx, topk_val, topk_idx);
}

extern "C" int b200bo_cpaths_argmin_topk_philox(b200bo_paths* const* sets, int G, const double* lb,
                                                const double* ub, uint64_t seed, const double* lo, const double* hi,
                                                int64_t m, int64_t index_base, int k, double* best_val,
                                                int64_t* best_idx, double* best_x, double* topk_val,
                                                int64_t* topk_idx, double* topk_x) {
    CPathsParams C;
    int rc;
    if ((rc = cpaths_check(sets, G, lb, ub, C))) return rc;
    if (!lo || !hi) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    b200bo_paths* s0 = sets[0];
    CU(cudaSetDevice(s0->device));
    NvtxRange nvtx_range("b200bo:cpaths_select");
    const int kk = k > 0 ? k : 1;
    if ((rc = s0->upload.ensure())) return rc;
    if ((rc = paths_set_pbounds(s0, lo, hi, s0->upload.exec))) return rc;
    if ((rc = cpaths_run(sets, C, nullptr, seed, m, index_base, kk, nullptr, nullptr))) return rc;
    if ((rc = read_records(s0->sel.p, C.q, k, best_val, best_idx, topk_val, topk_idx))) return rc;
    return philox_winner_rows(s0->prow, s0->pbounds, seed, s0->sel.as<SelRecord>(), C.q, k, s0->d, best_x, topk_x,
                              nullptr);
}

extern "C" int b200bo_cpaths_argmin_topk_philox_tr(b200bo_paths* const* sets, int G, const double* lb,
                                                   const double* ub, uint64_t seed, const double* lo, const double* hi,
                                                   const double* center, double p, int64_t m, int64_t index_base,
                                                   int k, double* best_val, int64_t* best_idx, double* best_x,
                                                   double* topk_val, int64_t* topk_idx, double* topk_x) {
    CPathsParams C;
    int rc;
    if ((rc = cpaths_check(sets, G, lb, ub, C))) return rc;
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    b200bo_paths* s0 = sets[0];
    CU(cudaSetDevice(s0->device));
    NvtxRange nvtx_range("b200bo:cpaths_select");
    const int kk = k > 0 ? k : 1;
    if ((rc = s0->upload.ensure())) return rc;
    if ((rc = paths_set_tr_bounds(s0, lo, hi, center, p, s0->upload.exec))) return rc;
    if ((rc = cpaths_run(sets, C, nullptr, seed, m, index_base, kk, nullptr, nullptr, nullptr, true, p))) return rc;
    if ((rc = read_records(s0->sel.p, C.q, k, best_val, best_idx, topk_val, topk_idx))) return rc;
    return philox_winner_rows(s0->prow, s0->pbounds, seed, s0->sel.as<SelRecord>(), C.q, k, s0->d, best_x, topk_x,
                              nullptr, true, p);
}

// ---------------------------------------------------------------------------------------
// multi-GPU (one process, G devices of one box): SURVEY.md 8e
// ---------------------------------------------------------------------------------------
extern "C" int b200bo_gp_replicate(const b200bo_gp* src, int device, b200bo_gp** out) {
    if (!src || !out) return set_err(B200BO_ERR_ARG, "NULL argument");
    if (!src->fitted) return set_err(B200BO_ERR_STATE, "source GP handle is not fitted");
    b200bo_gp* dst = nullptr;
    int rc;
    if ((rc = b200bo_gp_create(&dst, device))) return rc;
    NvtxRange nvtx_range("b200bo:replicate");
    copy_model_state(src, dst);
    dst->np = src->np;
    dst->replica = true;
    const size_t np = src->np, d = src->d;
    struct Item {
        DevBuf* to;
        const DevBuf* from;
        size_t bytes;
    } items[] = {
        {&dst->Xs, &src->Xs, sizeof(double) * np * d},        {&dst->WT, &src->WT, sizeof(double) * np * np},
        {&dst->W, &src->W, sizeof(double) * np * np},          {&dst->alphav, &src->alphav, sizeof(double) * np},
        {&dst->ls, &src->ls, sizeof(double) * B200BO_MAX_DIM}, {&dst->xf, &src->xf, sizeof(int) * B200BO_MAX_DIM},
    };
    for (const Item& it : items) {
        if ((rc = it.to->reserve(it.bytes))) {
            b200bo_gp_destroy(dst);
            return rc;
        }
        cudaError_t e = cudaMemcpyPeer(it.to->p, device, it.from->p, src->device, it.bytes);
        if (e != cudaSuccess) {
            b200bo_gp_destroy(dst);
            return set_err(B200BO_ERR_CUDA, "cudaMemcpyPeer %d -> %d failed: %s", src->device, device,
                           cudaGetErrorString(e));
        }
    }
    CU(cudaSetDevice(src->device));
    CU(cudaDeviceSynchronize());
    CU(cudaSetDevice(device));
    CU(cudaDeviceSynchronize());
    dst->fitted = true;
    *out = dst;
    return B200BO_OK;
}

// NCCL is reached through dlopen so that the library has no link-time dependency on it: inside a Python
// process that already imported torch this binds to torch's bundled libnccl.so.2, otherwise to the system one.
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_multi_mu;

static int load_nccl() {
    if (g_nccl.handle) return B200BO_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return set_err(B200BO_ERR_CUDA, "cannot load libnccl.so.2: %s", dlerror());
    g_nccl.CommInitAll = (decltype(g_nccl.CommInitAll))dlsym(h, "ncclCommInitAll");
    g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
    g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
    g_nccl.GroupStart = (decltype(g_nccl.GroupStart))dlsym(h, "ncclGroupStart");
    g_nccl.GroupEnd = (decltype(g_nccl.GroupEnd))dlsym(h, "ncclGroupEnd");
    g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
    if (!g_nccl.CommInitAll || !g_nccl.CommDestroy || !g_nccl.AllGather || !g_nccl.GroupStart || !g_nccl.GroupEnd ||
        !g_nccl.GetErrorString)
        return set_err(B200BO_ERR_CUDA, "libnccl.so.2 lacks a required symbol");
    g_nccl.handle = h;
    return B200BO_OK;
}

#define NC(call)                                                                                    \
    do {                                                                                            \
        ncclResult_t r__ = (call);                                                                  \
        if (r__ != ncclSuccess)                                                                     \
            return set_err(B200BO_ERR_CUDA, "%s failed: %s", #call, g_nccl.GetErrorString(r__));    \
    } while (0)

constexpr int kMaxDev = 16;
struct MultiCtx {
    int n = 0;
    int dev[kMaxDev];
    bool has_comm = false;
    ncclComm_t comm[kMaxDev];
    cudaStream_t stream[kMaxDev] = {};
    SelRecord* sel[kMaxDev] = {};     // (MAX_TOPK+1) local records on device g
    SelRecord* gather[kMaxDev] = {};  // n * (MAX_TOPK+1) records on device g
    SelRecord* merged = nullptr;      // (MAX_TOPK+1) on device 0
};
static std::map<std::vector<int>, MultiCtx*> g_multi;

// communicators, streams and exchange buffers of c->dev[0..n)
static int multi_ctx_init(MultiCtx* c) {
    NC(g_nccl.CommInitAll(c->comm, c->n, c->dev));
    c->has_comm = true;
    for (int g = 0; g < c->n; ++g) {
        CU(cudaSetDevice(c->dev[g]));
        CU(cudaStreamCreateWithFlags(&c->stream[g], cudaStreamNonBlocking));
        CU(cudaMalloc(&c->sel[g], sizeof(SelRecord) * (B200BO_MAX_TOPK + 1)));
        CU(cudaMalloc(&c->gather[g], sizeof(SelRecord) * (B200BO_MAX_TOPK + 1) * c->n));
    }
    CU(cudaSetDevice(c->dev[0]));
    CU(cudaMalloc(&c->merged, sizeof(SelRecord) * (B200BO_MAX_TOPK + 1)));
    return B200BO_OK;
}

// frees whatever multi_ctx_init built of c before it failed, then c
static void multi_ctx_free(MultiCtx* c) {
    for (int g = 0; g < c->n; ++g) {
        cudaSetDevice(c->dev[g]);
        if (c->has_comm) g_nccl.CommDestroy(c->comm[g]);
        if (c->stream[g]) cudaStreamDestroy(c->stream[g]);
        cudaFree(c->sel[g]);
        cudaFree(c->gather[g]);
        if (g == 0) cudaFree(c->merged);
    }
    delete c;
}

// communicators + exchange buffers for a device list (created on first use, kept for the process lifetime)
static int multi_ctx(const b200bo_acq* specs, int n_dev, MultiCtx** out) {
    if (!specs || n_dev < 1 || n_dev > kMaxDev) return set_err(B200BO_ERR_ARG, "n_dev=%d out of range [1,%d]", n_dev, kMaxDev);
    std::vector<int> devs;
    int rc;
    for (int g = 0; g < n_dev; ++g) {
        if ((rc = check_spec(&specs[g]))) return rc;
        if (specs[g].n_gps != specs[0].n_gps || specs[g].kind != specs[0].kind)
            return set_err(B200BO_ERR_ARG, "specs[%d] describes a different acquisition", g);
        const int dv = specs[g].gps[0]->device;
        for (int q : devs)
            if (q == dv) return set_err(B200BO_ERR_ARG, "device %d appears twice", dv);
        devs.push_back(dv);
    }
    auto it = g_multi.find(devs);
    if (it != g_multi.end()) {
        *out = it->second;
        return B200BO_OK;
    }
    if ((rc = load_nccl())) return rc;
    MultiCtx* c = new MultiCtx();
    c->n = n_dev;
    for (int g = 0; g < n_dev; ++g) c->dev[g] = devs[g];
    if ((rc = multi_ctx_init(c))) {
        multi_ctx_free(c);
        return rc;
    }
    g_multi[devs] = c;
    *out = c;
    return B200BO_OK;
}

static void shard_range(int64_t m, int g, int n, int64_t* s, int64_t* e) {
    const int64_t base = m / n, rem = m % n;
    *s = g * base + (g < rem ? g : rem);
    *e = *s + base + (g < rem ? 1 : 0);
}

// run fn(g) on one host thread per device; the first failing rc and its message come back to the caller
template <typename F>
static int per_device(int n_dev, F fn) {
    std::vector<int> rcs(n_dev, 0);
    std::vector<std::string> msgs(n_dev);
    std::vector<std::thread> th;
    for (int g = 0; g < n_dev; ++g)
        th.emplace_back([&, g]() {
            rcs[g] = fn(g);
            if (rcs[g]) msgs[g] = g_err;
        });
    for (auto& t : th) t.join();
    for (int g = 0; g < n_dev; ++g)
        if (rcs[g]) return set_err(rcs[g], "device slot %d: %s", g, msgs[g].c_str());
    return B200BO_OK;
}

// the ONE exchange step + merge; the (k+1) merged records land in sel_host
static int multi_exchange(MultiCtx* c, int k, SelRecord* sel_host) {
    NvtxRange nvtx_range("b200bo:exchange");
    const size_t bytes = sizeof(SelRecord) * (k + 1);
    NC(g_nccl.GroupStart());
    for (int g = 0; g < c->n; ++g)
        NC(g_nccl.AllGather(c->sel[g], c->gather[g], bytes, ncclInt8, c->comm[g], c->stream[g]));
    NC(g_nccl.GroupEnd());
    CU(cudaSetDevice(c->dev[0]));
    merge_records_kernel<<<1, 32, 0, c->stream[0]>>>(c->gather[0], c->n, k, c->merged);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(sel_host, c->merged, bytes, cudaMemcpyDeviceToHost, c->stream[0]));
    for (int g = 0; g < c->n; ++g) {
        CU(cudaSetDevice(c->dev[g]));
        CU(cudaStreamSynchronize(c->stream[g]));
    }
    return B200BO_OK;
}

extern "C" int b200bo_multi_gpu_acq_argmin_topk(const b200bo_acq* specs, int n_dev, const double* Xc, int64_t m,
                                                int k, double* best_val, int64_t* best_idx, double* topk_val,
                                                int64_t* topk_idx) {
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0 || !Xc) return set_err(B200BO_ERR_ARG, "bad candidates");
    std::lock_guard<std::mutex> lock(g_multi_mu);
    MultiCtx* c = nullptr;
    int rc;
    if ((rc = multi_ctx(specs, n_dev, &c))) return rc;
    if (specs[0].kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    const int kk = k > 0 ? k : 1;
    const int d = specs[0].gps[0]->d;
    rc = per_device(n_dev, [&](int g) -> int {
        int64_t s, e;
        shard_range(m, g, n_dev, &s, &e);
        b200bo_gp* g0 = specs[g].gps[0];
        CU(cudaSetDevice(g0->device));
        int r;
        const int64_t mg = e - s;
        if ((r = g0->xc.reserve(sizeof(double) * (size_t)(mg > 0 ? mg : 1) * d))) return r;
        if (mg > 0)
            CU(cudaMemcpyAsync(g0->xc.p, Xc + (size_t)s * d, sizeof(double) * (size_t)mg * d, cudaMemcpyHostToDevice,
                               c->stream[g]));
        CandSrc src;
        src.d_Xc = g0->xc.as<double>();
        return eval_core(&specs[g], src, mg, nullptr, nullptr, nullptr, kk, c->sel[g], s, c->stream[g]);
    });
    if (rc) return rc;
    SelRecord sel[B200BO_MAX_TOPK + 1];
    if ((rc = multi_exchange(c, kk, sel))) return rc;
    for (int g = 0; g < n_dev; ++g) {
        CU(cudaSetDevice(specs[g].gps[0]->device));
        if (specs[g].gps[0]->clamp.p && (rc = check_nonfinite(specs[g].gps[0]))) return rc;
    }
    unpack_records(sel, 1, k, best_val, best_idx, topk_val, topk_idx);
    return B200BO_OK;
}

extern "C" int b200bo_multi_gpu_acq_argmin_topk_philox(const b200bo_acq* specs, int n_dev, uint64_t seed,
                                                       const double* lo, const double* hi, int64_t m,
                                                       int64_t index_base, int k, double* best_val,
                                                       int64_t* best_idx, double* best_x, double* topk_val,
                                                       int64_t* topk_idx, double* topk_x) {
    if (k < 0 || k > B200BO_MAX_TOPK) return set_err(B200BO_ERR_ARG, "k=%d out of range", k);
    if (m <= 0) return set_err(B200BO_ERR_ARG, "m must be > 0");
    std::lock_guard<std::mutex> lock(g_multi_mu);
    MultiCtx* c = nullptr;
    int rc;
    if ((rc = multi_ctx(specs, n_dev, &c))) return rc;
    if (specs[0].kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    const int kk = k > 0 ? k : 1;
    rc = per_device(n_dev, [&](int g) -> int {
        int64_t s, e;
        shard_range(m, g, n_dev, &s, &e);
        CU(cudaSetDevice(specs[g].gps[0]->device));
        if (e == s) {
            CU(cudaMemsetAsync(c->sel[g], 0xFF, sizeof(SelRecord) * (kk + 1), c->stream[g]));
            return B200BO_OK;
        }
        CandSrc src;
        src.philox = true;
        src.seed = seed;
        src.lo = lo;
        src.hi = hi;
        return eval_core(&specs[g], src, e - s, nullptr, nullptr, nullptr, kk, c->sel[g], index_base + s, c->stream[g]);
    });
    if (rc) return rc;
    SelRecord sel[B200BO_MAX_TOPK + 1];
    if ((rc = multi_exchange(c, kk, sel))) return rc;
    unpack_records(sel, 1, k, best_val, best_idx, topk_val, topk_idx);
    if (!best_x && !(topk_x && k > 0)) return B200BO_OK;
    b200bo_gp* g0 = specs[0].gps[0];
    CU(cudaSetDevice(g0->device));
    return philox_winner_rows(g0->prow, g0->pbounds, seed, c->merged, 1, k, g0->d, best_x, topk_x, c->stream[0]);
}

extern "C" int b200bo_multi_gpu_acq_eval(const b200bo_acq* specs, int n_dev, const double* Xc, int64_t m,
                                         const int64_t* offsets, double* acq_neg) {
    if (m < 0 || (m > 0 && (!Xc || !acq_neg))) return set_err(B200BO_ERR_ARG, "bad candidates");
    if (!specs || n_dev < 1 || n_dev > kMaxDev) return set_err(B200BO_ERR_ARG, "n_dev=%d out of range", n_dev);
    int rc;
    for (int g = 0; g < n_dev; ++g) {
        if ((rc = check_spec(&specs[g]))) return rc;
        if (specs[g].kind == B200BO_ACQ_NONE) return set_err(B200BO_ERR_ARG, "kind NONE has no acquisition");
    }
    if (offsets) {
        if (offsets[0] != 0 || offsets[n_dev] != m) return set_err(B200BO_ERR_ARG, "offsets must span [0, m]");
        for (int g = 0; g < n_dev; ++g)
            if (offsets[g + 1] < offsets[g]) return set_err(B200BO_ERR_ARG, "offsets must be non-decreasing");
    }
    const int d = specs[0].gps[0]->d;
    return per_device(n_dev, [&](int g) -> int {
        int64_t s, e;
        if (offsets) {
            s = offsets[g];
            e = offsets[g + 1];
        } else {
            shard_range(m, g, n_dev, &s, &e);
        }
        if (e == s) return B200BO_OK;
        return run_host(&specs[g], Xc + (size_t)s * d, e - s, acq_neg + s, nullptr, nullptr, 0, nullptr, nullptr);
    });
}
