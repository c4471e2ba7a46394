// tc_common.cuh - thin inline-PTX layer for the sm_90a kernels: mbarriers, 1-D bulk async copies
// (TMA engine, no tensor map, optionally multicast in a thread-block cluster) and wgmma issue/commit/wait.  The descriptor bit layout
// follows the PTX ISA "matrix descriptor" table of the warpgroup-level MMA instructions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200bo {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- mbarrier -----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// mbar_wait with a budget of `budget` failed polls (each try_wait may also suspend the thread for a while): on expiry
// *err is set and the wait gives up, as does every later wait that sees *err set, so a protocol error ends the
// kernel with a reported error instead of a hang
__device__ __forceinline__ void mbar_wait_budget(uint64_t* bar, uint32_t parity, unsigned long long* err,
                                                 uint32_t budget) {
    for (uint32_t n = 0; !mbar_try_wait(bar, parity); ++n) {
        if (*reinterpret_cast<volatile unsigned long long*>(err)) return;
        if (n == budget) {
            atomicExch(err, 1ull);
            return;
        }
    }
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster (this CTA included)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(rank)
        : "memory");
}

// %tid.x through a volatile read: the compiler re-reads it where it is used instead of keeping values derived from
// it live in registers (or spilled) across a long loop
__device__ __forceinline__ int tid_x() {
    int t;
    asm volatile("mov.u32 %0, %%tid.x;\n" : "=r"(t));
    return t;
}

// ---- thread-block clusters ------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// named barrier among a subset of the CTA's warps (id 1..15; nthreads multiple of 32)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory");
}

// ---- 1-D bulk async copy global -> shared, completion on an mbarrier (bytes % 16 == 0) ----------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// the same with an L2 cache policy (createpolicy), and multicast to the CTAs of `cta_mask` in the cluster: the data
// and the complete_tx land at the same shared-memory offsets in every destination CTA
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar,
                                              unsigned long long pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], "
        "%4;\n" ::"r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s_multicast_hint(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                                        uint64_t* bar, uint16_t cta_mask, unsigned long long pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint "
        "[%0], [%1], %2, [%3], %4, %5;\n" ::"r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask), "l"(pol)
        : "memory");
}
// generic-proxy writes to global memory -> visible to the async proxy (bulk copies)
__device__ __forceinline__ void fence_proxy_async_global() {
    asm volatile("fence.proxy.async.global;\n" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}

// ---- wgmma (warpgroup MMA) ------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, no swizzle ("interleaved" core matrices): a core
// matrix is 8 rows x 16 bytes stored as 128 contiguous bytes; LBO = byte distance between core
// matrices adjacent in K, SBO = between core matrices adjacent in the M/N direction.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_noswz(uint32_t smem_addr, uint32_t lbo_bytes,
                                                            uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);       // [0,14)  start address >> 4
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;  // [16,30) leading byte offset >> 4
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;  // [32,46) stride byte offset >> 4
    return d;                                           // base offset 0, layout type 0 (no swizzle)
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}

// D(64x128, fp32 registers of the warpgroup) (+)= A(64x8 tf32, smem) * B(128x8 tf32, smem)^T.
// Thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8*i + 2*(t%4) (+1):
// d[4i + 0/1] = (row, col/col+1), d[4i + 2/3] = (row + 8, col/col+1), i = 0..15.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc,
                                                     uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// fp32 -> tf32 (round to nearest, ties away), result kept in a 32-bit container
__device__ __forceinline__ float to_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}

// Byte offset of element (row r, k) inside a 128-row x 32-k fp32 operand image
// (core matrix = 8 rows x 4 k; K-direction core matrices 2048 B apart, M-direction 128 B apart).
constexpr int kTcRows = 128, kTcK = 32;
constexpr int kTcImgBytes = kTcRows * kTcK * 4;  // 16384
constexpr int kTcLBO = (kTcRows / 8) * 128;      // 2048
constexpr int kTcSBO = 128;
__host__ __device__ constexpr int tc_img_offset(int r, int k) {
    return ((k >> 2) * (kTcRows / 8) + (r >> 3)) * 128 + (r & 7) * 16 + (k & 3) * 4;
}

}  // namespace tc
}  // namespace b200bo
