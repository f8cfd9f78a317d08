// Thin inline-PTX layer for the sm_90a tensor-core kernels: mbarrier, bulk async copy (UBLKCP), wgmma fence / commit /
// wait and the wgmma shared-memory descriptor (the MMA wrappers themselves are in wgmma.cuh).  The descriptor encoding
// follows the PTX ISA's "matrix descriptor" for wgmma -- the kernels are hand-written.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace mmrec {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap within ~2 s of wall time, not hang the GPU.  The clock is only consulted after
// the fast path failed a few thousand times.  (No printf here: a call inside a run of in-flight wgmmas makes ptxas
// serialise them.)
__device__ __forceinline__ uint64_t global_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins == 4096u) t0 = global_ns();
        if (spins > 4096u && (spins & 1023u) == 0 && global_ns() - t0 > 2000000000ull) __trap();
    }
}

// ---- bulk async copy global -> shared (non-tensor TMA, SASS UBLKCP), completion on an mbarrier ---------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// ---- wgmma (warpgroup MMA) ----------------------------------------------------------------------------------------
// Every thread of the issuing warpgroup executes these.  wgmma_fence orders earlier register / shared-memory accesses
// before the next wgmma; commit closes a group of issued wgmmas; wait_group<N> returns once at most N groups are in
// flight, after which the accumulators of the completed groups may be read and their shared-memory operands reused.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the accumulators live across the wait: no read of them may be scheduled above it
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one arrival per warp on `bar` once every lane of the warp is past this point (e.g. its wgmma reads are complete)
__device__ __forceinline__ void warp_arrive(uint32_t bar) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// ---- descriptors --------------------------------------------------------------------------------------------
// K-major, no swizzle ("interleave") canonical layout, in 16-byte units ((8,n),2):((1,SBO),LBO):
// a core matrix is 8 rows x 16 B stored as 128 contiguous bytes; SBO = byte distance between core matrices that
// are neighbours along M/N (next 8 rows), LBO = between neighbours along K (next 16 B of K).
__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                           // base_offset 0, layout_type 0 (no swizzle)
}

// 3xTF32 split: hi = x rounded to tf32 (RN, ties away), lo = (x - hi) rounded to tf32; x = hi + lo to ~2^-22 |x|
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t h, l;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(x - hi));
    lo = __uint_as_float(l);
}

// Cheaper split for streamed operands (2 instructions instead of 9): hi = x with the low 13 mantissa bits cleared, lo = x - hi
// exactly (< 2^-10 |x|); the tensor core reads the top 19 bits of lo.  x = hi + lo to ~2^-20 |x|: enough for the 1e-4
// bar of the projections, not for ranking scores (those use split_tf32).
__device__ __forceinline__ void split_tf32_trunc(float x, float& hi, float& lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u);
    lo = x - hi;
}

}  // namespace tc

// ---- tile geometry shared by the tensor-core kernels ---------------------------------------------------------
constexpr int TC_M = 128;          // users per CTA tile: two consumer warpgroups of 64 rows
constexpr int TC_N = 256;          // items per accumulator (128 fp32 registers per thread)
constexpr int TC_KC = 32;          // k per slab
constexpr int TC_SLAB_BYTES = TC_N * TC_KC * 4;    // 32 KB
constexpr int TC_THREADS = 288;    // warps 0..7 consumers (MMA + epilogue), warp 8 producer

// operand packing: split into tf32 hi/lo and re-tile as [tile][kblk = KP/4][row group = R/8][8 rows][4 floats], the
// canonical K-major no-swizzle layout of wgmma, so that a K slab of a tile is one contiguous byte range
template <int R>
__device__ __forceinline__ void pack_split_one(int64_t t, int64_t n_rows, const int64_t* __restrict__ idx, const float* __restrict__ E,
                                               int64_t ld, int d, int KP, float* __restrict__ hi, float* __restrict__ lo) {
    const int kblks = KP / 4;                                          // t = (padded row, kblk)
    const int64_t row = t / kblks;
    const int kb = (int)(t % kblks);
    float x[4] = {0.f, 0.f, 0.f, 0.f};
    if (row < n_rows) {
        const float* src = E + (idx ? idx[row] : row) * ld;
#pragma unroll
        for (int e = 0; e < 4; ++e)
            if (kb * 4 + e < d) x[e] = __ldg(src + kb * 4 + e);
    }
    float4 h, l;
    tc::split_tf32(x[0], h.x, l.x); tc::split_tf32(x[1], h.y, l.y); tc::split_tf32(x[2], h.z, l.z); tc::split_tf32(x[3], h.w, l.w);
    const int64_t tile = row / R;
    const int rr = (int)(row % R);
    const int64_t off = ((tile * kblks + kb) * (R / 8) + rr / 8) * 32 + (rr % 8) * 4;
    *reinterpret_cast<float4*>(hi + off) = h;
    *reinterpret_cast<float4*>(lo + off) = l;
}

template <int R>
__global__ void pack_split_kernel(int64_t n_rows, const int64_t* __restrict__ idx, const float* __restrict__ E, int64_t ld,
                                  int d, int KP, float* __restrict__ hi, float* __restrict__ lo, int64_t n_tiles) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per (padded row, kblk)
    if (t >= n_tiles * R * (KP / 4)) return;
    pack_split_one<R>(t, n_rows, idx, E, ld, d, KP, hi, lo);
}

}  // namespace mmrec
