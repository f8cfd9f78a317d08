// K3 on the tensor cores: S = U I^T with wgmma (tf32) and the 3xTF32 operand split
//     u = u_hi + u_lo,  i = i_hi + i_lo   (each part exactly representable in tf32)
//     <u, i> ~= u_hi.i_hi + u_lo.i_hi + u_hi.i_lo          (dropped term u_lo.i_lo ~ 2^-22 relative)
// accumulated in fp32 registers: fp32-level accuracy (the reference computes this GEMM in fp32 and the top-k
// order is not stable under single-pass TF32, BASELINE.md 2.3) at tensor-pipe speed.
//
// Data path
//   pack kernels   split + re-tile both operands ONCE into the canonical K-major no-swizzle layout of wgmma
//                  (8 x 16 B core matrices), so a tile slab is a contiguous byte range in global memory;
//   producer warp  cp.async.bulk (UBLKCP) global -> shared, completion on mbarriers; the 128-user tile (hi+lo)
//                  stays resident, item tiles stream as 32 KB slabs (256 items x 32 k) through a 3-4-slot ring;
//   consumers      two warpgroups, 64 users each: wgmma M64 N256 K8 into 128 fp32 registers per thread; a slot goes
//                  back to the producer once the wgmma group that read it has completed (one group kept in flight),
//                  and the finished accumulator is written straight from the registers as scores.
#include <type_traits>

#include "tc_common.cuh"

namespace mmrec {

using namespace tc;

struct ScoreTcParams {
    const float *Uhi, *Ulo, *Ihi, *Ilo;
    int KP, n_itiles, tiles_per_split, n_splits;
    int64_t B, n_items;
    float* S;
    int64_t ldS;
};

struct TcSmemLayout {
    uint32_t u_hi, u_lo, slab0, bars, total;
    int stages;
};
__host__ __device__ inline TcSmemLayout tc_smem_layout(int KP) {
    TcSmemLayout L;
    const uint32_t u_bytes = TC_M * KP * 4;
    L.stages = KP >= 128 ? 3 : 4;
    L.u_hi = 0; L.u_lo = u_bytes; L.slab0 = 2 * u_bytes;
    L.bars = L.slab0 + L.stages * TC_SLAB_BYTES;
    L.total = L.bars + 16 * 8;
    return L;
}
// barrier slots: 0 u_full | 1..4 full[s] | 5..8 empty[s] (one arrival per consumer warp)
constexpr int TC_CONSUMER_WARPS = 8;

__device__ __forceinline__ void tc_producer(const ScoreTcParams& p, const TcSmemLayout& L, uint32_t sbase, int ut, int it0, int it1) {
    const uint32_t bar = sbase + L.bars;
    const uint32_t u_bytes = TC_M * p.KP * 4;
    mbar_expect_tx(bar + 0 * 8, 2 * u_bytes);
    for (uint32_t o = 0; o < u_bytes; o += 16384) {
        bulk_g2s(sbase + L.u_hi + o, (const char*)(p.Uhi + (int64_t)ut * TC_M * p.KP) + o, 16384, bar);
        bulk_g2s(sbase + L.u_lo + o, (const char*)(p.Ulo + (int64_t)ut * TC_M * p.KP) + o, 16384, bar);
    }
    const int kchunks = p.KP / TC_KC;
    uint32_t s = 0;
    for (int it = it0; it < it1; ++it) {
        for (int c = 0; c < 2 * kchunks; ++c, ++s) {
            const uint32_t slot = s % L.stages, use = s / L.stages;
            mbar_wait(bar + (5 + slot) * 8, (use & 1) ^ 1);
            mbar_expect_tx(bar + (1 + slot) * 8, TC_SLAB_BYTES);
            const float* src = (c < kchunks ? p.Ihi : p.Ilo) + ((int64_t)it * p.KP / 4 + (c % kchunks) * (TC_KC / 4)) * (TC_N / 8) * 32;
            bulk_g2s(sbase + L.slab0 + slot * TC_SLAB_BYTES, src, TC_SLAB_BYTES, bar + (1 + slot) * 8);
        }
    }
}

// consumer warpgroup g: users [64 g, 64 g + 64) of the tile, all 256 items of each item tile
__device__ __forceinline__ void tc_consumer(const ScoreTcParams& p, const TcSmemLayout& L, uint32_t sbase, int ut, int it0, int it1, int g) {
    const uint32_t bar = sbase + L.bars;
    constexpr uint32_t LBO_A = (TC_M / 8) * 128, LBO_B = (TC_N / 8) * 128, SBO = 128;
    const int kchunks = p.KP / TC_KC;
    const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31;
    mbar_wait(bar + 0 * 8, 0);
    // descriptors are built once; per instruction only the address field moves
    const uint64_t a_hi0 = smem_desc(sbase + L.u_hi + g * 1024, LBO_A, SBO), a_lo0 = smem_desc(sbase + L.u_lo + g * 1024, LBO_A, SBO);
    const uint64_t b0 = smem_desc(sbase + L.slab0, LBO_B, SBO);
    const uint64_t ka = (2 * LBO_A) >> 4, kb = (2 * LBO_B) >> 4, slab_step = TC_SLAB_BYTES >> 4;
    const bool vec = ((p.ldS & 1) == 0) && ((((uintptr_t)p.S) & 7) == 0);
    float acc[TC_N / 2];
#pragma unroll
    for (int i = 0; i < TC_N / 2; ++i) acc[i] = 0.f;
    uint32_t slot = 0, ph = 0, prev = 0;
    uint64_t bd_slot = b0;
    for (int it = it0; it < it1; ++it) {
        uint32_t first = 0;
        uint64_t a_hi = a_hi0, a_lo = a_lo0;
        // slab c: k chunk c % kchunks of the items' hi parts (c < kchunks: u_hi.i_hi + u_lo.i_hi) or lo parts (u_hi.i_lo)
        auto slab = [&](int c, auto item_lo) {
            mbar_wait(bar + (1 + slot) * 8, ph);
            uint64_t bd = bd_slot;
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < TC_KC / 8; ++j) {
                wgmma_tf32<TC_N>(acc, a_hi, bd, first);
                first = 1;
                if (!decltype(item_lo)::value) wgmma_tf32<TC_N>(acc, a_lo, bd, 1);
                a_hi += ka; a_lo += ka; bd += kb;
            }
            wgmma_commit();
            if (c > 0) {                                          // the previous slab's group is done -> its slot goes back
                wgmma_wait<1>();
                warp_arrive(bar + (5 + prev) * 8);
            }
            prev = slot;
            bd_slot += slab_step;
            if (++slot == (uint32_t)L.stages) { slot = 0; ph ^= 1; bd_slot = b0; }
        };
        for (int c = 0; c < kchunks; ++c) slab(c, std::false_type());
        a_hi = a_hi0; a_lo = a_lo0;                               // second sweep over K: the items' lo parts
        for (int c = kchunks; c < 2 * kchunks; ++c) slab(c, std::true_type());
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        warp_arrive(bar + (5 + prev) * 8);
        const int64_t row0 = (int64_t)ut * TC_M + g * 64 + w * 16 + (lane >> 2);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = row0 + 8 * h;
            if (row >= p.B) continue;
            float* dst = p.S + row * p.ldS;
#pragma unroll
            for (int j = 0; j < TC_N / 8; ++j) {
                const int64_t col = (int64_t)it * TC_N + 8 * j + 2 * (lane & 3);
                const float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
                if (vec && col + 1 < p.n_items) *reinterpret_cast<float2*>(dst + col) = make_float2(x, y);
                else {
                    if (col < p.n_items) dst[col] = x;
                    if (col + 1 < p.n_items) dst[col + 1] = y;
                }
            }
        }
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1) score_tc_kernel(const ScoreTcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const TcSmemLayout L = tc_smem_layout(p.KP);
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar = sbase + L.bars;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 5; ++i) mbar_init(bar + i * 8, 1);
        for (int i = 5; i < 9; ++i) mbar_init(bar + i * 8, TC_CONSUMER_WARPS);
        mbar_fence_init();
    }
    __syncthreads();

    const int ut = blockIdx.x / p.n_splits, sp = blockIdx.x % p.n_splits;
    const int it0 = sp * p.tiles_per_split;
    const int it1 = min(p.n_itiles, it0 + p.tiles_per_split);
    if (it0 >= it1) return;
    if (warp == TC_CONSUMER_WARPS) {
        if (lane == 0) tc_producer(p, L, sbase, ut, it0, it1);
    } else {
        tc_consumer(p, L, sbase, ut, it0, it1, warp >> 2);
    }
}

static inline int kp_of(int d) { return d <= 32 ? 32 : (d <= 64 ? 64 : 128); }

size_t score_tc_workspace_bytes(int64_t B, int64_t n_items, int d) {
    if (d > 128 || B <= 0 || n_items <= 0) return 0;
    const int KP = kp_of(d);
    const int64_t ut = (B + TC_M - 1) / TC_M, it = (n_items + TC_N - 1) / TC_N;
    return (size_t)(2 * ut * TC_M + 2 * it * TC_N) * KP * sizeof(float) + 1024;
}

// returns 1 = done, 0 = shape not supported by this path (caller falls back to the fp32 CUDA-core kernel)
int score_tc(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items, const float* Ie, int64_t ldi,
             int d, float* S, int64_t ldS, void* ws, size_t ws_bytes, cudaStream_t stream) {
    if (d > 128 || !ws || ws_bytes < score_tc_workspace_bytes(B, n_items, d)) return 0;
    const int KP = kp_of(d);
    const int64_t n_ut = (B + TC_M - 1) / TC_M, n_it = (n_items + TC_N - 1) / TC_N;
    float* base = (float*)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
    float* Uhi = base;
    float* Ulo = Uhi + n_ut * TC_M * KP;
    float* Ihi = Ulo + n_ut * TC_M * KP;
    float* Ilo = Ihi + n_it * TC_N * KP;
    {
        const int64_t tu = n_ut * TC_M * (KP / 4), ti = n_it * TC_N * (KP / 4);
        pack_split_kernel<TC_M><<<(unsigned)((tu + 255) / 256), 256, 0, stream>>>(B, users, Ue, ldu, d, KP, Uhi, Ulo, n_ut);
        MMREC_LAUNCH_CHECK();
        pack_split_kernel<TC_N><<<(unsigned)((ti + 255) / 256), 256, 0, stream>>>(n_items, nullptr, Ie, ldi, d, KP, Ihi, Ilo, n_it);
        MMREC_LAUNCH_CHECK();
    }
    ScoreTcParams p;
    p.Uhi = Uhi; p.Ulo = Ulo; p.Ihi = Ihi; p.Ilo = Ilo; p.KP = KP; p.n_itiles = (int)n_it;
    p.B = B; p.n_items = n_items; p.S = S; p.ldS = ldS;
    // fill the machine: user tiles x item splits ~ a multiple of the SM count
    const int sms = sm_count();
    int splits = (int)(sms / n_ut);                // user tiles x item splits <= SM count: one wave, no tail
    if (splits > n_it) splits = (int)n_it;
    if (splits < 1) splits = 1;
    p.tiles_per_split = (int)((n_it + splits - 1) / splits);
    p.n_splits = (int)((n_it + p.tiles_per_split - 1) / p.tiles_per_split);
    const TcSmemLayout L = tc_smem_layout(KP);
    if (int rc = set_smem_once<score_tc_kernel>(227 * 1024)) return rc;
    score_tc_kernel<<<(unsigned)(n_ut * p.n_splits), TC_THREADS, L.total, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return 1;
}

}  // namespace mmrec

// ---- measurement aid: how many cycles does one wgmma (both operands in shared memory, K-major, no swizzle -- the form
// every tensor-core kernel of this library issues) take when nothing else runs?  One CTA per SM, one warpgroup issues
// `iters` wgmmas of M = 64, the given N and K = 32 bytes (8 tf32 / 16 bf16) into one accumulator, commits and waits.
namespace mmrec {
template <int N, int KIND>
__device__ __forceinline__ long long mma_rate_run(int iters, int distinct, uint32_t sbase) {
    constexpr uint32_t LBO_A = (64 / 8) * 128, LBO_B = (uint32_t)(N / 8) * 128;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    const long long t0 = clock64();
    tc::wgmma_fence();
    if (distinct == 0) {
        // lean issue loop: descriptors built once, only the address field moves (8 K steps, unrolled)
        const uint64_t a0 = tc::smem_desc(sbase, LBO_A, 128), b0 = tc::smem_desc(sbase + 65536, LBO_B, 128);
        const uint64_t ka = (2 * LBO_A) >> 4, kb = (2 * LBO_B) >> 4;
        for (int i = 0; i < iters; i += 8) {
            uint64_t ad = a0, bd = b0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (KIND == 0) tc::wgmma_tf32<N>(acc, ad, bd, (i | j) ? 1u : 0u);
                else tc::wgmma_bf16<N>(acc, ad, bd, (i | j) ? 1u : 0u);
                ad += ka; bd += kb;
            }
        }
    } else {
        for (int i = 0; i < iters; ++i) {
            const uint32_t off = (uint32_t)(i % distinct) * 2 * LBO_A;            // walk over `distinct` K steps of the operands
            const uint64_t ad = tc::smem_desc(sbase + off, LBO_A, 128);
            const uint64_t bd = tc::smem_desc(sbase + 65536 + (uint32_t)(i % distinct) * 2 * LBO_B, LBO_B, 128);
            if (KIND == 0) tc::wgmma_tf32<N>(acc, ad, bd, i > 0);
            else tc::wgmma_bf16<N>(acc, ad, bd, i > 0);
        }
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::wgmma_fence_regs(acc);
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) s += acc[i];
    return (t1 - t0) + (s == 1234.5f ? 1 : 0);                        // (keeps the accumulators, hence the MMAs, alive)
}

__global__ void __launch_bounds__(128, 1) mma_rate_kernel(int kind, int N, int iters, int distinct, long long* __restrict__ cycles) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = tc::smem_u32(smem);
    for (int i = threadIdx.x; i < 48 * 1024; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = 0;   // 192 KB of zeros
    tc::fence_proxy_async();
    __syncthreads();
    long long c;
    if (kind == 0) c = N == 64 ? mma_rate_run<64, 0>(iters, distinct, sbase)
                               : (N == 128 ? mma_rate_run<128, 0>(iters, distinct, sbase) : mma_rate_run<256, 0>(iters, distinct, sbase));
    else c = N == 64 ? mma_rate_run<64, 1>(iters, distinct, sbase)
                     : (N == 128 ? mma_rate_run<128, 1>(iters, distinct, sbase) : mma_rate_run<256, 1>(iters, distinct, sbase));
    if (threadIdx.x == 0) cycles[blockIdx.x] = c;
}
}  // namespace mmrec

extern "C" int mmrec_debug_mma_rate(int kind, int N, int iters, int distinct, long long* cycles_per_cta, void* stream_) {
    MMREC_CHECK_ARG((kind == 0 || kind == 1) && (N == 64 || N == 128 || N == 256) && iters >= 1 && distinct >= 0 && distinct <= 8 && cycles_per_cta,
                    "mma_rate: kind 0 (tf32) | 1 (bf16), N in {64,128,256}, 1 <= distinct <= 8");
    MMREC_CUDA(cudaFuncSetAttribute(mmrec::mma_rate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    mmrec::mma_rate_kernel<<<mmrec::sm_count(), 128, 192 * 1024, (cudaStream_t)stream_>>>(kind, N, iters, distinct, cycles_per_cta);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
