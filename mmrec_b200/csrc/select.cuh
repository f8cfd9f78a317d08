// CTA-wide top-k selection over order-preserving 32-bit keys (float_key, common.cuh), shared by topk_rows_kernel
// (topk.cu), cf_exact_kernel (score_cf.cu) and the kNN threshold / finalist kernels (knn_cf.cu), so that every one of
// them returns the same order: values descending, equal values by ascending item index -- the composite
// (key << 32 | ~index) sorted descending.
#pragma once
#include "common.cuh"

namespace mmrec {

constexpr int SELECT_THREADS = 256;     // the radix select's histogram has one bin per thread
constexpr int TOPK_MAXK = 1024;         // winners one CTA orders in shared memory

// bitonic sort of n (power of two) 64-bit composites in shared memory, DESCENDING
__device__ __forceinline__ void bitonic_desc(uint64_t* a, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
                int lo = 2 * t - (t & (stride - 1));
                int hi = lo + stride;
                bool desc = ((lo & size) == 0);
                uint64_t x = a[lo], y = a[hi];
                if ((x < y) == desc) { a[lo] = y; a[hi] = x; }
            }
        }
    }
    __syncthreads();
}

struct RadixSmem {
    unsigned hist[256];
    unsigned prefix, need;
};

struct TopkSmem {
    RadixSmem radix;
    uint64_t sel[TOPK_MAXK];
    unsigned count, base;
    unsigned warp_tot[SELECT_THREADS / 32];
};

// Radix select over the keys key_at(0 .. n-1), 8 bits per pass from the top.  On entry `need` is the rank wanted (k);
// on return the result is the top 8 * PASSES bits of the k-th largest key (the rest zero: with PASSES < 4, the lower edge of
// its bucket, so at least k keys are >= it) and `need` the number of keys in that bucket that belong to the top k.
template <int PASSES, int THREADS, class KeyAt>
__device__ __forceinline__ unsigned cta_radix_select(KeyAt key_at, int64_t n, unsigned& need, RadixSmem& sm) {
    static_assert(THREADS == SELECT_THREADS, "cta_radix_select: one histogram bin per thread, 256 threads");
    static_assert(PASSES >= 1 && PASSES <= 4, "cta_radix_select: 1 to 4 passes of 8 bits");
    const int tid = threadIdx.x;
    unsigned prefix = 0;
    for (int pass = 0; pass < PASSES; ++pass) {
        const int shift = 24 - 8 * pass;
        const unsigned hi_mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        sm.hist[tid] = 0;
        __syncthreads();
        for (int64_t i = tid; i < n; i += THREADS) {
            unsigned key = key_at(i);
            if ((key & hi_mask) == prefix) atomicAdd(&sm.hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned cum = 0;
            int dgt = 255;
            for (; dgt > 0; --dgt) {
                if (cum + sm.hist[dgt] >= need) break;
                cum += sm.hist[dgt];
            }
            sm.prefix = prefix | ((unsigned)dgt << shift);
            sm.need = need - cum;
        }
        __syncthreads();
        prefix = sm.prefix; need = sm.need;
        __syncthreads();
    }
    return prefix;
}

// The top k (k <= TOPK_MAXK) of the keys key_at(0 .. n-1), n < 2^32, in contract order: out_idx[t] = index + item_offset,
// out_val[t] = key_float(key).  Radix select of the k-th largest key; everything above it is gathered unordered, the ties
// on it are taken in index order (block-wide ordered compaction, stopping once enough are found), then a bitonic sort on
// the composite (key, ~index) puts the k winners in order.
template <int THREADS, class KeyAt>
__device__ __forceinline__ void cta_topk_from_keys(KeyAt key_at, int64_t n, int k, int64_t item_offset, int64_t* __restrict__ out_idx,
                                                   float* __restrict__ out_val, TopkSmem& sm) {
    const int tid = threadIdx.x;
    unsigned need = (unsigned)k;
    const unsigned kth = cta_radix_select<4, THREADS>(key_at, n, need, sm.radix);
    // ---- gather: strictly greater (any order), then ties in index order
    if (tid == 0) { sm.count = 0; sm.base = 0; }
    __syncthreads();
    for (int64_t i = tid; i < n; i += THREADS) {
        unsigned key = key_at(i);
        if (key > kth) {
            unsigned p = atomicAdd(&sm.count, 1u);
            sm.sel[p] = ((uint64_t)key << 32) | (uint32_t)(~(uint32_t)i);
        }
    }
    __syncthreads();
    const unsigned n_gt = sm.count;     // == k - need
    for (int64_t i0 = 0; i0 < n; i0 += THREADS) {
        if (sm.base >= need) break;
        const int64_t i = i0 + tid;
        const bool eq = i < n && key_at(i) == kth;
        const unsigned bal = __ballot_sync(0xffffffffu, eq);
        const int lane = tid & 31, wid = tid >> 5;
        if (lane == 0) sm.warp_tot[wid] = __popc(bal);
        __syncthreads();
        unsigned off = sm.base;
        for (int w = 0; w < wid; ++w) off += sm.warp_tot[w];
        const unsigned rank = off + __popc(bal & ((1u << lane) - 1u));
        if (eq && rank < need) sm.sel[n_gt + rank] = ((uint64_t)kth << 32) | (uint32_t)(~(uint32_t)i);
        __syncthreads();
        if (tid == 0) {
            unsigned tot = 0;
            for (int w = 0; w < THREADS / 32; ++w) tot += sm.warp_tot[w];
            sm.base += tot;
        }
        __syncthreads();
    }
    // ---- order the k winners
    int n2 = 1;
    while (n2 < k) n2 <<= 1;
    for (int t = k + tid; t < n2; t += THREADS) sm.sel[t] = 0;   // pads sort last (key 0 < any real key)
    __syncthreads();
    bitonic_desc(sm.sel, n2);
    for (int t = tid; t < k; t += THREADS) {
        uint64_t c = sm.sel[t];
        out_idx[t] = (int64_t)(uint32_t)(~(uint32_t)c) + item_offset;
        out_val[t] = key_float((uint32_t)(c >> 32));
    }
}

}  // namespace mmrec
