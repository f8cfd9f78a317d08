// CTA-wide top-k selection over order-preserving 32-bit keys (float_key, common.cuh), shared by topk_rows_kernel
// (topk.cu), cf_exact_kernel (score_cf.cu) and the kNN threshold / finalist kernels (knn_cf.cu), so that every one of
// them returns the same order: values descending, equal values by ascending item index -- the composite
// (key << 32 | ~index) sorted descending.  Its radix select also runs warp by warp (cf_thr_kernel, score_cf.cu).
#pragma once
#include "common.cuh"

namespace mmrec {

constexpr int SELECT_THREADS = 256;     // threads of a CTA that selects
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

// Radix select over the keys key_at(0 .. n-1), 8 bits per pass from the top, by a group of THREADS threads: one warp
// (THREADS = 32, each warp of the CTA with its own `sm`) or the whole CTA (THREADS = SELECT_THREADS = blockDim.x).  On entry
// `need` is the rank wanted (k); on return the result is the top 8 * PASSES bits of the k-th largest key (the rest zero:
// with PASSES < 4, the lower edge of its bucket, so at least k keys are >= it) and `need` the number of keys in that bucket
// that belong to the top k.  Per pass, the group counts the next digit of the keys under the prefix into `sm.hist`, then
// the first warp finds the digit: lane l owns bins 8l .. 8l + 7, a suffix sum over the lanes gives the count above them,
// and the highest lane whose bins reach `need` has the digit.
template <int PASSES, int THREADS, class KeyAt>
__device__ __forceinline__ unsigned radix_select(KeyAt key_at, int64_t n, unsigned& need, RadixSmem& sm) {
    static_assert(THREADS == 32 || THREADS == SELECT_THREADS, "radix_select: one warp or the 256-thread CTA");
    static_assert(PASSES >= 1 && PASSES <= 4, "radix_select: 1 to 4 passes of 8 bits");
    const int tid = THREADS == 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
    auto group_sync = [] { if (THREADS == 32) __syncwarp(); else __syncthreads(); };
    unsigned prefix = 0;
    for (int pass = 0; pass < PASSES; ++pass) {
        const int shift = 24 - 8 * pass;
        const unsigned hi_mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        for (int b = tid; b < 256; b += THREADS) sm.hist[b] = 0;
        group_sync();
        for (int64_t i = tid; i < n; i += THREADS) {
            unsigned key = key_at(i);
            if ((key & hi_mask) == prefix) atomicAdd(&sm.hist[(key >> shift) & 255u], 1u);
        }
        group_sync();
        if (tid < 32) {
            unsigned mine[8], tot = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { mine[j] = sm.hist[tid * 8 + j]; tot += mine[j]; }
            unsigned incl = tot;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned v = __shfl_down_sync(0xffffffffu, incl, o);
                if (tid + o < 32) incl += v;
            }
            unsigned cum = incl - tot;
            int dgt = -1;
#pragma unroll
            for (int j = 7; j >= 0; --j) {
                if (dgt < 0) {
                    if (cum + mine[j] >= need) dgt = tid * 8 + j;
                    else cum += mine[j];
                }
            }
            const unsigned found = __ballot_sync(0xffffffffu, dgt >= 0);     // (never empty: need <= keys under the prefix)
            const int win = found ? 31 - __clz(found) : 0;
            dgt = __shfl_sync(0xffffffffu, dgt, win);
            cum = __shfl_sync(0xffffffffu, cum, win);
            if (tid == 0) {
                sm.prefix = prefix | ((unsigned)(dgt < 0 ? 0 : dgt) << shift);
                sm.need = need - cum;
            }
        }
        group_sync();
        prefix = sm.prefix; need = sm.need;       // (no barrier after: the next pass writes them two group_syncs later)
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
    const unsigned kth = radix_select<4, THREADS>(key_at, n, need, sm.radix);
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
