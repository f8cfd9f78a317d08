// K3: full-catalog scoring fused with mask + top-k as a CERTIFIED FILTER on the tensor cores.
//
// The score matrix (115 MB per 4096 users at 7k items, 16 GB at 1M) is never written and no threshold depends on
// timing.  The tensor cores (wgmma f16, ONE pass over operands rounded to fp16 after a power-of-two scaling:
// the same 11-bit significand as tf32 at twice the MMA rate and half the operand bytes) compute APPROXIMATE scores
// s~ with a proven bound |s~ - s| <= eps * |u| * max|i| (+ a subnormal term that only matters for degenerate
// tables, see cf_thr_kernel); they are only used to decide which (user, item) pairs can
// be in the top-k.  Every pair that can is then scored again in full fp32 (fmaf chain, the arithmetic of the exact
// kernel below), and the final order is taken on those fp32 values -- so the result is the fp32 top-k, tie -> lower
// item index, exactly the contract of topk.cu.
//
//   cf_pack_kernel      operands -> fp16 (round to nearest) in the canonical K-major no-swizzle layout of wgmma, tiles of
//                       128 rows, scaled by a power of two (per user row; one for the whole catalogue) so that the
//                       largest element lands in [2^14, 2^15): no overflow, and fp16 subnormals only for elements
//                       2^-28 below the largest.  Scores, norms and thresholds of a row all live in that scaled domain
//                       (the exact re-scoring reads the original tables).  Row norms (users) / maximum row norm
//                       (catalogue).  The catalogue side is packed once per embedding table (mmrec_catalog_pack_f32), its
//                       scale from the table's largest magnitude (absmax_norm_kernel, knn_cf.cu).
//   cf_pass_kernel<1>   s~ for every (user, item); epilogue = maximum of every group of w = 16 gw consecutive items
//                       (accumulator registers -> max tree -> quad shuffles: group_max_store), written as gmax[row][group].
//                       No atomics.
//   cf_thr_kernel       per row: t = the need-th largest group maximum, need = k + (masked items of the row).  At
//                       least `need` distinct items have s~ >= t, so >= k unmasked ones have s >= t - eps'; hence every
//                       member of the true top-k has s~ >= thr = t - 2 eps' (set_threshold).
//   cf_pass_kernel<2>   s~ again (same instructions, same bits); epilogue = one bit per score, s~ >= thr, 128 bits per
//                       (row, item tile) written as one 16-byte store.  ~ (need + a few) bits per row are set.
//   cf_final_kernel     per row (one warp): the set bits -> drop masked items -> exact fp32 score from the ORIGINAL
//                       tables -> rank on (value desc, item asc) -> top-k.
//   cf_exact_kernel     rows the filter cannot serve (need > number of groups, > CF_CAP candidates, non-finite scores):
//                       all items in fp32 on CUDA cores + radix select; exits at once when no row is flagged.
// Work distribution of the passes: a unit = (pair of 128-user tiles, 128-item tile); the units are dealt to the CTAs
// (one per SM) in contiguous runs, so every SM gets the same number of units whatever the batch size (no wave
// quantisation), a 256-user operand stays resident while its run of item tiles streams through a bulk-copy ring, and
// every item slab read from L2 feeds two warpgroups' MMAs (one 128-user tile per CTA would need twice the L2 bandwidth
// per flop).  Each pass kernel: warpgroup h = 0 / 1 owns user half h of the pair (wgmma M64 N128 K16 twice per K step:
// 2 x 64 fp32 accumulator registers per thread) and runs the epilogue on its registers; warp 8 is the bulk-copy producer.
#include <climits>
#include <cstdio>
#include <cstdlib>

#include "batch_mask.cuh"
#include "select.cuh"
#include "tc_common.cuh"

namespace mmrec {

using namespace tc;

constexpr int CF_TILE = 128;                    // rows of one operand tile (users: one warpgroup; items: the MMA's N)
// An item slab is the whole K of a 128-item tile (8 / 16 / 32 KB at KP = 32 / 64 / 128): one barrier round trip per unit.
constexpr int CF_CONSUMER_WARPS = 8;            // two warpgroups, one per user half of the pair
constexpr int CF_THREADS = 32 * CF_CONSUMER_WARPS + 32;
constexpr int CF_MAX_STAGES = 10;
constexpr int CF_CAP = 512;                     // candidates one warp ranks per row
constexpr int CF_EX_SLOTS = 128;                // CTAs (and key buffers) of the exact kernel
constexpr float CF_EPS = 1.125f / 1024.f;       // |s~ - s| <= CF_EPS |u| |i|: two RN roundings to 11 significand bits (2^-11 each) + slack 2^-13 for the accumulation (<= 8 steps of 2^-20, knn_cf.cu (2)) and the fp32 chain
constexpr float CF_EPS_SUB = 1.0f / 16777216.f; // fp16 subnormal spacing 2^-24 (scaled domain): |dx| <= 2^-11 |x| + 2^-25 per element

struct CfSmem {
    uint32_t a, slab0, slab, bars, total;
    int stages;
};
__host__ __device__ inline CfSmem cf_smem(int KP) {
    CfSmem L;
    L.a = 0;
    L.slab0 = 2 * CF_TILE * KP * 2;             // the 256-user operand: two tiles of 128 rows, fp16
    const uint32_t slab = CF_TILE * KP * 2;
    L.slab = slab;
    L.stages = (int)((226u * 1024u - L.slab0 - 300u) / slab);        // as many slabs in flight as shared memory holds
    if (L.stages > CF_MAX_STAGES) L.stages = CF_MAX_STAGES;
    L.bars = L.slab0 + L.stages * slab;
    L.total = L.bars + 32 * 8;
    return L;
}
// barrier slots: AFULL (tx) | AFREE (one arrival per consumer warp) | FULL[s] (tx) | EMPTY[s] (one arrival per consumer warp)
enum { CB_AFULL = 0, CB_AFREE = 1, CB_FULL = 2, CB_EMPTY = 2 + CF_MAX_STAGES, CB_END = 2 + 2 * CF_MAX_STAGES };

struct CfParams {
    const char* Upk;                            // fp16 [pairs][2][KP/8][16][8][8]
    const char* Ipk;                            // fp16 [item tiles][KP/8][16][8][8]
    int KP, n_it;
    int64_t B, n_items, n_units;
    float* gmax; int G, gw;                     // pass 1: [B][G], G = n_it * (8 / gw)
    const float* thr; uint4* bitmap;            // pass 2: [B], [B][n_it]
    int dbg;                                    // tuning aid (env MMREC_CF_DEBUG): 2 = no MMAs issued, 16 = no item traffic
};

// ---- producer: the 256-user operand of the current pair, then its run of item slabs ----------------------------
__device__ __forceinline__ void cf_producer(const CfParams& p, const CfSmem& L, uint32_t sbase, int64_t u0, int64_t u1) {
    const uint32_t bar = sbase + L.bars;
    const uint32_t a_bytes = 2 * CF_TILE * p.KP * 2;
    const uint32_t piece = L.slab < 16384u ? L.slab : 16384u;        // bulk copies of at most 16 KB
    // (pair, it) and the ring position advance by counting: a 64-bit division per unit is several hundred cycles of a
    // single thread's dependent instructions, and this loop is what the slab ring's refill rate hangs on
    int64_t pair = u0 / p.n_it;
    int it = (int)(u0 - pair * p.n_it);
    bool new_pair = true;
    uint32_t a_cnt = 0, slot = 0, ph = 1;                            // ph: parity to wait for on the slot's "empty" barrier
    for (int64_t u = u0; u < u1; ++u) {
        if (new_pair) {
            if (a_cnt > 0) mbar_wait(bar + CB_AFREE * 8, (a_cnt - 1) & 1);   // every MMA that reads the old operand is done
            mbar_expect_tx(bar + CB_AFULL * 8, a_bytes);
            const char* src = p.Upk + pair * (int64_t)a_bytes;
            for (uint32_t o = 0; o < a_bytes; o += 16384) bulk_g2s(sbase + L.a + o, src + o, 16384, bar + CB_AFULL * 8);
            ++a_cnt;
            new_pair = false;
        }
        const char* src = p.Ipk + (int64_t)it * L.slab;
        const uint32_t fb = bar + (CB_FULL + slot) * 8;
        mbar_wait(bar + (CB_EMPTY + slot) * 8, ph);
        if (p.dbg & 16) {                                             // (tuning aid: no item traffic)
            mbar_arrive(fb);
        } else {
            mbar_expect_tx(fb, L.slab);
            const uint32_t dst = sbase + L.slab0 + slot * L.slab;
            for (uint32_t o = 0; o < L.slab; o += piece) bulk_g2s(dst + o, src + o, piece, fb);
        }
        if (++slot == (uint32_t)L.stages) { slot = 0; ph ^= 1; }
        if (++it == p.n_it) { it = 0; ++pair; new_pair = true; }
    }
}

// ---- consumer warpgroup h: MMAs of user half h of the pair for each unit, then the epilogue on the registers ---------
template <int PASS, int GPT>
__device__ __forceinline__ void cf_consumer(const CfParams& p, const CfSmem& L, uint32_t sbase, int64_t u0, int64_t u1, int h) {
    const uint32_t bar = sbase + L.bars;
    constexpr uint32_t LBO = (CF_TILE / 8) * 128, SBO = 128;         // both operands: tiles of 128 rows
    const int ksteps = p.KP / 16;
    const uint32_t half_bytes = CF_TILE * p.KP * 2;
    const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31, q = lane & 3;
    // descriptors are built once and only their address field (low word, 16-byte units) moves; rows 64..127 of the half
    // start 8 core-matrix rows (1024 B) further
    const uint64_t a_desc0 = smem_desc(sbase + L.a + h * half_bytes, LBO, SBO), a_desc1 = smem_desc(sbase + L.a + h * half_bytes + 1024, LBO, SBO);
    const uint64_t b_desc0 = smem_desc(sbase + L.slab0, LBO, SBO);
    const uint64_t kstep = (2 * LBO) >> 4;                           // one K step of 16 = two 16-byte k blocks
    const uint64_t slab_step = L.slab >> 4;
    float acc0[64], acc1[64];                                         // rows 16 w + lane / 4 (+ 8) and 64 + the same
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }   // (read by no MMA: the first K step overwrites)
    int64_t pair = u0 / p.n_it;
    int it = (int)(u0 - pair * p.n_it);
    bool new_pair = true, live = false;
    uint32_t a_cnt = 0, slot = 0, ph = 0;
    uint64_t bd_slot = b_desc0;
    int64_t row0 = 0;                                                 // row of accumulator row r = 2 m + e2: row0 + 64 m + 8 e2
    float thr[4];
    for (int64_t u = u0; u < u1; ++u) {
        if (new_pair) {
            mbar_wait(bar + CB_AFULL * 8, a_cnt & 1);
            ++a_cnt;
            const int64_t base = pair * (2 * CF_TILE) + h * CF_TILE;
            live = base < p.B;                                        // (a whole half beyond the batch: no MMAs, no output)
            row0 = base + 16 * w + (lane >> 2);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int64_t rr = row0 + 64 * (r >> 1) + 8 * (r & 1);
                if (PASS == 2) thr[r] = rr < p.B ? __ldg(p.thr + rr) : INFINITY;
            }
            new_pair = false;
        }
        mbar_wait(bar + (CB_FULL + slot) * 8, ph);
        if (live && !(p.dbg & 2)) {
            uint64_t ad0 = a_desc0, ad1 = a_desc1, bd = bd_slot;
            wgmma_fence();
#pragma unroll 4
            for (int j = 0; j < ksteps; ++j) {
                wgmma_f16<CF_TILE>(acc0, ad0, bd, j ? 1u : 0u);
                wgmma_f16<CF_TILE>(acc1, ad1, bd, j ? 1u : 0u);
                ad0 += kstep; ad1 += kstep; bd += kstep;
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc0);
            wgmma_fence_regs(acc1);
        }
        warp_arrive(bar + (CB_EMPTY + slot) * 8);                     // slab consumed -> slot back to the producer
        bd_slot += slab_step;
        if (++slot == (uint32_t)L.stages) { slot = 0; ph ^= 1; bd_slot = b_desc0; }
        const int cur_it = it;
        if (++it == p.n_it) { it = 0; ++pair; new_pair = true; }
        if (new_pair || u + 1 == u1) warp_arrive(bar + CB_AFREE * 8);  // this warp is done with the pair's user operand
        if (!live) continue;
        // ---- epilogue, one accumulator row at a time (r = 2 m + e2: set m, row half e2); columns >= n_valid (last item
        // tile only) read as -inf: never a maximum, never a hit
        const int n_valid = (int)(p.n_items - (int64_t)cur_it * CF_TILE);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float* acc = r < 2 ? acc0 : acc1;
            const int e2 = r & 1;
            const int64_t row = row0 + 64 * (r >> 1) + 8 * e2;
            auto val = [&](int j, int e) {                            // column 8 j + 2 q + e of the row
                const float v = acc[4 * j + 2 * e2 + e];
                return 8 * j + 2 * q + e < n_valid ? v : -INFINITY;
            };
            if (PASS == 1) {
                group_max_store<GPT>(r < 2 ? acc0 : acc1, e2, q, n_valid, row, p.B, [&] { return p.gmax + row * p.G + (int64_t)cur_it * GPT; });
            } else {
                // bit (31 - c) of word b: column 32 b + c passes, s~ >= thr (the sign of the exact difference)
                uint32_t wd[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        if (!(__float_as_uint(val(j, e) - thr[r]) >> 31)) wd[j >> 2] |= 1u << (31 - (8 * (j & 3) + 2 * q + e));
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    wd[b] |= __shfl_xor_sync(0xffffffffu, wd[b], 1);
                    wd[b] |= __shfl_xor_sync(0xffffffffu, wd[b], 2);
                }
                if (q == r && row < p.B) p.bitmap[row * p.n_it + cur_it] = make_uint4(wd[0], wd[1], wd[2], wd[3]);
            }
        }
    }
}

template <int PASS, int GPT>
__global__ void __launch_bounds__(CF_THREADS, 1) cf_pass_kernel(const CfParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const CfSmem L = cf_smem(p.KP);
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar = sbase + L.bars;
    if (threadIdx.x == 0) {
        mbar_init(bar + CB_AFULL * 8, 1);
        mbar_init(bar + CB_AFREE * 8, CF_CONSUMER_WARPS);
        for (int s = 0; s < CF_MAX_STAGES; ++s) {
            mbar_init(bar + (CB_FULL + s) * 8, 1);
            mbar_init(bar + (CB_EMPTY + s) * 8, CF_CONSUMER_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    // contiguous run of units for this CTA
    const int64_t u0 = (int64_t)blockIdx.x * p.n_units / gridDim.x;
    const int64_t u1 = (int64_t)(blockIdx.x + 1) * p.n_units / gridDim.x;
    if (warp == CF_CONSUMER_WARPS) {
        if (lane == 0) cf_producer(p, L, sbase, u0, u1);
    } else {
        cf_consumer<PASS, GPT>(p, L, sbase, u0, u1, warp >> 2);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// operand packing
// ------------------------------------------------------------------------------------------------------------------
// One thread per (padded row, k block of 8): scale, round to fp16, store 16 bytes into the tile layout; the KP/8 threads
// of a row are consecutive lanes and reduce the row's squared norm (and, for user rows, its largest magnitude) with
// shuffles.  `scale_src` = the catalogue-wide largest magnitude (items), or NULL: per-row scale (users).
__device__ __forceinline__ void cf_pack_one(int64_t t, int64_t n_rows, const int64_t* __restrict__ idx, const float* __restrict__ E, int64_t ld,
                                            int d, int KP, const uint32_t* __restrict__ scale_src, uint4* __restrict__ out,
                                            float* __restrict__ row_norm, uint32_t* __restrict__ max_norm) {
    const int kblks = KP / 8;
    const int64_t row = t / kblks;
    const int kb = (int)(t % kblks);
    float x[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = 0.f;
    if (row < n_rows) {
        const float* src = E + (idx ? idx[row] : row) * ld;
#pragma unroll
        for (int e = 0; e < 8; ++e)
            if (kb * 8 + e < d) x[e] = __ldg(src + kb * 8 + e);
    }
    uint32_t am = 0u;                                                 // largest |x| as a bit pattern (orders like the value; NaN above inf)
    if (!scale_src) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const uint32_t b = __float_as_uint(x[e]) & 0x7fffffffu; am = b > am ? b : am; }
        for (int o = kblks / 2; o > 0; o >>= 1) {
            const uint32_t a2 = __shfl_xor_sync(0xffffffffu, am, o);
            am = a2 > am ? a2 : am;
        }
    }
    const float sc = fp16_scale_for(scale_src ? __ldg(scale_src) : am);
    // the norm is taken of the scaled row: squares of unscaled elements below ~1e-19 underflow to 0 (and above ~1e19
    // overflow), which would shrink the margin of cf_thr_kernel to its subnormal term while the operands are full size
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) ss = fmaf(x[e] * sc, x[e] * sc, ss);              // (exact: a power of two, no overflow)
    for (int o = kblks / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    store_fp16x8(out, row / CF_TILE, kblks, kb, (int)(row % CF_TILE), x, sc);
    if (kb == 0 && row < n_rows) {
        const float nrm = sqrtf(ss) * (1.0f + 1e-6f);                 // norm of the scaled row (rounded up: the bound must hold)
        if (row_norm) row_norm[row] = nrm;
        if (max_norm) atomicMax(max_norm, __float_as_uint(nrm));      // non-negative floats order like their bit patterns
    }
}

__global__ void __launch_bounds__(256) cf_pack_items_kernel(int64_t n_items, const float* __restrict__ Ie, int64_t ldi, int d, int KP,
                                                            uint4* __restrict__ Ipk, uint32_t* __restrict__ header, int64_t n_threads) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_threads) return;                                       // (n_threads is a multiple of 32: whole warps leave together)
    if (t == 0) { header[1] = (uint32_t)n_items; header[2] = (uint32_t)d; header[3] = (uint32_t)KP; }
    cf_pack_one(t, n_items, nullptr, Ie, ldi, d, KP, header + 4, Ipk, nullptr, header);
}

// One launch per row block for everything the passes need prepared: the sorted pass of the batch mask CSR (first call
// only, batch_mask.cuh), the user operand + row norms, and the zeroing of the flags / slot counter.
__global__ void __launch_bounds__(256) cf_prep_kernel(int64_t mask_blocks, const BatchMask mask, int64_t nb, const int64_t* __restrict__ users,
                                                      const float* __restrict__ Ue, int64_t ldu, int d, int KP, uint4* __restrict__ Upk,
                                                      float* __restrict__ unorm, int64_t pack_threads, uint32_t* __restrict__ zero, int64_t zero_words) {
    if ((int64_t)blockIdx.x < mask_blocks) {
        mask_sorted_block(blockIdx.x, mask);
        return;
    }
    int64_t t = (blockIdx.x - mask_blocks) * (int64_t)blockDim.x + threadIdx.x;
    if (t < pack_threads) { cf_pack_one(t, nb, users, Ue, ldu, d, KP, nullptr, Upk, unorm, nullptr); return; }   // (multiple of 256: whole blocks)
    t -= pack_threads;
    if (t < zero_words) zero[t] = 0;
}

// ------------------------------------------------------------------------------------------------------------------
// threshold: the need-th largest group maximum of the row, minus the certified margin.  One warp per row: up to 1024
// groups the register search below, beyond that the warp's radix select (radix_select, select.cuh).
// ------------------------------------------------------------------------------------------------------------------
// The threshold does not have to be the exact need-th largest group maximum -- any value with at least `need` maxima at
// or above it is certified.  So the search runs on the top CF_THR_BITS bits of the order-preserving key only (bit by
// bit, counts by REDUX: no atomics, the values stay in registers) and takes the lower edge of that bucket: 16 bits =
// the value to 2^-7 relative, a handful of extra candidates per row for half the dependent steps.
constexpr int CF_THR_BITS = 16;
template <int NV>
__device__ __forceinline__ uint32_t cf_warp_kth_coarse(const float* __restrict__ g, int G, int need, int lane) {
    uint32_t key[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int t = j * 32 + lane;
        key[j] = t < G ? float_key(__ldg(g + t)) : 0u;
    }
    // bits above the first one in which the row's largest and smallest key differ are common to all keys: nothing to search
    uint32_t kmax = 0u, kmin = 0xffffffffu;
#pragma unroll
    for (int j = 0; j < NV; ++j) {                                   // (-inf = a group of padding columns: not part of the range)
        kmax = max(kmax, key[j]);
        if (j * 32 + lane < G && key[j] > 0x007fffffu) kmin = min(kmin, key[j]);
    }
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    kmin = __reduce_min_sync(0xffffffffu, kmin);
    const int top = 31 - __clz((kmax ^ kmin) | (1u << (32 - CF_THR_BITS)));    // >= the lowest searched bit
    uint32_t prefix = top >= 31 ? 0u : (kmax & ~((2u << top) - 1u));
#pragma unroll 1
    for (int b = top; b >= 32 - CF_THR_BITS; --b) {
        const uint32_t cand = prefix | (1u << b);
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < NV; ++j) cnt += key[j] >= cand;
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (cnt >= need) prefix = cand;
    }
    return prefix;                                                   // <= the need-th largest key, same top bits
}

__global__ void __launch_bounds__(256) cf_thr_kernel(int64_t nb, int G, int G_valid, int k, int d, const float* __restrict__ gmax, const float* __restrict__ unorm,
                                                     const uint32_t* __restrict__ max_norm, const int32_t* __restrict__ mask_ptr,
                                                     float* __restrict__ thr, int32_t* __restrict__ flags) {
    __shared__ RadixSmem radix_all[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= nb) return;
    const int need = k + (mask_ptr ? mask_ptr[row + 1] - mask_ptr[row] : 0);
    if (need > G_valid) {                                            // more finalists wanted than there are (non-padding) groups: exact kernel
        if (lane == 0) { thr[row] = INFINITY; flags[row] = 1; }
        return;
    }
    const float* g = gmax + row * G;
    uint32_t kth;
    if (G <= 16 * 32) kth = cf_warp_kth_coarse<16>(g, G, need, lane);
    else if (G <= 32 * 32) kth = cf_warp_kth_coarse<32>(g, G, need, lane);
    else {
        unsigned need_u = (unsigned)need;
        kth = radix_select<4, 32>([=](int64_t t) { return float_key(__ldg(g + t)); }, G, need_u, radix_all[warp]);
    }
    if (lane == 0) {
        // scaled domain.  Per element |dx| <= 2^-11 |x| + 2^-25 (fp16 subnormals), so
        //   |s~ - s| <= 2^-10 |u| |i| (1 + 2^-12) + 2^-25 sqrt(d) (|u| + |i|) + (2^-25)^2 d + accumulation  <=  eps' below;
        // with the largest elements scaled into [2^14, 2^15) the second term is ~2^-38 of the first
        const float un = unorm[row], mn = __uint_as_float(*max_norm);
        set_threshold(key_float(kth), 2.0f * (CF_EPS * un * mn + CF_EPS_SUB * sqrtf((float)d) * (un + mn + 1.0f)), thr + row, flags + row);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// exact fp32 score of one (user, item) pair.  THE arithmetic of this file's results, chosen so that a group of lanes can
// compute it from one coalesced read of the item row:
//     L = 8 / 16 / 32 blocks of four elements (d <= 32 / 64 / 128; elements beyond d count as 0),
//     p_l = fmaf(u[4l+3], v[4l+3], fmaf(u[4l+2], v[4l+2], fmaf(u[4l+1], v[4l+1], fmaf(u[4l], v[4l], 0)))),
//     then the butterfly tree  p_a += p_(a + w)  for a < w,  w = L/2, L/4, ..., 1;  the score is p_0.
// cf_dot_thread is one thread doing all of it (exact kernel: every item of a flagged row); cf_dot_round is a warp doing
// 32 candidates, L lanes per item row, the tree run as a transposed butterfly so that each lane ends up with the
// complete score of one candidate.  Float addition commutes, so both give the same bits.
// ------------------------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int cf_lpr(int d) { return d <= 32 ? 8 : (d <= 64 ? 16 : 32); }

__device__ __forceinline__ float4 cf_load4(const float* __restrict__ row, int l, int d, bool vec_ok) {
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (vec_ok) {                                                    // d % 4 == 0, rows 16-byte aligned
        if (4 * l < d) x = ldg4(row + 4 * l);
    } else {
        if (4 * l < d) x.x = __ldg(row + 4 * l);
        if (4 * l + 1 < d) x.y = __ldg(row + 4 * l + 1);
        if (4 * l + 2 < d) x.z = __ldg(row + 4 * l + 2);
        if (4 * l + 3 < d) x.w = __ldg(row + 4 * l + 3);
    }
    return x;
}
__device__ __forceinline__ float cf_chain4(const float4 u, const float4 x) {
    return fmaf(u.w, x.w, fmaf(u.z, x.z, fmaf(u.y, x.y, fmaf(u.x, x.x, 0.f))));
}

template <int LPR>
__device__ __forceinline__ float cf_dot_thread_t(const float* __restrict__ u_sm /* zero-padded to 128 */, const float* __restrict__ v, int d, bool vec_ok) {
    float p[LPR];
#pragma unroll
    for (int l0 = 0; l0 < LPR; l0 += 8) {                            // 8 x 16 bytes of the item row in flight
        float4 x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = cf_load4(v, l0 + i, d, vec_ok);
#pragma unroll
        for (int i = 0; i < 8; ++i) p[l0 + i] = cf_chain4(*reinterpret_cast<const float4*>(u_sm + 4 * (l0 + i)), x[i]);
    }
#pragma unroll
    for (int w = LPR / 2; w >= 1; w >>= 1)
#pragma unroll
        for (int a = 0; a < w; ++a) p[a] = p[a] + p[a + w];
    return p[0];
}
__device__ __forceinline__ float cf_dot_thread(const float* __restrict__ u_sm, const float* __restrict__ v, int d, bool vec_ok) {
    return d <= 32 ? cf_dot_thread_t<8>(u_sm, v, d, vec_ok) : (d <= 64 ? cf_dot_thread_t<16>(u_sm, v, d, vec_ok) : cf_dot_thread_t<32>(u_sm, v, d, vec_ok));
}

// 32 candidates cand[t0 .. t0 + 31] (negative = dropped, beyond n = absent): returns, in lane (sub, l) = (lane / LPR, lane % LPR),
// the score of candidate t0 + l * (32 / LPR) + sub.  `uu` = this lane's four elements 4l .. 4l + 3 of the user row.
// One load instruction covers 32 / LPR whole item rows (contiguous 16-byte pieces: every 128-byte line is touched once
// -- a lane per candidate touches 32 lines per instruction and the L1 tag stage becomes the limit).
template <int LPR>
__device__ __forceinline__ float cf_dot_round(const float4 uu, const float* __restrict__ Ie, int64_t ldi, int d, bool vec_ok,
                                              const int32_t* cand, int t0, int n, int lane) {
    constexpr int RPI = 32 / LPR, NI = LPR;
    const int l = lane & (LPR - 1), sub = lane / LPR;
    float p[NI];
#pragma unroll
    for (int h = 0; h < NI; h += 8) {
        float4 x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int t = t0 + (h + i) * RPI + sub;
            const int item = t < n ? cand[t] : -1;
            x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (item >= 0) x[i] = cf_load4(Ie + (int64_t)item * ldi, l, d, vec_ok);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) p[h + i] = cf_chain4(uu, x[i]);
    }
    // transposed butterfly: at width w the lanes with bit w set keep the upper half of their values, the others the lower
    // half, and each adds what its partner sends of the same candidates; value count and lane-group size halve together
#pragma unroll
    for (int w = LPR / 2; w >= 1; w >>= 1) {
        const bool up = (l & w) != 0;
#pragma unroll
        for (int a = 0; a < w; ++a) {
            const float keep = up ? p[a + w] : p[a];
            const float send = up ? p[a] : p[a + w];
            p[a] = keep + __shfl_xor_sync(0xffffffffu, send, w);
        }
    }
    return p[0];
}

// ------------------------------------------------------------------------------------------------------------------
// finalists: set bits of the row's bitmap -> unmasked -> exact fp32 -> top-k in contract order.  One warp per row, written
// for instruction count (the kernel is issue-bound at large batches: ~70 candidates per row, 20,000 rows):
//   * the set bits come out in ascending item order (lane = bitmap word, positions by a warp prefix sum);
//   * the mask is applied from the mask's side: lane q looks its masked item up in the sorted candidate list (binary
//     search), O(m log n) instead of n x m comparisons;
//   * exact scores 32 candidates at a time, 8 / 16 / 32 lanes per item row (cf_dot_round: coalesced reads);
//   * ranking counts, per element, the larger 32-bit value keys (one LDS broadcast feeds up to four elements of the
//     lane); equal values are ordered by item index = list position in a second pass that runs only when the rank sum
//     shows that two candidates share a value.
// ------------------------------------------------------------------------------------------------------------------
template <int E>
__device__ __forceinline__ void cf_rank_sweeps(const int32_t* cand, const uint32_t* keys, int n, int kept, int k, int lane, int64_t row,
                                               int64_t item_offset, int64_t* __restrict__ out_idx, float* __restrict__ out_val) {
    for (int e0 = 0; e0 * 32 < n; e0 += E) {
        uint32_t mk[E];
        int rk[E];
#pragma unroll
        for (int e = 0; e < E; ++e) { const int t = (e0 + e) * 32 + lane; mk[e] = t < n ? keys[t] : 0u; rk[e] = 0; }
        int u2 = 0;
        for (; u2 + 8 <= n; u2 += 8) {                               // 8 broadcast loads in flight, then the compares
            uint32_t ku[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) ku[i] = keys[u2 + i];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < E; ++e) rk[e] += ku[i] > mk[e];
        }
        for (; u2 < n; ++u2) {
            const uint32_t ku = keys[u2];
#pragma unroll
            for (int e = 0; e < E; ++e) rk[e] += ku > mk[e];
        }
        // all value keys distinct <=> the ranks of the live elements are a permutation of 0 .. kept-1 (checkable when one
        // sweep covers the list; with several sweeps the tie pass always runs)
        bool tie = n > 32 * E;
        if (!tie) {
            int sr = 0;
#pragma unroll
            for (int e = 0; e < E; ++e) sr += mk[e] != 0u ? rk[e] : 0;
            tie = __reduce_add_sync(0xffffffffu, sr) != kept * (kept - 1) / 2;
        }
        if (tie) {                                                   // equal values: lower item index (= list position) first
            for (int u2 = 0; u2 < n; ++u2) {
                const uint32_t ku = keys[u2];
#pragma unroll
                for (int e = 0; e < E; ++e) rk[e] += (ku == mk[e]) && (u2 < (e0 + e) * 32 + lane);
            }
        }
#pragma unroll
        for (int e = 0; e < E; ++e) {
            if (mk[e] != 0u && rk[e] < k) {
                out_idx[row * k + rk[e]] = (int64_t)cand[(e0 + e) * 32 + lane] + item_offset;
                out_val[row * k + rk[e]] = key_float(mk[e]);
            }
        }
    }
}

constexpr int CF_FIN_WARPS = 4;
template <int LPR>
__global__ void __launch_bounds__(32 * CF_FIN_WARPS, LPR <= 16 ? 8 : 6) cf_final_kernel(int64_t nb, int n_it, int64_t n_items, int d, int k, int64_t item_offset,
                                                                     const uint4* __restrict__ bitmap, const int64_t* __restrict__ users,
                                                                     const float* __restrict__ Ue, int64_t ldu, const float* __restrict__ Ie, int64_t ldi,
                                                                     const int32_t* __restrict__ mask_ptr, const int32_t* __restrict__ mask_items,
                                                                     int32_t* __restrict__ flags, int32_t* __restrict__ counter,
                                                                     int32_t* __restrict__ row_of_slot, int64_t* __restrict__ out_idx,
                                                                     float* __restrict__ out_val) {
    __shared__ int32_t cand_all[CF_FIN_WARPS][CF_CAP];
    __shared__ uint32_t key_all[CF_FIN_WARPS][CF_CAP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t row = (int64_t)blockIdx.x * CF_FIN_WARPS + warp;
    if (row >= nb) return;
    auto condemn = [&](int why) {                                    // the exact kernel takes the row
        if (lane == 0) {
            if (why) flags[row] = why;
            row_of_slot[atomicAdd(counter, 1)] = (int32_t)row;
        }
    };
    // everything that depends on the row number only is requested at once
    const int flagged = __ldg(flags + row);
    const int m0 = mask_ptr ? __ldg(mask_ptr + row) : 0, m1 = mask_ptr ? __ldg(mask_ptr + row + 1) : 0;
    const int64_t urow = users ? __ldg(users + row) : row;
    const uint4* bm = bitmap + row * n_it;
    uint4 b0 = make_uint4(0u, 0u, 0u, 0u);
    if (lane < n_it) b0 = __ldg(bm + lane);
    if (flagged) { condemn(0); return; }
    int32_t* cand = cand_all[warp];
    uint32_t* keys = key_all[warp];
    // 1. set bits -> candidate list in ascending item order; keys[] = 1 marks a live candidate
    int n = 0;
    for (int w0 = 0; w0 < n_it; w0 += 32) {
        const int wi = w0 + lane;
        uint4 b = b0;
        if (w0 > 0) { b = make_uint4(0u, 0u, 0u, 0u); if (wi < n_it) b = __ldg(bm + wi); }
        const int mine = __popc(b.x) + __popc(b.y) + __popc(b.z) + __popc(b.w);
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        int pos = n + incl - mine;
        n += __shfl_sync(0xffffffffu, incl, 31);
        if (mine) {
            const uint32_t ws[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint32_t x = ws[q];
                while (x) {
                    const int j = __clz(x);                          // bit (31 - j) <-> column 32 q + j of the tile
                    x &= ~(0x80000000u >> j);
                    if (pos < CF_CAP) { cand[pos] = wi * CF_TILE + q * 32 + j; keys[pos] = 1u; }
                    ++pos;
                }
            }
        }
    }
    if (n > CF_CAP) { condemn(4); return; }
    __syncwarp();
    // 2. masked train positives out: each masked item is looked up in the sorted list, its key becomes 0 (= dropped)
    for (int q0 = m0; q0 < m1; q0 += 32) {
        const int q = q0 + lane;
        if (q < m1) {
            const int item = __ldg(mask_items + q);
            int lo = 0, hi = n;                                      // first position with cand >= item
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (cand[mid] < item) lo = mid + 1; else hi = mid;
            }
            if (lo < n && cand[lo] == item) keys[lo] = 0u;
        }
    }
    __syncwarp();
    // 3. exact fp32 scores (float_key of a real score is never 0; -NaN would be: such a candidate is dropped).  Dropped
    //    candidates are marked in cand[] first (sign bit) so that a round reads one word per candidate.
    for (int t = lane; t < n; t += 32)
        if (keys[t] == 0u || cand[t] >= n_items) cand[t] |= (int32_t)0x80000000;
    __syncwarp();
    const bool vec_ok = (ldi & 3) == 0 && (d & 3) == 0 && ((((uintptr_t)Ie) & 15) == 0);
    const bool vec_u = (ldu & 3) == 0 && (d & 3) == 0 && ((((uintptr_t)Ue) & 15) == 0);
    const float4 uu = cf_load4(Ue + urow * ldu, lane & (LPR - 1), d, vec_u);
    int kept = 0;
    for (int t0 = 0; t0 < n; t0 += 32) {
        const float sc = cf_dot_round<LPR>(uu, Ie, ldi, d, vec_ok, cand, t0, n, lane);
        const int t = t0 + (lane & (LPR - 1)) * (32 / LPR) + lane / LPR;
        if (t < n) {
            const uint32_t key = cand[t] >= 0 ? float_key(sc) : 0u;
            kept += key != 0u;
            keys[t] = key;
        }
    }
    kept = __reduce_add_sync(0xffffffffu, kept);
    __syncwarp();
    if (kept < k) { condemn(8); return; }                            // (cannot happen for finite scores: the threshold is certified)
    // 4. rank = number of candidates with a larger value key; E elements of this lane per sweep of the list
    if (n <= 64) cf_rank_sweeps<2>(cand, keys, n, kept, k, lane, row, item_offset, out_idx, out_val);
    else if (n <= 96) cf_rank_sweeps<3>(cand, keys, n, kept, k, lane, row, item_offset, out_idx, out_val);
    else cf_rank_sweeps<4>(cand, keys, n, kept, k, lane, row, item_offset, out_idx, out_val);
}

// ------------------------------------------------------------------------------------------------------------------
// exact fp32 rows (flagged only): all items on CUDA cores, mask, then the selection of mmrec_topk_rows_f32
// (cta_topk_from_keys, select.cuh).  CTA `sl` serves the flagged rows sl, sl + CF_EX_SLOTS, ... with its own key buffer;
// all CTAs exit at once when nothing was flagged.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cf_exact_kernel(const int64_t* __restrict__ users, const float* __restrict__ Ue, int64_t ldu,
                                                       int64_t n_items, const float* __restrict__ Ie, int64_t ldi, int d, int k,
                                                       int64_t item_offset, const int32_t* __restrict__ mask_ptr,
                                                       const int32_t* __restrict__ mask_items, const int32_t* __restrict__ counter,
                                                       const int32_t* __restrict__ row_of_slot, unsigned* __restrict__ keys_all,
                                                       int64_t* __restrict__ out_idx, float* __restrict__ out_val) {
    __shared__ TopkSmem sm;
    __shared__ __align__(16) float u_ex[128];
    const int n_flagged = *counter;
    const int tid = threadIdx.x;
    unsigned* keys = keys_all + (int64_t)blockIdx.x * n_items;
    for (int fr = blockIdx.x; fr < n_flagged; fr += gridDim.x) {
        const int64_t row = row_of_slot[fr];
        __syncthreads();
        // ---- keys: one thread per item, cf_dot_thread's arithmetic (the row gets the same bits whichever kernel served it)
        const float* u = Ue + (users ? users[row] : row) * ldu;
        if (tid < 128) u_ex[tid] = tid < d ? u[tid] : 0.f;
        __syncthreads();
        const bool vec_ok = (ldi & 3) == 0 && (d & 3) == 0 && ((((uintptr_t)Ie) & 15) == 0);
        for (int64_t i = tid; i < n_items; i += 256) keys[i] = float_key(cf_dot_thread(u_ex, Ie + i * ldi, d, vec_ok));
        __syncthreads();
        const int m0 = mask_ptr ? mask_ptr[row] : 0, m1 = mask_ptr ? mask_ptr[row + 1] : 0;
        for (int q = m0 + tid; q < m1; q += 256) {
            const int64_t item = mask_items[q];
            if (item >= 0 && item < n_items) keys[item] = float_key(-1e10f);          // src/common/trainer.py:307
        }
        __syncthreads();
        cta_topk_from_keys<256>([=](int64_t i) { return keys[i]; }, n_items, k, item_offset, out_idx + row * k, out_val + row * k, sm);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
static inline int cf_kp(int d) { return d <= 32 ? 32 : (d <= 64 ? 64 : 128); }
static inline int cf_gw(int64_t n_items) { return n_items <= 16384 ? 1 : (n_items <= 32768 ? 2 : (n_items <= 65536 ? 4 : 8)); }

constexpr size_t CF_CAT_HEADER = 1024;          // {max scaled item norm (fp32 bits), n_items, d, KP, largest |element| (fp32 bits)} + padding

size_t cf_catalog_bytes(int64_t n_items, int d) {
    if (n_items <= 0 || d < 1 || d > 128) return 0;
    const int64_t n_it = (n_items + CF_TILE - 1) / CF_TILE;
    return CF_CAT_HEADER + (size_t)n_it * CF_TILE * cf_kp(d) * 2;
}

int cf_catalog_pack(int64_t n_items, const float* Ie, int64_t ldi, int d, void* cat, size_t cat_bytes, cudaStream_t stream) {
    const size_t need = cf_catalog_bytes(n_items, d);
    if (!need || !cat || cat_bytes < need || (((uintptr_t)cat) & 1023)) { set_error("catalog_pack: bad shape, or buffer null / not 1024-byte aligned / smaller than mmrec_catalog_bytes"); return MMREC_EINVAL; }
    const int KP = cf_kp(d);
    const int64_t n_it = (n_items + CF_TILE - 1) / CF_TILE;
    // header: word 0 = running maximum (scaled) norm, word 4 = largest magnitude of the table, both zeroed here; thread 0
    // of the pack kernel fills in the rest
    MMREC_CUDA(cudaMemsetAsync(cat, 0, CF_CAT_HEADER, stream));
    {
        const int64_t blocks = (n_items + 7) / 8;
        absmax_norm_kernel<<<(unsigned)(blocks < 2368 ? blocks : 2368), 256, 0, stream>>>(n_items, Ie, ldi, d, nullptr, (uint32_t*)cat + 4, nullptr);
        MMREC_LAUNCH_CHECK();
    }
    const int64_t threads = n_it * CF_TILE * (KP / 8);
    cf_pack_items_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(n_items, Ie, ldi, d, KP, (uint4*)((char*)cat + CF_CAT_HEADER),
                                                                                  (uint32_t*)cat, threads);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

struct CfPlan {
    int KP, gw, G;
    int64_t n_it, rows_blk, rows_pad, n_pairs;
    size_t off_cat, off_upk, off_unorm, off_gmax, off_thr, off_bitmap, off_flags, off_mask, off_keys, total;
};

static CfPlan cf_plan(int64_t B, int64_t n_items, int d, int64_t mask_nnz, bool with_cat) {
    CfPlan P;
    P.KP = cf_kp(d);
    P.gw = cf_gw(n_items);
    P.n_it = (n_items + CF_TILE - 1) / CF_TILE;
    P.G = (int)(P.n_it * (8 / P.gw));
    // row block: group maxima + bitmap of a block stay below ~512 MB
    const int64_t per_row = (int64_t)P.G * 4 + P.n_it * 16;
    int64_t rb = (512ll << 20) / per_row / (2 * CF_TILE) * (2 * CF_TILE);
    if (rb < 2 * CF_TILE) rb = 2 * CF_TILE;
    if (rb > 65536) rb = 65536;
    P.rows_blk = B < rb ? B : rb;
    P.rows_pad = (P.rows_blk + 2 * CF_TILE - 1) / (2 * CF_TILE) * (2 * CF_TILE);
    P.n_pairs = P.rows_pad / (2 * CF_TILE);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes, 1024); return o; };
    P.off_cat = take(with_cat ? cf_catalog_bytes(n_items, d) : 0);
    P.off_upk = take((size_t)P.rows_pad * P.KP * 2);
    P.off_unorm = take((size_t)P.rows_pad * 4);
    P.off_gmax = take((size_t)P.rows_blk * P.G * 4);
    P.off_thr = take((size_t)P.rows_pad * 4);
    P.off_bitmap = take((size_t)P.rows_blk * P.n_it * 16);
    P.off_flags = take((size_t)(2 * P.rows_blk + 2) * 4);            // flags [rows_blk] | counter | row_of_slot [rows_blk]   (flags + counter zeroed per block)
    P.off_mask = take(batch_mask(nullptr, mask_nnz, nullptr, nullptr, B, 0, 0).bytes);
    P.off_keys = take((size_t)CF_EX_SLOTS * n_items * 4);
    P.total = off + 1024;
    return P;
}

bool score_cf_supported(int64_t B, int64_t n_items, int d, int k) {
    if (!(B > 0 && d >= 1 && d <= 128 && k >= 1 && k <= 256 && n_items < (1ll << 31))) return false;
    const int64_t G = (n_items + CF_TILE - 1) / CF_TILE * (8 / cf_gw(n_items));
    return G >= 2 * (int64_t)k;                                      // enough groups for need = k + masked items (rows that want more go to the exact kernel)
}

size_t score_cf_workspace_bytes(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat) {
    if (!score_cf_supported(B, n_items, d, k)) return 0;
    return cf_plan(B, n_items, d, mask_nnz, with_cat).total;
}

// Stage timing (tuning aid): with env MMREC_CF_TIMING set, the stages of the LAST score_cf call are bracketed by CUDA events
// (not under stream capture); mmrec_debug_cf_timing reads them back in microseconds.
static cudaEvent_t g_cf_ev[10];
static int g_cf_nev = 0, g_cf_timing = -1;
static inline void cf_mark(cudaStream_t stream) {
    if (g_cf_timing <= 0 || g_cf_nev >= 10) return;
    if (!g_cf_ev[g_cf_nev]) cudaEventCreate(&g_cf_ev[g_cf_nev]);
    cudaEventRecord(g_cf_ev[g_cf_nev++], stream);
}
int score_cf_timing(float* us, int cap) {
    int n = 0;
    for (int i = 0; i + 1 < g_cf_nev && n < cap; ++i) {
        cudaEventSynchronize(g_cf_ev[i + 1]);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, g_cf_ev[i], g_cf_ev[i + 1]);
        us[n++] = ms * 1000.f;
    }
    return n;
}

// returns 1 = done, 0 = unsupported shape / workspace (caller uses the unfused path), <0 error.  `cat` = a catalogue packed
// by cf_catalog_pack for exactly (n_items, Ie, d), or NULL: then it is packed into the workspace first.
int score_cf(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items, const float* Ie, int64_t ldi,
             int d, const void* cat, int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int k, int64_t item_offset,
             int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, cudaStream_t stream) {
    if (!score_cf_supported(B, n_items, d, k) || !ws) return 0;
    const CfPlan P = cf_plan(B, n_items, d, mask_nnz, cat == nullptr);
    char* base = (char*)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
    if (ws_bytes < P.total + (size_t)(base - (char*)ws)) return 0;
    if (int rc = set_smem_once<cf_pass_kernel<1, 8>, cf_pass_kernel<1, 4>, cf_pass_kernel<1, 2>, cf_pass_kernel<1, 1>, cf_pass_kernel<2, 8>>(227 * 1024))
        return rc;
    if (g_cf_timing < 0) g_cf_timing = getenv("MMREC_CF_TIMING") ? 1 : 0;
    g_cf_nev = 0;
    cf_mark(stream);                                                  // stages: pack | prep + mask | pass 1 | thr | pass 2 | final | exact
    if (!cat) {
        int rc = cf_catalog_pack(n_items, Ie, ldi, d, base + P.off_cat, cf_catalog_bytes(n_items, d), stream);
        if (rc) return rc;
        cat = base + P.off_cat;
    }
    cf_mark(stream);
    const uint32_t* max_norm = (const uint32_t*)cat;
    const char* Ipk = (const char*)cat + CF_CAT_HEADER;
    uint4* Upk = (uint4*)(base + P.off_upk);
    float *unorm = (float*)(base + P.off_unorm), *gmax = (float*)(base + P.off_gmax), *thr = (float*)(base + P.off_thr);
    uint4* bitmap = (uint4*)(base + P.off_bitmap);
    int32_t* flags = (int32_t*)(base + P.off_flags);
    int32_t* counter = flags + P.rows_blk;
    int32_t* row_of_slot = counter + 1;
    const BatchMask M = batch_mask(base + P.off_mask, mask_nnz, mask_rows, mask_cols, B, item_offset, n_items);
    unsigned* keys = (unsigned*)(base + P.off_keys);
    constexpr int T = MC_SORTED_THREADS;                              // (256: cf_prep_kernel's blocks run the sorted mask pass)
    const bool has_mask = mask_nnz > 0;
    const bool small_mask = has_mask && mask_small(B, mask_nnz);
    if (has_mask && !small_mask) {
        int rc = batch_mask_large(M, stream);
        if (rc) return rc;
    }
    const CfSmem L = cf_smem(P.KP);
    const int sms = sm_count();
    for (int64_t r0 = 0; r0 < B; r0 += P.rows_blk) {
        const int64_t nb = (B - r0) < P.rows_blk ? (B - r0) : P.rows_blk;
        const int64_t nb_pad = (nb + 2 * CF_TILE - 1) / (2 * CF_TILE) * (2 * CF_TILE);
        const int64_t n_pairs = nb_pad / (2 * CF_TILE);
        const int64_t* ub = users ? users + r0 : nullptr;
        const float* ue = users ? Ue : Ue + r0 * ldu;
        const int32_t* mp = has_mask ? M.ptr + r0 : nullptr;
        // prep: [mask CSR of the whole batch (first block, sorted case)] + user operand + zeroed flags / counter
        const int64_t mask_blocks = (small_mask && r0 == 0) ? mask_sorted_blocks(mask_nnz) : 0;
        const int64_t pack_threads = nb_pad * (P.KP / 8);
        const int64_t zero_words = P.rows_blk + 1;
        cf_prep_kernel<<<(unsigned)(mask_blocks + (pack_threads + zero_words + T - 1) / T), T, 0, stream>>>(
            mask_blocks, M, nb, ub, ue, ldu, d, P.KP, Upk, unorm, pack_threads, (uint32_t*)flags, zero_words);
        MMREC_LAUNCH_CHECK();
        if (mask_blocks) {
            int rc = batch_mask_unsorted(M, stream);
            if (rc) return rc;
        }
        cf_mark(stream);
        CfParams p;
        p.Upk = (const char*)Upk; p.Ipk = Ipk; p.KP = P.KP; p.n_it = (int)P.n_it; p.B = nb; p.n_items = n_items; p.n_units = n_pairs * P.n_it;
        p.gmax = gmax; p.G = P.G; p.gw = P.gw; p.thr = thr; p.bitmap = bitmap;
        { static int dbg = -1; if (dbg < 0) { const char* e = getenv("MMREC_CF_DEBUG"); dbg = e ? atoi(e) : 0; } p.dbg = dbg; }
        const unsigned grid = (unsigned)(p.n_units < sms ? p.n_units : sms);
        switch (P.gw) {
            case 1: cf_pass_kernel<1, 8><<<grid, CF_THREADS, L.total, stream>>>(p); break;
            case 2: cf_pass_kernel<1, 4><<<grid, CF_THREADS, L.total, stream>>>(p); break;
            case 4: cf_pass_kernel<1, 2><<<grid, CF_THREADS, L.total, stream>>>(p); break;
            default: cf_pass_kernel<1, 1><<<grid, CF_THREADS, L.total, stream>>>(p); break;
        }
        MMREC_LAUNCH_CHECK();
        cf_mark(stream);
        cf_thr_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, stream>>>(nb, P.G, (int)((n_items + 16 * P.gw - 1) / (16 * P.gw)), k, d, gmax, unorm, max_norm, mp, thr, flags);
        MMREC_LAUNCH_CHECK();
        cf_mark(stream);
        cf_pass_kernel<2, 8><<<grid, CF_THREADS, L.total, stream>>>(p);
        MMREC_LAUNCH_CHECK();
        cf_mark(stream);
        {
            const unsigned fg = (unsigned)((nb + CF_FIN_WARPS - 1) / CF_FIN_WARPS);
#define CF_FINAL(LPR) cf_final_kernel<LPR><<<fg, 32 * CF_FIN_WARPS, 0, stream>>>(nb, (int)P.n_it, n_items, d, k, item_offset, bitmap, ub, ue, ldu, Ie, ldi, mp, \
                                                                            M.items, flags, counter, row_of_slot, out_idx + r0 * k, out_val + r0 * k)
            if (cf_lpr(d) == 8) CF_FINAL(8); else if (cf_lpr(d) == 16) CF_FINAL(16); else CF_FINAL(32);
#undef CF_FINAL
        }
        MMREC_LAUNCH_CHECK();
        cf_mark(stream);
        cf_exact_kernel<<<CF_EX_SLOTS, 256, 0, stream>>>(ub, ue, ldu, n_items, Ie, ldi, d, k, item_offset, mp, M.items, counter, row_of_slot, keys,
                                                         out_idx + r0 * k, out_val + r0 * k);
        MMREC_LAUNCH_CHECK();
        cf_mark(stream);
    }
    return 1;
}

// The scratch layout of a call with these arguments (diagnostic, host only): the dimensions and byte offsets from the
// 1024-aligned workspace base that mmrec_debug_cf_scratch documents.  Returns the number of entries, -1 = not fused.
int score_cf_scratch(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat, int64_t* out, int cap) {
    if (!score_cf_supported(B, n_items, d, k)) return -1;
    const CfPlan P = cf_plan(B, n_items, d, mask_nnz, with_cat);
    const int64_t v[] = {P.rows_blk, P.rows_pad, P.KP, P.gw, P.n_it, P.G, (n_items + 16 * P.gw - 1) / (16 * P.gw),
                         with_cat ? (int64_t)P.off_cat : -1, (int64_t)CF_CAT_HEADER, (int64_t)P.off_upk, (int64_t)P.off_unorm,
                         (int64_t)P.off_gmax, (int64_t)P.off_thr, (int64_t)P.off_bitmap, (int64_t)P.off_flags, (int64_t)P.total};
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n && i < cap; ++i) out[i] = v[i];
    return n;
}

// rows of the last row block that went to the exact kernel (synchronises; diagnostic)
int64_t score_cf_fallback_rows(const void* ws, int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat) {
    if (!score_cf_supported(B, n_items, d, k) || !ws) return -1;
    const CfPlan P = cf_plan(B, n_items, d, mask_nnz, with_cat);
    const char* base = (const char*)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
    int32_t n = 0;
    if (cudaMemcpy(&n, base + P.off_flags + (size_t)P.rows_blk * 4, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    if (getenv("MMREC_DEBUG")) {
        const int64_t nb = B % P.rows_blk ? B % P.rows_blk : P.rows_blk;
        int32_t* h = (int32_t*)malloc((size_t)nb * 4);
        if (h && cudaMemcpy(h, base + P.off_flags, (size_t)nb * 4, cudaMemcpyDeviceToHost) == cudaSuccess) {
            long long why[4] = {0, 0, 0, 0};
            for (int64_t i = 0; i < nb; ++i)
                for (int b = 0; b < 4; ++b) why[b] += (h[i] >> b) & 1;
            fprintf(stderr, "mmrec: exact-path rows %d of %lld (need > groups %lld, non-finite %lld, > %d candidates %lld, < k kept %lld)\n", n,
                    (long long)nb, why[0], why[1], CF_CAP, why[2], why[3]);
        }
        free(h);
    }
    return n;
}

}  // namespace mmrec
