// K7: item-item cosine kNN (`sim = X X^T; torch.topk(sim, k)`, src/models/freedom.py:79-91, src/utils/utils.py:165-172)
// as a CERTIFIED FILTER on the tensor cores with the top-k fused, for feature tables of any width F.
//
// Result contract: for each query row q, the top-k of s(q, i) = X[q] . X[i] over all n items, values descending, equal
// values by ascending index -- exactly what mmrec_score_f32 on its CUDA-core path (gemm_simt.cuh) followed by
// mmrec_topk_rows_f32 returns, bit for bit.  That route is one fmaf chain per output over k ascending from 0.f, K padded with
// zeros to a multiple of 32 (a padding step fmaf(0, 0, acc) turns a -0.0 sum into +0.0), ranked on float_key (common.cuh).
// Every value this file returns is that chain (knn_exact below), and the order is taken on those values.
//
//   absmax_norm_kernel  one warp per table row: largest |element| of the table (its bit pattern; inf / NaN patterns sort
//                       above every finite one, so a non-finite element is detected here) and each row's norm, rounded up.
//   knn_pack_kernel     X (and per row block the query rows) -> fp16, round to nearest, after ONE power-of-two scale sc for
//                       the whole table that brings the largest element into [2^14, 2^15) (fp16_scale_for,
//                       tc_common.cuh), into the canonical K-major no-swizzle wgmma layout (store_fp16x8): tiles of 128
//                       rows, K padded to a multiple of 64 with zeros; a 64-wide K chunk of a tile is one contiguous 16 KB
//                       range.
//   knn_pass_kernel     s~ = the scaled score on the tensor cores (wgmma m64n128k16 f16 -> fp32), K-loop over F in chunks of
//                       64 streamed through a 4-stage bulk-copy / mbarrier ring (48 KB per stage: 256 query rows + 128
//                       items).  Epilogue (group_max_store<8>): the maximum of every group of 16 consecutive items,
//                       gmax[row][group].  A unit = (pair of 128-row query tiles, 128-item tile); units are dealt to the
//                       CTAs in contiguous runs, the query pair varies fastest so that consecutive units reuse the item
//                       tile from L2.
//   knn_thr_kernel      one CTA per row: t = a value <= the k-th largest group maximum with at least k maxima >= t (radix
//                       select on the top 24 key bits, lower bucket edge); thr = t - 2 eps' (set_threshold).
//   knn_final_kernel    one CTA per row: every group with gmax >= thr -> every item of those groups scored EXACTLY (knn_exact,
//                       from the original fp32 rows) -> bitonic sort on (float_key, ~index) -> top-k.
//   exact route         rows the filter does not serve (fewer than k groups, more than KN_CAP candidates, a non-finite
//                       margin) are listed; after each row block the host reads the count and runs the existing route on
//                       them (exact_rows.cuh): gemm_nt_kernel (gemm_simt.cuh, the same template instance as mmrec_score_f32)
//                       on the gathered rows + mmrec_topk_rows_f32, then a scatter.  Bit-identical by construction.  A
//                       table with any non-finite element (a zero row normalises to NaN) takes that route for every row.
//
// ERROR BOUND (scaled domain: a = sc X[q], b = sc X[i]; the exact value s is the fp32 chain above times sc^2, exact for a
// power of two barring underflow).  Write s* for the real dot product a . b.
//   (1) operands: fp16 round to nearest, |da| <= 2^-11 |a_k| + 2^-25 (2^-25: half the fp16 subnormal spacing), so
//       |a^ . b^ - s*| <= (2^-10 + 2^-22) |a| |b| + 2^-25 sqrt(F) (|a| + |b|) + F 2^-50                 (Cauchy-Schwarz);
//       the products a^_k b^_k (11 x 11 significand bits) are exact in fp32.
//   (2) tensor-core accumulation over S = F_pad / 16 MMA steps.  ASSUMPTION about the hardware: one m64n128k16 step adds its
//       16 exact products to the fp32 accumulator c with an error of at most 2^-20 (|c| + sum_j |p_j|) -- eight fp32 ulps
//       of the magnitude sum.  The H100 adder, as measured on an H100 SXM (tests/test_gpu_filter_stages.py: one product
//       2^28 at the bottom of its binade beside 3 / 7 / 15 products just below 2^(5 - g), g = 0 .. 3, and the same after a
//       large accumulator; reproduced exactly by the model in tests/test_filter_stages_host.py): every addend (c and the
//       16 products) is aligned to the largest one's exponent and truncated 2 bits below its ulp, the aligned sum is
//       exact and is then truncated to 24 bits.  So the 16 smaller addends lose < 16 x ulp / 4 and the final truncation
//       < one ulp of the result: < 5 x 2^-23 (|c| + sum |p|) = 2.5 x 2^-22; the worst measured is 2.25 x 2^-22 (15
//       products just below ulp / 2).  2^-20 leaves a factor 1.6 on the model.  Summed over the steps, with
//       |c_s| <= sum of the earlier |p| (1 + small):
//       |s~ - a^ . b^| <= S 2^-20 (1 + 2^-10) sum_k |a^_k b^_k| <= S 2^-20 (1 + 2^-9) |a| |b|.
//   (3) the exact value itself is an fp32 chain of F fmaf: |s - s*| <= gamma_F sum |a_k b_k|, gamma_F = F 2^-24 / (1 - F 2^-24)
//       (<= F 2^-24 (1 + 2^-9) for F <= 2^15; longer rows only make the margin larger through the formula below).
//   Hence |s~ - s| <= eps(F) |a| |b| + sub(F),  eps(F) = 2^-10 + 2^-22 + (S 2^-20 + F 2^-24)(1 + 2^-9),
//   sub(F) = 2^-25 sqrt(F) (|a| + |b|) + F 2^-50 + F 2^-149 sc^2 (subnormal steps of the unscaled chain).
//   At F = 4096: eps = 9.77e-4 + 2.44e-4 + 2.44e-4 = 1.47e-3.  eps' (per query row) uses |a| = the row's norm and max|b| =
//   the largest row norm, both rounded up; the margin is 2 eps' inflated by 2^-8 for the rounding of its own arithmetic.
// CERTIFICATE: at least k groups have a maximum >= t, so at least k distinct items have s~ >= t and s >= t - eps'; the k-th
// largest exact value s_k is >= t - eps'.  Every member of the true top-k and every item tied with s_k has s >= s_k, so its
// s~ >= t - 2 eps' >= thr and its group survives.  The exact ranking of the survivors therefore equals the ranking of all
// items, ties included.
//
// SHRINK ROUTE (mmrec_knn_topk_shrink_f32, ItemKNNCBF: src/models/itemknncbf.py:56-65).  The ranking value is
// v = s / D, D = fl(fl(nq ni) + shrink) with the caller's norms nq = norms[q], ni = norms[i], and an IEEE division; every
// returned value is that division of the exact chain (shrink_div).  The three kernels take it as the template parameter
// SHRINK (the cosine instances are unchanged); the pass epilogue turns each scaled score into v~ = fl((s~ / sc^2) / D)
// (knn_shrink_tile), the exact route divides its score block elementwise (knn_shrink_rows_kernel).
// BOUND.  Write A = rnorm[q], B_i = rnorm[i] (the kernel's norms, rounded up), unscaled, E_i = eps(F) A B_i + sub_i the
// bound above on |s~ / sc^2 - s| (sub_i = sub(F) / sc^2 + the underflow of the two exact power-of-two products).  Then
//   |v~ - v| <= E_i / D + 2^-24 (|v~| + |v|)                                        (the two divisions round once each),
//   A B_i / D <= (A / nq)(B_i / ni) (nq ni) / D <= Rq Rmax f (1 + 2^-22),
// Rq = A / nq, Rmax = max_i B_i / ni (0 for a zero row), and f = nq nmax / (nq nmax + shrink) <= 1: x / (x + shrink) grows with
// x, so the largest given norm nmax bounds it -- the key fact |q||i| / (|q||i| + shrink) <= 1, which scales eps down by up to
// shrink / (|q||i| + shrink).  With RR = Rq Rmax f (rounded up), Dmin <= nq nmin + shrink (rounded down, nmin the smallest
// given norm) and vmax = RR (1 + 2 eps) + sub / Dmin >= |v|, |v~|:
//   |v~ - v| <= e = eps RR + sub / Dmin + 2^-23 vmax,   thr = t - 2 e (1 + 2^-8),
// and the certificate above holds with v in place of s.  A negative or non-finite shrink, a non-finite norm, or shrink = 0
// beside a zero norm (0 / 0) sends every row to the exact route; a NaN / inf margin (a zero norm beside a non-zero row)
// sends that row.
#include <cstdio>
#include <cstdlib>

#include "exact_rows.cuh"
#include "gemm_simt.cuh"
#include "select.cuh"
#include "tc_common.cuh"

namespace mmrec {

using namespace tc;

constexpr int KN_TILE = 128;                            // rows of an operand tile
constexpr int KN_KC = 64;                               // halfs of K per ring stage
constexpr uint32_t KN_CHUNK = KN_TILE * KN_KC * 2;      // 16 KB: one tile, one K chunk
constexpr uint32_t KN_STAGE = 3 * KN_CHUNK;             // query tiles 2p, 2p+1 | item tile
constexpr int KN_STAGES = 4;
constexpr int KN_CONSUMER_WARPS = 8;
constexpr int KN_THREADS = 32 * KN_CONSUMER_WARPS + 128;     // + one producer warpgroup (one thread issues the copies)
constexpr uint32_t KN_BARS = KN_STAGES * KN_STAGE;      // FULL[s] | EMPTY[s]
constexpr uint32_t KN_SMEM = KN_BARS + 2 * KN_STAGES * 8;
constexpr int KN_GROUP = 16;                            // items per group maximum
constexpr int KN_CAP = 4096;                            // candidates (16 x surviving groups) one CTA scores per row
constexpr int KN_FIN_THREADS = 256;

// ---- table norms / largest magnitude (declared in tc_common.cuh; score_cf.cu runs it without the norms) -------------
__global__ void __launch_bounds__(256) absmax_norm_kernel(int64_t n, const float* __restrict__ X, int64_t ldx, int F, float* __restrict__ rnorm,
                                                          uint32_t* __restrict__ amax_out, uint32_t* __restrict__ nmax_out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * 8;
    // a per-lane chain of ceil(F / 32) squares and a 5-level tree: relative error of the sum of squares below (F/32 + 6) 2^-24
    const float up = 1.0f + (float)(F / 32 + 8) * 0x1p-23f;
    uint32_t amax = 0u, nmax = 0u;
    for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += warps) {
        const float* row = X + r * ldx;
        float ss = 0.f;
        for (int c = lane; c < F; c += 32) {
            const float x = __ldg(row + c);
            ss = fmaf(x, x, ss);
            const uint32_t b = __float_as_uint(x) & 0x7fffffffu;
            amax = b > amax ? b : amax;
        }
        if (rnorm) {
            ss = warp_sum(ss);
            const float nrm = sqrtf(ss) * up;
            if (lane == 0) rnorm[r] = nrm;
            const uint32_t nb = __float_as_uint(nrm);
            nmax = nb > nmax ? nb : nmax;
        }
    }
    amax = __reduce_max_sync(0xffffffffu, amax);
    if (lane == 0 && amax) atomicMax(amax_out, amax);
    if (lane == 0 && nmax) atomicMax(nmax_out, nmax);                // (a NaN norm only happens with a non-finite element)
}

// One thread per (tile, k block of 8, row of the tile): consecutive threads write one contiguous 2 KB core-matrix column and
// read one 32-byte sector each.  Source row = idx ? idx[row] : row_off + row; rows >= n_rows are zero.
__global__ void __launch_bounds__(256) knn_pack_kernel(int64_t n_rows, const int64_t* __restrict__ idx, int64_t row_off,
                                                       const float* __restrict__ X, int64_t ldx, int F, int KP,
                                                       const uint32_t* __restrict__ header, uint4* __restrict__ out, int64_t n_threads) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_threads) return;
    const int kblks = KP / 8;
    const int rr = (int)(t % KN_TILE);
    const int64_t tk = t / KN_TILE;
    const int kb = (int)(tk % kblks);
    const int64_t tile = tk / kblks;
    const int64_t row = tile * KN_TILE + rr;
    const float sc = fp16_scale_for(__ldg(header));
    float x[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = 0.f;
    if (row < n_rows) {
        const float* src = X + (idx ? __ldg(idx + row) : row_off + row) * ldx + kb * 8;
        if (kb * 8 + 8 <= F && ((ldx & 3) == 0) && ((((uintptr_t)src) & 15) == 0)) {
            const float4 a = ldg4(src), b = ldg4(src + 4);
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (kb * 8 + e < F) x[e] = __ldg(src + e);
        }
    }
    store_fp16x8(out, tile, kblks, kb, rr, x, sc);
}

// ---- the tensor-core pass ---------------------------------------------------------------------------------------------
struct KnnParams {
    const char* Qpk;                            // query rows of the block, fp16 tiles [rows_pad / 128][KP/8][16][8][8]
    const char* Xpk;                            // all items, the same layout
    int KP, nc;                                 // padded K, chunks of 64
    int n_pairs, nb, n;                         // query tile pairs and rows of the block, items
    int64_t n_units;
    float* gmax; int G;                         // [nb][G], G = 8 n_it
    // shrink route only: v = s / (norms[q] norms[i] + shrink); query q = rows ? rows[row] : row_off + row
    const float* norms; float shrink;
    const int64_t* rows; int64_t row_off;
    const uint32_t* header;
};

// The shrink denominator, two IEEE roundings (multiply, then add) and an IEEE division: `ij.div(i_norm * i_norm.T + shrink)`.
__device__ __forceinline__ float shrink_div(float s, float nq, float ni, float shrink) {
    return __fdiv_rn(s, __fadd_rn(__fmul_rn(nq, ni), shrink));
}

// Shrink route, pass epilogue: this thread's 4 rows x 32 columns of scaled scores s~ become v~ = (s~ / sc^2) / D, D the
// exact route's denominator.  (1 / sc is a power of two: the two products are exact barring underflow.)
__device__ __forceinline__ void knn_shrink_tile(const KnnParams& p, float (&acc0)[64], float (&acc1)[64], int row0, int q, int cur_it,
                                                int n_valid) {
    const float isc = 1.0f / fp16_scale_for(__ldg(p.header));
    float qn[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int row = row0 + 64 * (r >> 1) + 8 * (r & 1);
        qn[r] = row < p.nb ? __ldg(p.norms + (p.rows ? __ldg(p.rows + row) : p.row_off + row)) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * q + e;
            const float ni = c < n_valid ? __ldg(p.norms + (int64_t)cur_it * KN_TILE + c) : 0.f;
#pragma unroll
            for (int e2 = 0; e2 < 2; ++e2) {
                acc0[4 * j + 2 * e2 + e] = shrink_div(acc0[4 * j + 2 * e2 + e] * isc * isc, qn[e2], ni, p.shrink);
                acc1[4 * j + 2 * e2 + e] = shrink_div(acc1[4 * j + 2 * e2 + e] * isc * isc, qn[2 + e2], ni, p.shrink);
            }
        }
    }
}

__device__ __forceinline__ void knn_producer(const KnnParams& p, uint32_t sbase, int64_t u0, int64_t u1) {
    const uint32_t bar = sbase + KN_BARS;
    const int64_t tile_bytes = (int64_t)KN_TILE * p.KP * 2;
    uint32_t slot = 0, ph = 1;
    for (int64_t u = u0; u < u1; ++u) {
        const int64_t it = u / p.n_pairs, pair = u - it * p.n_pairs;
        const char* a0 = p.Qpk + 2 * pair * tile_bytes;
        const char* b0 = p.Xpk + it * tile_bytes;
        for (int c = 0; c < p.nc; ++c) {
            const uint32_t full = bar + slot * 8;
            mbar_wait(bar + (KN_STAGES + slot) * 8, ph);
            mbar_expect_tx(full, KN_STAGE);
            const uint32_t dst = sbase + slot * KN_STAGE;
            const int64_t off = (int64_t)c * KN_CHUNK;
            bulk_g2s(dst, a0 + off, KN_CHUNK, full);
            bulk_g2s(dst + KN_CHUNK, a0 + tile_bytes + off, KN_CHUNK, full);
            bulk_g2s(dst + 2 * KN_CHUNK, b0 + off, KN_CHUNK, full);
            if (++slot == KN_STAGES) { slot = 0; ph ^= 1; }
        }
    }
}

template <bool SHRINK>
__device__ __forceinline__ void knn_consumer(const KnnParams& p, uint32_t sbase, int64_t u0, int64_t u1, int h) {
    const uint32_t bar = sbase + KN_BARS;
    constexpr uint32_t LBO = (KN_TILE / 8) * 128, SBO = 128;
    constexpr uint64_t KSTEP = (2 * LBO) >> 4;                         // one K step of 16 = two 16-byte k blocks
    const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31, q = lane & 3;
    float acc0[64], acc1[64];                                          // rows 16 w + lane / 4 (+ 8) and 64 + the same
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    uint32_t slot = 0, ph = 0;
    int it = (int)(u0 / p.n_pairs), pair = (int)(u0 - (int64_t)it * p.n_pairs);
    for (int64_t u = u0; u < u1; ++u) {
        const int base = pair * (2 * KN_TILE) + h * KN_TILE;
        const bool live = base < p.nb;                                 // (a whole half beyond the block: no MMAs, no output)
        uint32_t prev = 0;
        for (int c = 0; c < p.nc; ++c) {
            mbar_wait(bar + slot * 8, ph);
            if (live) {
                const uint32_t st = sbase + slot * KN_STAGE;
                uint64_t ad0 = smem_desc(st + h * KN_CHUNK, LBO, SBO), ad1 = smem_desc(st + h * KN_CHUNK + 1024, LBO, SBO);
                uint64_t bd = smem_desc(st + 2 * KN_CHUNK, LBO, SBO);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < KN_KC / 16; ++j) {
                    const uint32_t accum = (c > 0 || j > 0) ? 1u : 0u;
                    wgmma_f16<KN_TILE>(acc0, ad0, bd, accum);
                    wgmma_f16<KN_TILE>(acc1, ad1, bd, accum);
                    ad0 += KSTEP; ad1 += KSTEP; bd += KSTEP;
                }
                wgmma_commit();
                wgmma_wait<1>();                                       // the previous chunk's MMAs are done: its stage is free
                if (c > 0) warp_arrive(bar + (KN_STAGES + prev) * 8);
            } else {
                warp_arrive(bar + (KN_STAGES + slot) * 8);
            }
            prev = slot;
            if (++slot == KN_STAGES) { slot = 0; ph ^= 1; }
        }
        const int cur_it = it;
        if (++pair == p.n_pairs) { pair = 0; ++it; }
        if (!live) continue;
        wgmma_wait<0>();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        warp_arrive(bar + (KN_STAGES + prev) * 8);
        // ---- epilogue: maxima of the 8 groups of 16 columns of rows row0 + 8 e2 (acc0) and row0 + 64 + 8 e2 (acc1)
        const int n_valid = p.n - cur_it * KN_TILE;
        const int row0 = base + 16 * w + (lane >> 2);
        if constexpr (SHRINK) knn_shrink_tile(p, acc0, acc1, row0, q, cur_it, n_valid);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = row0 + 64 * (r >> 1) + 8 * (r & 1);
            // (row * G < 2^27: a row block's maxima stay below 512 MB)
            group_max_store<8>(r < 2 ? acc0 : acc1, r & 1, q, n_valid, row, p.nb, [&] { return p.gmax + (row * p.G + cur_it * 8); });
        }
    }
}

template <bool SHRINK>
__global__ void __launch_bounds__(KN_THREADS, 1) knn_pass_kernel(const KnnParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar = sbase + KN_BARS;
    if (threadIdx.x == 0) {
        for (int s = 0; s < KN_STAGES; ++s) {
            mbar_init(bar + s * 8, 1);
            mbar_init(bar + (KN_STAGES + s) * 8, KN_CONSUMER_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    const int64_t u0 = (int64_t)blockIdx.x * p.n_units / gridDim.x;
    const int64_t u1 = (int64_t)(blockIdx.x + 1) * p.n_units / gridDim.x;
    // registers move from the producer warpgroup to the consumers (128 accumulators each): 2 x 128 x 232 + 128 x 40 <= 64 K
    if (warp >= KN_CONSUMER_WARPS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp == KN_CONSUMER_WARPS && lane == 0) knn_producer(p, sbase, u0, u1);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        knn_consumer<SHRINK>(p, sbase, u0, u1, warp >> 2);
    }
}

// ---- threshold ------------------------------------------------------------------------------------------------------
// One CTA per row.  Radix select (radix_select, select.cuh) over the keys of the row's group maxima, top 24 bits: the
// result is the lower edge of the bucket holding the k-th largest maximum, so at least k maxima are >= it.
template <bool SHRINK>
__global__ void __launch_bounds__(256) knn_thr_kernel(int64_t nb, int64_t G, int64_t G_valid, int k, int F, const float* __restrict__ gmax,
                                                      const int64_t* __restrict__ rows, int64_t row_off, const float* __restrict__ rnorm,
                                                      const uint32_t* __restrict__ header, float* __restrict__ thr, int32_t* __restrict__ flags,
                                                      const float* __restrict__ norms, float shrink) {
    __shared__ RadixSmem sm;
    const int64_t row = blockIdx.x;
    const int tid = threadIdx.x;
    if (row >= nb) return;
    if ((int64_t)k > G_valid) {                                        // fewer groups than wanted neighbours: exact route
        if (tid == 0) { thr[row] = INFINITY; flags[row] = 1; }
        return;
    }
    const float* g = gmax + row * G;
    unsigned need = (unsigned)k;
    const unsigned prefix = radix_select<3, 256>([=](int64_t i) { return float_key(__ldg(g + i)); }, G_valid, need, sm);
    if (SHRINK && tid == 0) {
        // header words: [0] largest |element|, [1] largest rnorm, [2] largest rnorm[i] / norms[i] (rounded up), [3] 0x7fffffff
        // minus the bits of the smallest norms[i], [5] the largest norms[i]
        const float isc = 1.0f / fp16_scale_for(header[0]);
        const int64_t qrow = rows ? rows[row] : row_off + row;
        const float A = rnorm[qrow], nq = norms[qrow], Bm = __uint_as_float(header[1]);
        const float Rmax = __uint_as_float(header[2]), nmin = __uint_as_float(0x7fffffffu - header[3]);
        const float nmx = __uint_as_float(header[5]);
        // |q||i| / D_i <= Rq R_i (nq ni) / D_i, and nq ni / (nq ni + shrink) grows with ni: at most its value at the largest norm
        const float fac = __fdiv_ru(__fmul_ru(nq, nmx), __fadd_rd(__fmul_rd(nq, nmx), shrink));
        const float RR = __fmul_ru(__fmul_ru(A == 0.f ? 0.f : __fdiv_ru(A, nq), Rmax), fac) * (1.0f + 0x1p-20f);
        const float Dmin = __fmul_rd(__fadd_rd(__fmul_rd(nq, nmin), shrink), 1.0f - 0x1p-22f);
        const float steps = (float)((F + KN_KC - 1) / KN_KC * (KN_KC / 16));
        const float eps = 0x1p-10f + 0x1p-22f + (steps * 0x1p-20f + (float)F * 0x1p-24f) * (1.0f + 0x1p-9f);
        const float sub = (0x1p-25f * sqrtf((float)F) * (A + Bm) * isc + (float)F * 0x1p-50f * isc * isc + 0x1p-120f) / Dmin;
        const float vmax = RR * (1.0f + 2.0f * eps) + sub;
        set_threshold(key_float(prefix), 2.0f * (eps * RR + sub + 0x1p-23f * vmax) * (1.0f + 0x1p-8f), thr + row, flags + row);
    }
    if (!SHRINK && tid == 0) {
        const float sc = fp16_scale_for(header[0]);
        const int64_t qrow = rows ? rows[row] : row_off + row;
        const float un = rnorm[qrow] * sc, mn = __uint_as_float(header[1]) * sc;
        const float steps = (float)((F + KN_KC - 1) / KN_KC * (KN_KC / 16));
        const float eps = 0x1p-10f + 0x1p-22f + (steps * 0x1p-20f + (float)F * 0x1p-24f) * (1.0f + 0x1p-9f);
        const float sub = 0x1p-25f * sqrtf((float)F) * (un + mn) + (float)F * 0x1p-50f + ((float)F * 0x1p-75f * sc) * (0x1p-74f * sc);
        set_threshold(key_float(prefix), 2.0f * (eps * un * mn + sub) * (1.0f + 0x1p-8f), thr + row, flags + row);
    }
}

// ---- finalists ------------------------------------------------------------------------------------------------------
// THE arithmetic of the result: gemm_nt_kernel's per-output chain (fmaf(query_k, item_k, acc), k ascending, from 0.f, one
// extra fmaf(0, 0, acc) when F is not a multiple of its 32-wide K slab).
__device__ __forceinline__ float knn_exact(const float* __restrict__ q, const float* __restrict__ x, int F, bool vec) {
    float acc = 0.f;
    int k = 0;
    if (vec) {
        for (; k + 32 <= F; k += 32) {
            float4 xv[8], qv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) { xv[i] = ldg4(x + k + 4 * i); qv[i] = ldg4(q + k + 4 * i); }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                acc = fmaf(qv[i].x, xv[i].x, acc);
                acc = fmaf(qv[i].y, xv[i].y, acc);
                acc = fmaf(qv[i].z, xv[i].z, acc);
                acc = fmaf(qv[i].w, xv[i].w, acc);
            }
        }
    }
    for (; k < F; ++k) acc = fmaf(__ldg(q + k), __ldg(x + k), acc);
    if (F & 31) acc = fmaf(0.f, 0.f, acc);
    return acc;
}

template <bool SHRINK>
__global__ void __launch_bounds__(KN_FIN_THREADS) knn_final_kernel(int64_t nb, int64_t n, const float* __restrict__ X, int64_t ldx, int F, int k,
                                                                   const int64_t* __restrict__ rows, int64_t row_off, int64_t G_valid,
                                                                   const float* __restrict__ gmax, int64_t G, const float* __restrict__ thr,
                                                                   const int32_t* __restrict__ flags, int32_t* __restrict__ counter,
                                                                   int64_t* __restrict__ fb_rows, int64_t* __restrict__ fb_pos,
                                                                   int64_t* __restrict__ out_idx, float* __restrict__ out_val,
                                                                   const float* __restrict__ norms, float shrink) {
    __shared__ uint64_t comp[KN_CAP];
    __shared__ int32_t glist[KN_CAP / KN_GROUP];
    __shared__ int s_cnt;
    const int64_t row = blockIdx.x;
    const int tid = threadIdx.x;
    if (row >= nb) return;
    const int64_t qrow = rows ? rows[row] : row_off + row;
    auto to_exact = [&]() {
        if (tid == 0) {
            const int slot = atomicAdd(counter, 1);
            fb_rows[slot] = qrow;
            fb_pos[slot] = row;
        }
    };
    if (flags[row]) { to_exact(); return; }
    const float th = thr[row];
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    const float* g = gmax + row * G;
    for (int64_t i = tid; i < G_valid; i += KN_FIN_THREADS)
        if (__ldg(g + i) >= th) {
            const int pos = atomicAdd(&s_cnt, 1);
            if (pos < KN_CAP / KN_GROUP) glist[pos] = (int32_t)i;
        }
    __syncthreads();
    const int cnt = s_cnt;
    if (cnt * KN_GROUP > KN_CAP) { to_exact(); return; }
    const int nc = cnt * KN_GROUP;
    int n2 = 1;
    while (n2 < nc) n2 <<= 1;
    const float* qv = X + qrow * ldx;
    const bool vec = (ldx & 3) == 0 && (F & 3) == 0 && ((((uintptr_t)X) & 15) == 0);
    for (int c = tid; c < n2; c += KN_FIN_THREADS) {
        uint64_t v = 0;                                                // (padding: below every real composite)
        if (c < nc) {
            const int64_t item = (int64_t)glist[c / KN_GROUP] * KN_GROUP + (c % KN_GROUP);
            if (item < n) {
                float s = knn_exact(qv, X + item * ldx, F, vec);
                if constexpr (SHRINK) s = shrink_div(s, __ldg(norms + qrow), __ldg(norms + item), shrink);
                v = ((uint64_t)float_key(s) << 32) | (uint32_t)(~(uint32_t)item);
            }
        }
        comp[c] = v;
    }
    bitonic_desc(comp, n2);
    for (int t = tid; t < k; t += KN_FIN_THREADS) {
        const uint64_t c = comp[t];
        out_idx[row * k + t] = (int64_t)(uint32_t)(~(uint32_t)c);
        out_val[row * k + t] = key_float((uint32_t)(c >> 32));
    }
}

// Shrink route: the exact route's elementwise denominator on a score block (row j = table row src[j], or row0 + j).
__global__ void knn_shrink_rows_kernel(int64_t c, int64_t n, float* __restrict__ S, const int64_t* __restrict__ src, int64_t row0,
                                       const float* __restrict__ norms, float shrink) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= c * n) return;
    const int64_t j = t / n, i = t - j * n;
    S[t] = shrink_div(S[t], __ldg(norms + (src ? __ldg(src + j) : row0 + j)), __ldg(norms + i), shrink);
}

// Shrink route, table summary of the given norms next to the kernel's own (rounded-up) ones: header[2] = the largest
// rnorm[i] / norms[i] rounded up (0 for a zero row; inf / NaN when a norm is 0 or NaN beside a non-zero row), header[3] =
// 0x7fffffff minus the bits of the smallest norms[i], header[4] = 1 if any norms[i] is not finite, header[5] = the largest
// norms[i].
__global__ void knn_shrink_prep_kernel(int64_t n, const float* __restrict__ rnorm, const float* __restrict__ norms, uint32_t* __restrict__ header) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    uint32_t ratio = 0u, nmin = 0u, bad = 0u, nmax = 0u;
    if (i < n) {
        const float r = rnorm[i], ni = norms[i];
        ratio = __float_as_uint(r == 0.f ? 0.f : __fdiv_ru(r, ni)) & 0x7fffffffu;
        nmin = 0x7fffffffu - (__float_as_uint(ni) & 0x7fffffffu);
        bad = !(fabsf(ni) < INFINITY);
        nmax = bad ? 0u : __float_as_uint(ni) & 0x7fffffffu;
    }
    ratio = __reduce_max_sync(0xffffffffu, ratio);
    nmin = __reduce_max_sync(0xffffffffu, nmin);
    bad = __reduce_or_sync(0xffffffffu, bad);
    nmax = __reduce_max_sync(0xffffffffu, nmax);
    if ((threadIdx.x & 31) == 0) {
        if (ratio) atomicMax(header + 2, ratio);
        if (nmin) atomicMax(header + 3, nmin);
        if (bad) atomicOr(header + 4, 1u);
        if (nmax) atomicMax(header + 5, nmax);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
struct KnnPlan {
    int KP;
    int64_t n_it, G, G_valid, rows_blk, rows_pad, s_rows;
    size_t off_hdr, off_xpk, off_rnorm, off_qpk, off_gmax, off_thr, off_flags, off_cnt, off_fbr, off_fbp, off_ex, total;
};

static KnnPlan knn_plan(int64_t n, int F, int64_t m, int k) {
    KnnPlan P;
    P.KP = (F + KN_KC - 1) / KN_KC * KN_KC;
    P.n_it = (n + KN_TILE - 1) / KN_TILE;
    P.G = P.n_it * (KN_TILE / KN_GROUP);
    P.G_valid = (n + KN_GROUP - 1) / KN_GROUP;
    // row block: group maxima of a block below ~512 MB (250 KB per row at 10^6 items)
    int64_t rb = (512ll << 20) / (P.G * 4) / (2 * KN_TILE) * (2 * KN_TILE);
    if (rb < 2 * KN_TILE) rb = 2 * KN_TILE;
    if (rb > 65536) rb = 65536;
    const int64_t m_pad = (m + 2 * KN_TILE - 1) / (2 * KN_TILE) * (2 * KN_TILE);
    P.rows_blk = m_pad < rb ? m_pad : rb;
    P.rows_pad = P.rows_blk;                                          // (a multiple of 256)
    P.s_rows = exact_block_rows(n, m);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes > 0 ? bytes : 1, 1024); return o; };
    P.off_hdr = take(1024);
    P.off_xpk = take((size_t)P.n_it * KN_TILE * P.KP * 2);
    P.off_rnorm = take((size_t)n * 4);
    P.off_qpk = take((size_t)P.rows_pad * P.KP * 2);
    P.off_gmax = take((size_t)P.rows_blk * P.G * 4);
    P.off_thr = take((size_t)P.rows_blk * 4);
    P.off_flags = take((size_t)P.rows_blk * 4);
    P.off_cnt = take(4);
    P.off_fbr = take((size_t)P.rows_blk * 8);
    P.off_fbp = take((size_t)P.rows_blk * 8);
    P.off_ex = take(exact_rows_bytes(P.s_rows, n, k));
    P.total = off + 1024;
    return P;
}

static int64_t g_knn_fallback_rows = -1;

// The existing route for `cnt` query rows (table rows src_rows[j], or j when src_rows is NULL): exact fp32 scores of
// gemm_nt_kernel (+ the shrink division), mmrec_topk_rows_f32, then rows j go to output rows dst_pos[j] (or j).
static int knn_exact_rows(int64_t cnt, const int64_t* src_rows, const int64_t* dst_pos, int64_t n, const float* X, int64_t ldx, int F, int k,
                          const KnnPlan& P, char* base, int64_t* out_idx, float* out_val, cudaStream_t stream, const float* norms, float shrink) {
    return exact_rows_topk(cnt, dst_pos, n, k, P.s_rows, base + P.off_ex, out_idx, out_val, stream, [&](int64_t c0, int64_t c, float* S) {
        GemmNT g;
        g.A = src_rows ? X : X + c0 * ldx; g.lda = ldx; g.a_idx = src_rows ? src_rows + c0 : nullptr; g.M = c;
        g.B = X; g.ldb = ldx; g.N = n; g.K = F; g.bias = nullptr; g.C = S; g.ldc = n; g.l2_normalize = 0;
        int rc = launch_gemm_nt<128, 128, 8, 8>(g, stream);
        if (rc || !norms) return rc;
        knn_shrink_rows_kernel<<<(unsigned)((c * n + 255) / 256), 256, 0, stream>>>(c, n, S, src_rows ? src_rows + c0 : nullptr, c0, norms, shrink);
        MMREC_LAUNCH_CHECK();
        return MMREC_OK;
    });
}

}  // namespace mmrec

using namespace mmrec;

extern "C" size_t mmrec_knn_topk_workspace_bytes(int64_t n, int F, int64_t m, int k) {
    if (n < 1 || F < 1 || m < 0 || k < 1 || k > 1024 || k > n) return 0;
    return knn_plan(n, F, m > 0 ? m : 1, k).total;
}

extern "C" int64_t mmrec_debug_knn_fallback_rows(void) { return g_knn_fallback_rows; }

extern "C" int mmrec_debug_knn_scratch(int64_t n, int F, int64_t m, int k, int64_t* out, int cap) {
    MMREC_CHECK_ARG(out != nullptr || cap <= 0, "debug_knn_scratch: null output");
    if (!mmrec_knn_topk_workspace_bytes(n, F, m, k)) return -1;
    const KnnPlan P = knn_plan(n, F, m > 0 ? m : 1, k);
    const int64_t v[] = {P.rows_blk, P.rows_pad, P.KP, KN_GROUP, P.n_it, P.G, P.G_valid, (int64_t)P.off_hdr, (int64_t)P.off_xpk,
                         (int64_t)P.off_rnorm, (int64_t)P.off_qpk, (int64_t)P.off_gmax, (int64_t)P.off_thr, (int64_t)P.off_flags,
                         (int64_t)P.total};
    const int cnt = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < cnt && i < cap; ++i) out[i] = v[i];
    return cnt;
}

template <bool SHRINK>
static int knn_topk_impl(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k, const float* norms,
                         float shrink, int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, cudaStream_t stream);

extern "C" int mmrec_knn_topk_f32(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k,
                                  int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, void* stream_) {
    return knn_topk_impl<false>(n, X, ldx, F, m, rows, k, nullptr, 0.f, out_idx, out_val, ws, ws_bytes, (cudaStream_t)stream_);
}

extern "C" int mmrec_knn_topk_shrink_f32(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k,
                                         const float* norms, float shrink, int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes,
                                         void* stream_) {
    MMREC_CHECK_ARG(norms != nullptr || m == 0, "knn_topk_shrink: null norms");
    return knn_topk_impl<true>(n, X, ldx, F, m, rows, k, norms, shrink, out_idx, out_val, ws, ws_bytes, (cudaStream_t)stream_);
}

template <bool SHRINK>
static int knn_topk_impl(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k, const float* norms,
                         float shrink, int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, cudaStream_t stream) {
    MMREC_CHECK_ARG(n >= 1 && F >= 1 && m >= 0, "knn_topk: bad sizes (need n >= 1, F >= 1, m >= 0)");
    MMREC_CHECK_ARG(k >= 1 && k <= 1024 && k <= n, "knn_topk: need 1 <= k <= min(1024, n)");
    MMREC_CHECK_ARG(n < (1ll << 31), "knn_topk: n must fit 31 bits");
    MMREC_CHECK_ARG(rows != nullptr || m == n, "knn_topk: rows == NULL means all n rows (m == n)");
    if (m == 0) return MMREC_OK;
    MMREC_CHECK_ARG(X && ldx >= F && out_idx && out_val, "knn_topk: null pointer or ldx < F");
    const KnnPlan P = knn_plan(n, F, m, k);
    char* base = (char*)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
    if (!ws || ws_bytes < P.total + (size_t)(base - (char*)ws)) {
        set_error("knn_topk: workspace %zu < %zu", ws_bytes, P.total + 1024);
        return MMREC_EWORKSPACE;
    }
    if (int rc = set_smem_once<knn_pass_kernel<SHRINK>>((int)KN_SMEM)) return rc;
    uint32_t* header = (uint32_t*)(base + P.off_hdr);
    float* rnorm = (float*)(base + P.off_rnorm);
    const char* Xpk = base + P.off_xpk;
    char* Qpk = base + P.off_qpk;
    float* gmax = (float*)(base + P.off_gmax);
    float* thr = (float*)(base + P.off_thr);
    int32_t* flags = (int32_t*)(base + P.off_flags);
    int32_t* counter = (int32_t*)(base + P.off_cnt);
    int64_t* fb_rows = (int64_t*)(base + P.off_fbr);
    int64_t* fb_pos = (int64_t*)(base + P.off_fbp);
    // 1. norms + largest magnitude; a non-finite element sends the whole call to the exact route.  Header words: [0] largest
    //    |element| bits, [1] largest row norm bits (unscaled, rounded up)
    MMREC_CUDA(cudaMemsetAsync(header, 0, 1024, stream));
    {
        const int64_t blocks = (n + 7) / 8;
        absmax_norm_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, stream>>>(n, X, ldx, F, rnorm, header, header + 1);
        MMREC_LAUNCH_CHECK();
    }
    if (SHRINK) {
        knn_shrink_prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(n, rnorm, norms, header);
        MMREC_LAUNCH_CHECK();
    }
    uint32_t h[5] = {0, 0, 0, 0, 0};
    MMREC_CUDA(cudaMemcpyAsync(h, header, sizeof(h), cudaMemcpyDeviceToHost, stream));
    MMREC_CUDA(cudaStreamSynchronize(stream));
    // shrink route: the certificate needs a finite shrink >= 0, finite norms and, with shrink 0, no zero norm (0 / 0)
    const bool shrink_exact = SHRINK && (!(shrink >= 0.f && shrink < INFINITY) || h[4] || (shrink == 0.f && h[3] == 0x7fffffffu));
    if (h[0] >= 0x7f800000u || shrink_exact) {
        int rc = knn_exact_rows(m, rows, nullptr, n, X, ldx, F, k, P, base, out_idx, out_val, stream, norms, shrink);
        if (rc) return rc;
        g_knn_fallback_rows = m;
        return MMREC_OK;
    }
    // 2. the item operand, once
    {
        const int64_t threads = P.n_it * KN_TILE * (P.KP / 8);
        knn_pack_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(n, nullptr, 0, X, ldx, F, P.KP, header, (uint4*)Xpk, threads);
        MMREC_LAUNCH_CHECK();
    }
    const int sms = sm_count();
    int64_t n_fb = 0;
    for (int64_t r0 = 0; r0 < m; r0 += P.rows_blk) {
        const int64_t nb = (m - r0) < P.rows_blk ? (m - r0) : P.rows_blk;
        const int64_t nb_pad = (nb + 2 * KN_TILE - 1) / (2 * KN_TILE) * (2 * KN_TILE);
        const int64_t* rb = rows ? rows + r0 : nullptr;
        {
            const int64_t threads = nb_pad * (P.KP / 8);
            knn_pack_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(nb, rb, r0, X, ldx, F, P.KP, header, (uint4*)Qpk, threads);
            MMREC_LAUNCH_CHECK();
        }
        MMREC_CUDA(cudaMemsetAsync(counter, 0, 4, stream));
        KnnParams p;
        p.Qpk = Qpk; p.Xpk = Xpk; p.KP = P.KP; p.nc = P.KP / KN_KC;
        p.n_pairs = (int)(nb_pad / (2 * KN_TILE)); p.n_units = p.n_pairs * P.n_it; p.nb = (int)nb; p.n = (int)n;
        p.gmax = gmax; p.G = (int)P.G;
        p.norms = norms; p.shrink = shrink; p.rows = rb; p.row_off = r0; p.header = header;
        const unsigned grid = (unsigned)(p.n_units < sms ? p.n_units : sms);
        knn_pass_kernel<SHRINK><<<grid, KN_THREADS, KN_SMEM, stream>>>(p);
        MMREC_LAUNCH_CHECK();
        knn_thr_kernel<SHRINK><<<(unsigned)nb, 256, 0, stream>>>(nb, P.G, P.G_valid, k, F, gmax, rb, r0, rnorm, header, thr, flags, norms, shrink);
        MMREC_LAUNCH_CHECK();
        knn_final_kernel<SHRINK><<<(unsigned)nb, KN_FIN_THREADS, 0, stream>>>(nb, n, X, ldx, F, k, rb, r0, P.G_valid, gmax, P.G, thr, flags,
                                                                              counter, fb_rows, fb_pos, out_idx + r0 * k, out_val + r0 * k,
                                                                              norms, shrink);
        MMREC_LAUNCH_CHECK();
        const int64_t cnt = read_count(counter, stream);
        if (cnt < 0) return (int)cnt;
        int rc = knn_exact_rows(cnt, fb_rows, fb_pos, n, X, ldx, F, k, P, base, out_idx + r0 * k, out_val + r0 * k, stream, norms, shrink);
        if (rc) return rc;
        n_fb += cnt;
    }
    g_knn_fallback_rows = n_fb;
    return MMREC_OK;
}
