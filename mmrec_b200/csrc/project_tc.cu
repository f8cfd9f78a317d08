// K2 on the tensor cores: Y = gather(table, idx) @ W^T (+ bias, optional row L2-norm) with wgmma (tf32) and the 3xTF32
// split (fp32-level accuracy; the bar for projections is 1e-4 relative, single-pass TF32 misses it).
//
// The feature table is the big operand (115 MB at 7k x 4096) and is read from HBM exactly once, as fp32, so its hi/lo
// split happens IN the kernel:
//   converter warps (8)  two warpgroups.  Coalesced 16-byte loads of the gathered rows (two register rings of PJ_DEPTH
//                        K chunks: one in flight while the other is converted; 384 contiguous bytes per row visit at
//                        N = 64), split each value into tf32 hi (mantissa truncated to 10 bits) + lo (the exact
//                        remainder, which the tensor core truncates), store both into shared memory directly in the
//                        canonical K-major layout of wgmma (8 x 16 B core matrices; K stride padded to 2064 B so the
//                        stores are conflict-free), fence.proxy.async, arrive on the stage's mbarrier.  Once the whole
//                        stage is in (both warpgroups + the weights), each warpgroup issues 12 x wgmma M64 N{64,128,256}
//                        K8 per 32-wide K chunk (hi.hi + lo.hi + hi.lo) for its 64 rows of the tile into registers,
//                        keeps one chunk's group in flight and hands the stage before it back;
//   producer warp        cp.async.bulk of the pre-split, pre-tiled weight slab (hi and lo) of the same K chunk;
//   epilogue             the accumulator registers are written as one fp32 partial per K split.
// Grid = row tiles x K splits <= SM count (one wave); project_reduce_kernel adds the K splits, the bias and applies
// the row normalisation.  Per launch the kernel moves 4 n F (+ weights) bytes for 2 n F d useful flops -> HBM-bound.
#include "tc_common.cuh"

namespace mmrec {

using namespace tc;

constexpr int PJ_M = 128;                 // rows per CTA tile
constexpr int PJ_KC = 32;                 // k per stage
constexpr int PJ_LBO_A = 2064;            // 16 row groups x 128 B + 16 B pad: K-adjacent core matrices land on different banks
constexpr int PJ_A_BYTES = (PJ_KC / 4) * PJ_LBO_A;            // one of hi / lo for one stage = 16512 B
constexpr int PJ_CONV = 256;              // converter threads = the two MMA warpgroups
constexpr int PJ_THREADS = PJ_CONV + 32;  // warps 0..7 converters / MMA, warp 8 weight producer
// chunks of table reads in flight per converter thread (16 KB per SM and chunk).  A block that issues wgmma is sized
// in whole warpgroups (288 -> 384 threads: at most 168 registers per thread), so the ring shrinks as N's accumulators
// grow (N = 256 still spills a few)
template <int N> constexpr int pj_depth() { return N == 64 ? 3 : (N == 128 ? 2 : 1); }

struct ProjParams {
    const float* table; int64_t F; const int64_t* idx; int64_t n_out;
    const float *Whi, *Wlo;               // packed [k chunk][8 kblk][N/8][8][4]
    int N, n_chunks, chunks_per_split, n_splits, stages, vec_ok, n_tiles;
    float* partial;                       // [n_splits][n_tiles * 128][N]
    int64_t rows_padded;
};

struct PjSmem {
    uint32_t a0, b0, bars, total, stage_bytes, b_bytes;
};
__host__ __device__ inline PjSmem pj_smem(int N, int stages) {
    PjSmem L;
    L.b_bytes = (uint32_t)N * PJ_KC * 4;                      // one of hi / lo
    L.stage_bytes = 2 * PJ_A_BYTES + 2 * L.b_bytes;
    L.a0 = 0;
    L.b0 = 2 * PJ_A_BYTES;                                     // inside a stage: A_hi | A_lo | B_hi | B_lo
    L.bars = stages * L.stage_bytes;
    L.total = L.bars + 32 * 8;
    return L;
}
// barriers: a_full[s] = 0..7 (PJ_CONV arrivals) | b_full[s] = 8..15 (tx) | empty[s] = 16..23 (one arrival per converter warp)

template <int N, bool FAST>
__global__ void __launch_bounds__(PJ_THREADS, 1) project_tc_kernel(const ProjParams p) {
    constexpr int PJ_DEPTH = pj_depth<N>();
    extern __shared__ __align__(1024) uint8_t smem[];
    const PjSmem L = pj_smem(N, p.stages);
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar = sbase + L.bars;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < 8; ++s) { mbar_init(bar + s * 8, PJ_CONV); mbar_init(bar + (8 + s) * 8, 1); mbar_init(bar + (16 + s) * 8, PJ_CONV / 32); }
        mbar_fence_init();
    }
    __syncthreads();

    const int tile = blockIdx.x / p.n_splits, sp = blockIdx.x % p.n_splits;
    const int c0 = sp * p.chunks_per_split;
    const int c1 = min(p.n_chunks, c0 + p.chunks_per_split);
    const int n_my = c1 - c0;
    // K rotation: CTA `tile` starts its K loop at a different chunk.  With a power-of-two row pitch (F = 4096: 16 KB) all
    // CTAs would otherwise read the same few-hundred-byte window of every row at the same time -- the same address bits,
    // hence the same few HBM channels.  Spreading the windows over the row restores the channel interleave; the
    // accumulation order differs per row tile but not run to run.
    const int rot = n_my > 0 ? ((int)(((int64_t)tile * n_my) / p.n_tiles) / PJ_DEPTH * PJ_DEPTH) % n_my : 0;

    if (warp == PJ_CONV / 32) {
        if (lane == 0) {
            int s = 0;
            uint32_t par = 1;
            for (int c = 0; c < n_my; ++c) {
                mbar_wait(bar + (16 + s) * 8, par);
                mbar_expect_tx(bar + (8 + s) * 8, 2 * L.b_bytes);
                const int64_t off = (int64_t)(c0 + (c + rot) % n_my) * (L.b_bytes / 4);
                bulk_g2s(sbase + s * L.stage_bytes + L.b0, p.Whi + off, L.b_bytes, bar + (8 + s) * 8);
                bulk_g2s(sbase + s * L.stage_bytes + L.b0 + L.b_bytes, p.Wlo + off, L.b_bytes, bar + (8 + s) * 8);
                if (++s == p.stages) { s = 0; par ^= 1; }
            }
        }
        return;
    }
    // ---------------- converters: thread t owns kblk t % 8 of rows t / 8 + 32 i, i = 0..3; PJ_DEPTH chunks of its
    // 16-byte reads are in flight at any time (registers are the staging buffer)
    const int t = threadIdx.x;
    const int g = t >> 7;                                             // warpgroup: MMA rows [64 g, 64 g + 64) of the tile
    const int kb = t & 7;
    const float* rowp[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t r = (int64_t)tile * PJ_M + (t >> 3) + 32 * i;
        rowp[i] = r < p.n_out ? p.table + (p.idx ? p.idx[r] : r) * p.F : nullptr;
    }
    // FAST (16-byte aligned table, F a multiple of 32: every BASELINE shape): the loop is bound by the instruction stream
    // of the 8 converter warps, so the chunk rotation is a running counter instead of a modulo, and a load is one
    // predicated 16-byte request per row.
    int ld_c = rot;                                               // chunk (inside this split) the next load reads
    const float* kp[4];                                           // FAST: row pointers advanced to this thread's k block
#pragma unroll
    for (int i = 0; i < 4; ++i) kp[i] = rowp[i] ? rowp[i] + (int64_t)c0 * PJ_KC + kb * 4 : nullptr;
    auto load_chunk = [&](int c, float4 (&x)[4]) {
        if (FAST) {
            const bool on = c < n_my;                             // (warp-uniform)
#pragma unroll
            for (int i = 0; i < 4; ++i)
                x[i] = (on && kp[i]) ? __ldg(reinterpret_cast<const float4*>(kp[i] + ld_c * PJ_KC)) : make_float4(0.f, 0.f, 0.f, 0.f);
            if (on && ++ld_c == n_my) ld_c = 0;
            return;
        }
        const int64_t k = (int64_t)(c0 + (c + rot) % n_my) * PJ_KC + kb * 4;    // (c >= n_my: not loaded, see below)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rowp[i] && c < n_my) {
                if (p.vec_ok && k + 3 < p.F) v = __ldg(reinterpret_cast<const float4*>(rowp[i] + k));
                else {
                    if (k + 0 < p.F) v.x = __ldg(rowp[i] + k + 0);
                    if (k + 1 < p.F) v.y = __ldg(rowp[i] + k + 1);
                    if (k + 2 < p.F) v.z = __ldg(rowp[i] + k + 2);
                    if (k + 3 < p.F) v.w = __ldg(rowp[i] + k + 3);
                }
            }
            x[i] = v;
        }
    };
    // MMA side: descriptors built once, per instruction only the address field (16-byte units) moves
    const uint32_t LBO_B = (uint32_t)(N / 8) * 128;
    const uint64_t a_hi0 = smem_desc(sbase + L.a0 + g * 1024, PJ_LBO_A, 128), a_lo0 = smem_desc(sbase + L.a0 + PJ_A_BYTES + g * 1024, PJ_LBO_A, 128);
    const uint64_t b_hi0 = smem_desc(sbase + L.b0, LBO_B, 128), b_lo0 = smem_desc(sbase + L.b0 + L.b_bytes, LBO_B, 128);
    const uint64_t ka = (2 * PJ_LBO_A) >> 4, kbs = (2 * LBO_B) >> 4;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    uint32_t first = 0;
    int prev = 0;
    // Two register rings of PJ_DEPTH chunks each: while one is converted the other is in flight.  A ring is (re)filled
    // in one burst, so a row is visited once per PJ_DEPTH chunks for PJ_DEPTH x 128 contiguous bytes -- with a
    // power-of-two row pitch (F = 4096: 16 KB) the 128 rows of a tile sit in the same HBM bank, every visit is a row
    // activate, and short visits serialise on the bank.
    float4 ringA[PJ_DEPTH][4], ringB[PJ_DEPTH][4];
    int s = 0;                                                    // smem stage of the next chunk, and its "empty" parity
    uint32_t par = 1;
    int done = 0;                                                 // chunks issued to the tensor cores
    auto fill = [&](int cbase, float4 (&ring)[PJ_DEPTH][4]) {
#pragma unroll
        for (int q = 0; q < PJ_DEPTH; ++q) load_chunk(cbase + q, ring[q]);
    };
    auto drain = [&](int cbase, float4 (&ring)[PJ_DEPTH][4]) {
#pragma unroll
        for (int q = 0; q < PJ_DEPTH; ++q) {
            if (cbase + q < n_my) {
                mbar_wait(bar + (16 + s) * 8, par);
                uint8_t* st = smem + s * L.stage_bytes;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = (t >> 3) + 32 * i;
                    const uint32_t off = kb * PJ_LBO_A + (r >> 3) * 128 + (r & 7) * 16;
                    float4 h, l;
                    split_tf32_trunc(ring[q][i].x, h.x, l.x); split_tf32_trunc(ring[q][i].y, h.y, l.y);
                    split_tf32_trunc(ring[q][i].z, h.z, l.z); split_tf32_trunc(ring[q][i].w, h.w, l.w);
                    *reinterpret_cast<float4*>(st + L.a0 + off) = h;
                    *reinterpret_cast<float4*>(st + L.a0 + PJ_A_BYTES + off) = l;
                }
                fence_proxy_async();                              // generic-proxy stores -> visible to the MMA's async reads
                mbar_arrive(bar + s * 8);
                // the whole stage (both warpgroups' rows, the weight slab) -> this warpgroup's 64 rows
                mbar_wait(bar + s * 8, par ^ 1);
                mbar_wait(bar + (8 + s) * 8, par ^ 1);
                const uint64_t st_off = (uint64_t)(s * L.stage_bytes) >> 4;
                uint64_t a_hi = a_hi0 + st_off, a_lo = a_lo0 + st_off, b_hi = b_hi0 + st_off, b_lo = b_lo0 + st_off;
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < PJ_KC / 8; ++j) {
                    wgmma_tf32<N>(acc, a_hi, b_hi, first);
                    first = 1;
                    wgmma_tf32<N>(acc, a_lo, b_hi, 1);
                    wgmma_tf32<N>(acc, a_hi, b_lo, 1);
                    a_hi += ka; a_lo += ka; b_hi += kbs; b_lo += kbs;
                }
                wgmma_commit();
                if (done++ > 0) {                                 // the previous chunk's group is done -> its stage goes back
                    wgmma_wait<1>();
                    warp_arrive(bar + (16 + prev) * 8);
                }
                prev = s;
                if (++s == p.stages) { s = 0; par ^= 1; }
            }
        }
    };
    fill(0, ringA);
    for (int cb = 0; cb < n_my; cb += 2 * PJ_DEPTH) {
        fill(cb + PJ_DEPTH, ringB);
        drain(cb, ringA);
        fill(cb + 2 * PJ_DEPTH, ringA);
        drain(cb + PJ_DEPTH, ringB);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    // ---------------- epilogue: partial tile of this K split, straight from the accumulator registers
    const int w = (t >> 5) & 3;
    const int64_t row0 = (int64_t)tile * PJ_M + g * 64 + w * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* dst = p.partial + ((int64_t)sp * p.rows_padded + row0 + 8 * h) * N + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
            *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
}

// Y[r, :] = sum over K splits of partial[s, r, :d] + bias, optional row L2 normalisation.  One warp per row.
__global__ void __launch_bounds__(256) project_reduce_kernel(int64_t n_out, int d, int N, int n_splits, int64_t rows_padded,
                                                             const float* __restrict__ partial, const float* __restrict__ bias,
                                                             int l2, float* __restrict__ Y, int64_t ldy) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_out) return;
    float acc[8];                                                      // d <= 256
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = lane + 32 * i;
        float a = 0.f;
        if (c < d) {
            for (int s = 0; s < n_splits; ++s) a += partial[((int64_t)s * rows_padded + row) * N + c];
            if (bias) a += __ldg(bias + c);
            ss += a * a;
        }
        acc[i] = a;
    }
    float inv = 1.f;
    if (l2) { ss = warp_sum(ss); inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f); }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = lane + 32 * i;
        if (c < d) Y[row * ldy + c] = l2 ? acc[i] * inv : acc[i];
    }
}

struct PjPlan {
    int N, KP, n_chunks, n_splits, chunks_per_split, stages;
    int64_t n_tiles, rows_padded;
    size_t off_whi, off_wlo, off_partial, total;
};

static bool pj_plan(int64_t n_out, int64_t F, int d, PjPlan& P) {
    if (d > 256 || n_out <= 0 || F < 1) return false;
    P.N = d <= 64 ? 64 : (d <= 128 ? 128 : 256);
    P.KP = (int)((F + PJ_KC - 1) / PJ_KC * PJ_KC);
    P.n_chunks = P.KP / PJ_KC;
    P.n_tiles = (n_out + PJ_M - 1) / PJ_M;
    P.rows_padded = P.n_tiles * PJ_M;
    const int sms = sm_count();
    int splits = (int)(sms / P.n_tiles);
    if (splits < 1) splits = 1;
    if (splits > P.n_chunks / 4) splits = P.n_chunks / 4 > 0 ? P.n_chunks / 4 : 1;     // at least 4 chunks per CTA
    if (splits > 32) splits = 32;
    P.chunks_per_split = (P.n_chunks + splits - 1) / splits;
    P.n_splits = (P.n_chunks + P.chunks_per_split - 1) / P.chunks_per_split;
    const uint32_t stage = 2 * PJ_A_BYTES + 2 * (uint32_t)P.N * PJ_KC * 4;
    P.stages = (int)((220 * 1024) / stage);
    if (P.stages > 8) P.stages = 8;
    if (P.stages < 2) return false;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes, 1024); return o; };
    P.off_whi = take((size_t)P.N * P.KP * 4);
    P.off_wlo = take((size_t)P.N * P.KP * 4);
    P.off_partial = take((size_t)P.n_splits * P.rows_padded * P.N * 4);
    P.total = off + 1024;
    return true;
}

size_t project_tc_workspace_bytes(int64_t n_out, int64_t F, int d) {
    PjPlan P;
    return pj_plan(n_out, F, d, P) ? P.total : 0;
}

template <int R>
static int pack_weights(const float* W, int64_t F, int d, int KP, float* hi, float* lo, cudaStream_t stream) {
    const int64_t total = (int64_t)R * (KP / 4);
    pack_split_kernel<R><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d, nullptr, W, F, (int)F, KP, hi, lo, 1);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

// 1 = done, 0 = shape not supported by this path (caller uses the fp32 CUDA-core kernel), < 0 error
int project_tc(int64_t n_out, const int64_t* idx, const float* table, int64_t F, const float* W, const float* bias, int d,
               int l2_normalize, float* Y, int64_t ldy, void* ws, size_t ws_bytes, cudaStream_t stream) {
    PjPlan P;
    if (!ws || !pj_plan(n_out, F, d, P) || ws_bytes < P.total || F >= (1ll << 31)) return 0;
    char* base = (char*)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
    float *Whi = (float*)(base + P.off_whi), *Wlo = (float*)(base + P.off_wlo), *partial = (float*)(base + P.off_partial);
    int rc = P.N == 64 ? pack_weights<64>(W, F, d, P.KP, Whi, Wlo, stream)
                       : (P.N == 128 ? pack_weights<128>(W, F, d, P.KP, Whi, Wlo, stream) : pack_weights<256>(W, F, d, P.KP, Whi, Wlo, stream));
    if (rc) return rc;
    ProjParams p;
    p.table = table; p.F = F; p.idx = idx; p.n_out = n_out; p.Whi = Whi; p.Wlo = Wlo; p.N = P.N; p.n_chunks = P.n_chunks;
    p.chunks_per_split = P.chunks_per_split; p.n_splits = P.n_splits; p.stages = P.stages;
    p.n_tiles = (int)P.n_tiles;
    p.vec_ok = ((F & 3) == 0) && ((((uintptr_t)table) & 15) == 0);
    p.partial = partial; p.rows_padded = P.rows_padded;
    const PjSmem L = pj_smem(P.N, P.stages);
    {   // the opt-in is per device
        static bool attr_set[64] = {false};
        int dev = 0;
        MMREC_CUDA(cudaGetDevice(&dev));
        if (dev < 0 || dev >= 64 || !attr_set[dev]) {
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<256, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            MMREC_CUDA(cudaFuncSetAttribute(project_tc_kernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            if (dev >= 0 && dev < 64) attr_set[dev] = true;
        }
    }
    const bool fast = p.vec_ok && (F % PJ_KC) == 0;
    const unsigned grid = (unsigned)(P.n_tiles * P.n_splits);
    if (P.N == 64) {
        if (fast) project_tc_kernel<64, true><<<grid, PJ_THREADS, L.total, stream>>>(p);
        else project_tc_kernel<64, false><<<grid, PJ_THREADS, L.total, stream>>>(p);
    } else if (P.N == 128) {
        if (fast) project_tc_kernel<128, true><<<grid, PJ_THREADS, L.total, stream>>>(p);
        else project_tc_kernel<128, false><<<grid, PJ_THREADS, L.total, stream>>>(p);
    } else {
        if (fast) project_tc_kernel<256, true><<<grid, PJ_THREADS, L.total, stream>>>(p);
        else project_tc_kernel<256, false><<<grid, PJ_THREADS, L.total, stream>>>(p);
    }
    MMREC_LAUNCH_CHECK();
    project_reduce_kernel<<<(unsigned)((n_out + 7) / 8), 256, 0, stream>>>(n_out, d, P.N, P.n_splits, P.rows_padded, partial, bias,
                                                                         l2_normalize, Y, ldy);
    MMREC_LAUNCH_CHECK();
    return 1;
}

}  // namespace mmrec
