// K8: full-table exp-sum of LGMRec's hypergraph contrastive loss (src/models/lgmrec.py:159-166) and its backward,
// on the tensor cores, without the [B, M] score matrix.
//
//     ttl[b] = sum_j exp(<q_b, t_j> * inv_tau)                        (forward, e_bj = exp(<q_b, t_j> * inv_tau))
//     dQ[b]  = g_b * inv_tau * sum_j e_bj t_j                         (backward, g = upstream gradient of ttl)
//     dT[j]  = inv_tau * sum_b g_b e_bj q_b
//
// One kernel serves all three: a CTA (one warpgroup) holds a 64-row X tile and streams 64-row Y tiles of one chunk of
// the other table.  Per Y tile, S = X Y^T (64 x 64) is one run of wgmma m64n64k8 in 3xTF32 (x = x_hi + x_lo, products
// hi.hi + lo.hi + hi.lo, as score_tc.cu); e = exp(S * inv_tau) is formed in the accumulator registers.
//   forward   (X = Q, Y = T): e is added into two per-thread row sums (CUDA-core fp32, round to nearest).
//   backward  (X = Q, Y = T for dQ; X = T, Y = Q with weights w_y = g_y for dT): P = e * w_y is split into tf32 hi / lo
//             and written to shared memory as the A operand of a second 3xTF32 wgmma, P Y (64 x d, K = 64), whose
//             accumulator is started fresh per tile and added to a CUDA-core running sum.  [B, M] is never stored
//             (the flash-attention recompute), the workspace is O((B + M) d).
// No maximum is subtracted (the reference does not): a term or a sum overflows to inf where fp32 exp / add does.
// Determinism: every output is a fixed sequence of fp32 operations.  Chunks of Y tiles write partials to the workspace
// and a second kernel adds them in chunk order; no atomics.  The chunking depends on B and M only, not on the device.
//
// Error bound against exact arithmetic (u = 2^-24; tf32 keeps 10 fraction bits, cvt.rna rounds to nearest):
//   split      x_hi = rna(x): |x - x_hi| <= 2^-11 |x|;  x_lo = rna(x - x_hi): |x - x_hi - x_lo| <= 2^-22 |x|.
//   products   tf32 x tf32 is exact in fp32.  Dropped: x_lo.y_lo (<= 2^-22 |x||y| elementwise) and the two lo roundings
//              (<= 2 * 2^-22): the represented sum differs from <x, y> by <= 3 * 2^-22 |x||y| (Cauchy-Schwarz over k).
//   accumulate 3 d / 8 wgmma steps add into one fp32 accumulator, each adds a K = 8 partial (a tree of depth 3).  Allowing
//              the tensor core's adder to truncate (error < 2u relative per addition, an assumption about the hardware,
//              as in knn_cf.cu), every partial sum is bounded by sum_k |x_k y_k| (1 + 2^-10) <= |x||y| (1 + 2^-10):
//              |S - <x, y>| <= delta = ((3 d / 8 + 3) 2u + 3 * 2^-22) |x||y|
//              (d = 64: 3.9e-6 |x||y|; d = 32: 2.5e-6; d = 128: 6.8e-6).
//   exp        S * inv_tau adds u relative, expf <= 2 ulp:  |e~ - e| <= e * eps_e,  eps_e = delta * inv_tau + 2^-21
//              (unit rows, tau = 0.2: 1.3e-5 at d = 32, 2.0e-5 at d = 64, 3.5e-5 at d = 128).
//   ttl        all terms are positive: relative error <= eps_e + n_add * u, n_add = the additions on the path of one output:
//              16 per Y tile of its chunk, 2 quad shuffles, one per chunk in the reduce (chunking: es_plan below).
//   dQ, dT     per output element, relative to the magnitude sum_j |g_j| e_j |y_jc| (times |g_b| inv_tau for dQ):
//              eps_e (e) + 3 * 2^-22 (split of P and Y) + 27 * 2u (per-tile accumulator, K = 64) + n_add * u (running sum
//              over the tiles of a chunk and the chunk reduce), + u for the final scaling.
// A non-finite P (overflowed e) splits into a NaN lo part: the backward of an overflowed term is NaN, torch's is inf/NaN.
#include "tc_common.cuh"

namespace mmrec {

using namespace tc;

constexpr int ES_T = 64;            // rows of an X tile and of a Y tile
constexpr int ES_THREADS = 128;     // one warpgroup
constexpr int ES_TARGET_CTAS = 256; // X tiles x chunks aimed for (about two waves of 132 SMs)
constexpr int ES_MAX_CHUNKS = 32;

template <int KP, bool BWD>
struct EsSmem {                                 // offsets in floats
    static constexpr int tile = ES_T * KP;
    static constexpr int xh = 0, xl = tile, yh = 2 * tile, yl = 3 * tile;
    static constexpr int yth = 4 * tile, ytl = 5 * tile, ph = 6 * tile, pl = 6 * tile + ES_T * ES_T;   // backward only
    static constexpr int floats = BWD ? 6 * tile + 2 * ES_T * ES_T : 4 * tile;
    static constexpr int bytes = floats * 4;
};

// canonical K-major no-swizzle wgmma layout of an R-row operand: [k / 4][r / 8][r % 8][k % 4]
__device__ __forceinline__ int canon(int r, int k, int R) { return ((k >> 2) * (R >> 3) + (r >> 3)) * 32 + (r & 7) * 4 + (k & 3); }

// rows [r0, r0 + 64) of src (zeros past n) -> tf32 hi / lo in shared memory; TRANS also stores the transpose (KP rows, K = 64)
template <int KP, bool TRANS>
__device__ __forceinline__ void es_load_tile(const float* __restrict__ src, int64_t ld, int64_t r0, int64_t n, bool vec, float* sh,
                                             float* sl, float* sth, float* stl) {
    constexpr int Q4 = KP / 4;
    for (int i = threadIdx.x; i < ES_T * Q4; i += ES_THREADS) {
        const int r = i / Q4, kb = i % Q4;
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (r0 + r < n) {
            const float* s = src + (r0 + r) * ld + kb * 4;
            if (vec) {
                const float4 v = ldg4(s);
                x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = __ldg(s + e);
            }
        }
        float h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) split_tf32(x[e], h[e], l[e]);
        *reinterpret_cast<float4*>(sh + canon(r, kb * 4, ES_T)) = make_float4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<float4*>(sl + canon(r, kb * 4, ES_T)) = make_float4(l[0], l[1], l[2], l[3]);
        if (TRANS) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                sth[canon(kb * 4 + e, r, KP)] = h[e];
                stl[canon(kb * 4 + e, r, KP)] = l[e];
            }
        }
    }
}

struct EsParams {
    const float* X;
    int64_t ldx, nX;
    const float* Y;
    int64_t ldy, nY;
    const float* wy;        // backward: weight of each Y row (g for dT), or null (1)
    const float* gx;        // backward: per-X factor of the direct write (g for dQ), or null (1)
    float inv_tau;
    int tiles_per_chunk, n_chunks;
    int64_t x_pad;          // rows of one partial slab
    float* part;            // forward: [n_chunks][x_pad]; backward: [n_chunks][x_pad][KP], or null: write `out` directly
    float* out;
    int64_t ldo;
};

template <int KP, bool BWD>
__global__ void __launch_bounds__(ES_THREADS) expsum_kernel(const EsParams p) {
    extern __shared__ __align__(1024) float sm[];
    using L = EsSmem<KP, BWD>;
    const int xt = blockIdx.x / p.n_chunks, ch = blockIdx.x % p.n_chunks;
    const int64_t x0 = (int64_t)xt * ES_T;
    const int64_t y_tiles = (p.nY + ES_T - 1) / ES_T;
    const int64_t yt0 = (int64_t)ch * p.tiles_per_chunk;
    const int64_t yt1 = min(y_tiles, yt0 + p.tiles_per_chunk);
    const bool vx = (p.ldx & 3) == 0 && ((uintptr_t)p.X & 15) == 0;
    const bool vy = (p.ldy & 3) == 0 && ((uintptr_t)p.Y & 15) == 0;
    const int t = threadIdx.x, w = t >> 5, lane = t & 31;
    es_load_tile<KP, false>(p.X, p.ldx, x0, p.nX, vx, sm + L::xh, sm + L::xl, nullptr, nullptr);

    constexpr uint32_t LBO64 = (ES_T / 8) * 128, LBOT = (KP / 8) * 128;
    const uint32_t sb = smem_u32(sm);
    const uint64_t dxh = smem_desc(sb + 4 * L::xh, LBO64, 128), dxl = smem_desc(sb + 4 * L::xl, LBO64, 128);
    const uint64_t dyh = smem_desc(sb + 4 * L::yh, LBO64, 128), dyl = smem_desc(sb + 4 * L::yl, LBO64, 128);
    const uint64_t k64 = (2 * LBO64) >> 4, kT = (2 * LBOT) >> 4;

    float rs[2] = {0.f, 0.f};
    float run[BWD ? KP / 2 : 1];
#pragma unroll
    for (int i = 0; i < (BWD ? KP / 2 : 1); ++i) run[i] = 0.f;

    for (int64_t yt = yt0; yt < yt1; ++yt) {
        const int64_t y0 = yt * ES_T;
        __syncthreads();                                       // the previous tile's wgmmas are complete in every warp
        es_load_tile<KP, BWD>(p.Y, p.ldy, y0, p.nY, vy, sm + L::yh, sm + L::yl, sm + L::yth, sm + L::ytl);
        fence_proxy_async();
        __syncthreads();
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        wgmma_fence();
        {
            uint64_t ah = dxh, al = dxl, bh = dyh, bl = dyl;
#pragma unroll
            for (int k = 0; k < KP / 8; ++k) {
                wgmma_tf32<64>(s, ah, bh, k > 0 ? 1u : 0u);
                wgmma_tf32<64>(s, al, bh, 1u);
                wgmma_tf32<64>(s, ah, bl, 1u);
                ah += k64; al += k64; bh += k64; bl += k64;
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        // fragment: s[4 j + e] is row 16 w + lane / 4 + 8 (e / 2), column 8 j + 2 (lane % 4) + e % 2
        if constexpr (!BWD) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (y0 + 8 * j + 2 * (lane & 3) + (e & 1) < p.nY) rs[e >> 1] += expf(s[4 * j + e] * p.inv_tau);
        } else {
            float* ph = sm + L::ph;
            float* pl = sm + L::pl;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = 8 * j + 2 * (lane & 3) + (e & 1), r = 16 * w + (lane >> 2) + 8 * (e >> 1);
                    const int64_t y = y0 + col;
                    float v = 0.f;
                    if (y < p.nY) {
                        v = expf(s[4 * j + e] * p.inv_tau);
                        if (p.wy) v *= __ldg(p.wy + y);
                    }
                    float h, l;
                    split_tf32(v, h, l);
                    ph[canon(r, col, ES_T)] = h;
                    pl[canon(r, col, ES_T)] = l;
                }
            fence_proxy_async();
            __syncthreads();
            float o[KP / 2];
#pragma unroll
            for (int i = 0; i < KP / 2; ++i) o[i] = 0.f;
            wgmma_fence();
            {
                uint64_t ah = smem_desc(sb + 4 * L::ph, LBO64, 128), al = smem_desc(sb + 4 * L::pl, LBO64, 128);
                uint64_t bh = smem_desc(sb + 4 * L::yth, LBOT, 128), bl = smem_desc(sb + 4 * L::ytl, LBOT, 128);
#pragma unroll
                for (int k = 0; k < ES_T / 8; ++k) {
                    wgmma_tf32<KP>(o, ah, bh, k > 0 ? 1u : 0u);
                    wgmma_tf32<KP>(o, al, bh, 1u);
                    wgmma_tf32<KP>(o, ah, bl, 1u);
                    ah += k64; al += k64; bh += kT; bl += kT;
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(o);
#pragma unroll
            for (int i = 0; i < KP / 2; ++i) run[i] += o[i];
        }
    }

    const int64_t xr = x0 + 16 * w + (lane >> 2);
    if constexpr (!BWD) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float v = rs[h];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            if ((lane & 3) == 0 && xr + 8 * h < p.nX) p.part[ch * p.x_pad + xr + 8 * h] = v;
        }
    } else {
#pragma unroll
        for (int j = 0; j < KP / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t row = xr + 8 * (e >> 1);
                const int c = 8 * j + 2 * (lane & 3) + (e & 1);
                if (row >= p.nX) continue;
                if (p.part) p.part[((int64_t)ch * p.x_pad + row) * KP + c] = run[4 * j + e];
                else p.out[row * p.ldo + c] = run[4 * j + e] * (p.inv_tau * (p.gx ? __ldg(p.gx + row) : 1.f));
            }
    }
}

// ttl[i] = sum over chunks (in chunk order) of part[c][i]; no chunks: 0
__global__ void expsum_reduce_rows_kernel(int64_t n, int chunks, int64_t x_pad, const float* __restrict__ part, float* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[c * x_pad + i];
    out[i] = s;
}

// out[r][c] = (inv_tau * gx[r]) * sum over chunks of part[ch][r][c]; no chunks: 0
__global__ void expsum_reduce_vec_kernel(int64_t n, int d, int chunks, int64_t x_pad, const float* __restrict__ part,
                                         const float* __restrict__ gx, float inv_tau, float* __restrict__ out, int64_t ldo) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * d) return;
    const int64_t r = i / d;
    const int c = (int)(i % d);
    float s = 0.f;
    for (int ch = 0; ch < chunks; ++ch) s += part[(ch * x_pad + r) * d + c];
    out[r * ldo + c] = s * (inv_tau * (gx ? gx[r] : 1.f));
}

static inline int64_t es_tiles(int64_t n) { return (n + ES_T - 1) / ES_T; }

struct EsPlan {
    int chunks, tiles_per_chunk;
};
// Y tiles split into chunks so that X tiles x chunks reaches ES_TARGET_CTAS; depends on the sizes only
static EsPlan es_plan(int64_t nX, int64_t nY) {
    EsPlan P{0, 0};
    const int64_t xt = es_tiles(nX), yt = es_tiles(nY);
    if (xt == 0 || yt == 0) return P;
    int64_t c = (ES_TARGET_CTAS + xt - 1) / xt;
    c = c < ES_MAX_CHUNKS ? c : ES_MAX_CHUNKS;
    c = c < yt ? c : yt;
    const int64_t tpc = (yt + c - 1) / c;
    P.tiles_per_chunk = (int)tpc;
    P.chunks = (int)((yt + tpc - 1) / tpc);
    return P;
}

static size_t es_fwd_bytes(int64_t B, int64_t M) { return align_up((size_t)es_plan(B, M).chunks * es_tiles(B) * ES_T * 4, 256); }
// partials of one backward output (X rows, Y rows): none when one chunk writes the output directly
static size_t es_bwd_part_bytes(int64_t nX, int64_t nY, int d) {
    const EsPlan P = es_plan(nX, nY);
    return P.chunks > 1 ? align_up((size_t)P.chunks * es_tiles(nX) * ES_T * d * 4, 256) : 0;
}

template <int KP, bool BWD>
static int es_launch(const EsParams& p, cudaStream_t st) {
    constexpr int bytes = EsSmem<KP, BWD>::bytes;
    MMREC_CUDA(cudaFuncSetAttribute(expsum_kernel<KP, BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    expsum_kernel<KP, BWD><<<(unsigned)(es_tiles(p.nX) * p.n_chunks), ES_THREADS, bytes, st>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

template <bool BWD>
static int es_dispatch(int d, const EsParams& p, cudaStream_t st) {
    if (d == 32) return es_launch<32, BWD>(p, st);
    if (d == 64) return es_launch<64, BWD>(p, st);
    return es_launch<128, BWD>(p, st);
}

// one backward output: out[x] = inv_tau * gx[x] * sum_y w_y exp(<x, y> inv_tau) y
static int es_bwd_one(const float* X, int64_t ldx, int64_t nX, const float* Y, int64_t ldy, int64_t nY, int d, float inv_tau,
                      const float* wy, const float* gx, float* out, int64_t ldo, float* part, cudaStream_t st) {
    if (nX == 0) return MMREC_OK;
    const EsPlan P = es_plan(nX, nY);
    if (P.chunks == 1) {
        EsParams p{X, ldx, nX, Y, ldy, nY, wy, gx, inv_tau, P.tiles_per_chunk, 1, es_tiles(nX) * ES_T, nullptr, out, ldo};
        return es_dispatch<true>(d, p, st);
    }
    if (P.chunks > 1) {
        EsParams p{X, ldx, nX, Y, ldy, nY, wy, gx, inv_tau, P.tiles_per_chunk, P.chunks, es_tiles(nX) * ES_T, part, out, ldo};
        const int rc = es_dispatch<true>(d, p, st);
        if (rc != MMREC_OK) return rc;
    }
    const int64_t n = nX * d;                                  // chunks == 0 (nY == 0): zeros
    expsum_reduce_vec_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(nX, d, P.chunks, es_tiles(nX) * ES_T, part, gx, inv_tau,
                                                                          out, ldo);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

}  // namespace mmrec

using namespace mmrec;

static inline bool es_d_ok(int d) { return d == 32 || d == 64 || d == 128; }

extern "C" size_t mmrec_expsum_rows_workspace_bytes(int64_t B, int64_t M, int d) {
    if (!es_d_ok(d) || B < 0 || M < 0) return 0;
    const size_t fwd = es_fwd_bytes(B, M);
    const size_t bwd = es_bwd_part_bytes(B, M, d) + es_bwd_part_bytes(M, B, d);
    const size_t need = fwd > bwd ? fwd : bwd;
    return need ? need + 256 : 0;
}

extern "C" int mmrec_expsum_rows_f32(int64_t B, const float* Q, int64_t ldq, int64_t M, const float* T, int64_t ldt, int d, float inv_tau,
                                     float* ttl, void* ws, size_t ws_bytes, void* stream) {
    MMREC_CHECK_ARG(es_d_ok(d), "expsum_rows: d must be 32, 64 or 128 (got %d)", d);
    MMREC_CHECK_ARG(B >= 0 && M >= 0, "expsum_rows: negative size (B %lld, M %lld)", (long long)B, (long long)M);
    MMREC_CHECK_ARG((B == 0 || (Q && ttl && ldq >= d)) && (M == 0 || (T && ldt >= d)),
                    "expsum_rows: null pointer or leading dimension below d");
    if (B == 0) return MMREC_OK;
    const size_t need = mmrec_expsum_rows_workspace_bytes(B, M, d);
    MMREC_CHECK_ARG(need == 0 || ws, "expsum_rows: null workspace");
    if (ws_bytes < need) {
        set_error("expsum_rows: workspace %zu bytes < %zu", ws_bytes, need);
        return MMREC_EWORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    float* part = (float*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    const EsPlan P = es_plan(B, M);
    const int64_t x_pad = es_tiles(B) * ES_T;
    if (P.chunks > 0) {
        EsParams p{Q, ldq, B, T, ldt, M, nullptr, nullptr, inv_tau, P.tiles_per_chunk, P.chunks, x_pad, part, nullptr, 0};
        const int rc = es_dispatch<false>(d, p, st);
        if (rc != MMREC_OK) return rc;
    }
    expsum_reduce_rows_kernel<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(B, P.chunks, x_pad, part, ttl);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_expsum_rows_bwd_f32(int64_t B, const float* Q, int64_t ldq, int64_t M, const float* T, int64_t ldt, int d,
                                         float inv_tau, const float* g, float* dQ, int64_t lddq, float* dT, int64_t lddt, void* ws,
                                         size_t ws_bytes, void* stream) {
    MMREC_CHECK_ARG(es_d_ok(d), "expsum_rows_bwd: d must be 32, 64 or 128 (got %d)", d);
    MMREC_CHECK_ARG(B >= 0 && M >= 0, "expsum_rows_bwd: negative size (B %lld, M %lld)", (long long)B, (long long)M);
    MMREC_CHECK_ARG(dQ || dT, "expsum_rows_bwd: neither dQ nor dT requested");
    MMREC_CHECK_ARG((B == 0 || (Q && g && ldq >= d)) && (M == 0 || (T && ldt >= d)),
                    "expsum_rows_bwd: null pointer or leading dimension below d");
    MMREC_CHECK_ARG((!dQ || lddq >= d) && (!dT || lddt >= d), "expsum_rows_bwd: output leading dimension below d");
    const size_t need = mmrec_expsum_rows_workspace_bytes(B, M, d);
    MMREC_CHECK_ARG(need == 0 || ws, "expsum_rows_bwd: null workspace");
    if (ws_bytes < need) {
        set_error("expsum_rows_bwd: workspace %zu bytes < %zu", ws_bytes, need);
        return MMREC_EWORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    float* part_q = (float*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    float* part_t = part_q + es_bwd_part_bytes(B, M, d) / 4;
    if (dQ) {
        const int rc = es_bwd_one(Q, ldq, B, T, ldt, M, d, inv_tau, nullptr, g, dQ, lddq, part_q, st);
        if (rc != MMREC_OK) return rc;
    }
    if (dT) {
        const int rc = es_bwd_one(T, ldt, M, Q, ldq, B, d, inv_tau, g, nullptr, dT, lddt, part_t, st);
        if (rc != MMREC_OK) return rc;
    }
    return MMREC_OK;
}
