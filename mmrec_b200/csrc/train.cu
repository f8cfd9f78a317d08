// f1 -- the feature-table gradient path and the optimiser step (SURVEY.md 8f row f1).
//
// The reference trains the raw modality tables (`nn.Embedding.from_pretrained(v_feat, freeze=False)`,
// src/models/freedom.py:58,61; bm3.py / mgcn.py alike) through `nn.Linear` (freedom.py:59,62,205-209), so every training
// batch runs, per modality, the backward of that linear layer over the WHOLE [n_items, F] table -- dW = g^T X, db = sum g,
// dX = g W, a dense [n_items, F] gradient -- and then `torch.optim.Adam.step` (src/common/trainer.py:117-118,185-189) over
// the table: BASELINE.md 2.1 puts 45-60 % of the reference's training time here.  The kernels of this file:
//
//   index_sum_rows   G[i,:] = sum_{j: idx[j] = i} g[j,:]   (ascending j: bit-reproducible).  By linearity the gradient of
//                    a gathered projection `Linear(table)[idx]` w.r.t. the table is G W -- the scatter happens on the
//                    d-wide side (64 floats per row) instead of on F-wide rows (4096).
//   linear_wgrad     dW = g^T X[idx], db = column sums of g: CUDA-core fp32, every CTA owns 512 contiguous columns and
//                    a run of rows (2 KB bursts per table row, cp.async double buffering), per-CTA partials summed in a
//                    fixed order by a second kernel.
//   linear_dgrad     T = G W.  Two epilogues: store T (the dense gradient autograd expects), or -- the point of the
//                    file -- the Adam update of the table with T as the gradient, so that the [n_items, F] gradient
//                    never exists in HBM: the table, exp_avg and exp_avg_sq are read and written exactly once per step
//                    (6 x 4 bytes per element; the unfused sequence moves >= 8 x).
//   adam_multi       torch.optim.Adam's arithmetic for all remaining parameters in one launch per <= 24 tensors.
//
// All arithmetic is IEEE fp32 (fmaf chains, sqrtf, division), in the operation order of torch's `_multi_tensor_adam`.
#include <cuda_runtime.h>
#include <stdlib.h>

#include "common.cuh"

namespace mmrec {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// index_sum_rows: CTA = 32 table rows x 64 columns; warp w owns rows 4w .. 4w+3 and scans the index list ONCE (four
// 32-entry groups per step), a lane owns columns lane and lane + 32 of its warp's four rows -- its accumulators sit in
// shared memory only because the row of a match is a run-time value; nobody else touches them.
// ------------------------------------------------------------------------------------------------
constexpr int ISR_CHUNK = 8192;   // indices staged in shared memory at a time
constexpr int ISR_ROWS = 32;      // table rows per CTA (4 per warp)
constexpr int ISR_COLS = 64;      // columns per CTA

__global__ void __launch_bounds__(256) index_sum_rows_kernel(int64_t n_idx, const int64_t* __restrict__ idx, const float* __restrict__ g,
                                                             int64_t ldg, int d, int64_t n_rows, float* __restrict__ G, int64_t ldG) {
    __shared__ int s_idx[ISR_CHUNK];
    __shared__ float s_acc[8][4][ISR_COLS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row_base = (int64_t)blockIdx.x * ISR_ROWS;
    const int cb = blockIdx.y * ISR_COLS;
    const bool c0_ok = cb + lane < d, c1_ok = cb + lane + 32 < d;
#pragma unroll
    for (int q = 0; q < 4; ++q) { s_acc[warp][q][lane] = 0.f; s_acc[warp][q][lane + 32] = 0.f; }
    for (int64_t c0 = 0; c0 < n_idx; c0 += ISR_CHUNK) {
        const int len = (int)((n_idx - c0) < ISR_CHUNK ? (n_idx - c0) : ISR_CHUNK);
        __syncthreads();
        for (int e = threadIdx.x; e < ISR_CHUNK; e += 256) {
            int rel = -1;
            if (e < len) {
                const int64_t v = idx[c0 + e];
                if (v >= row_base && v < row_base + ISR_ROWS && v < n_rows) rel = (int)(v - row_base);   // others: never matched
            }
            s_idx[e] = rel;
        }
        __syncthreads();
        const int lo = warp * 4;
        for (int it = 0; it < len; it += 128) {                           // (entries beyond len hold -1)
            int v[4];
            unsigned m[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = (it + 32 * u + lane < ISR_CHUNK) ? s_idx[it + 32 * u + lane] - lo : -1;
#pragma unroll
            for (int u = 0; u < 4; ++u) m[u] = __ballot_sync(0xffffffffu, v[u] >= 0 && v[u] < 4);
            if ((m[0] | m[1] | m[2] | m[3]) == 0u) continue;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                unsigned mm = m[u];
                while (mm) {                                                 // ascending j: bit-reproducible sums
                    const int b = __ffs(mm) - 1;
                    mm &= mm - 1;
                    const int q = __shfl_sync(0xffffffffu, v[u], b);
                    const float* src = g + (c0 + it + 32 * u + b) * ldg + cb;
                    if (c0_ok) s_acc[warp][q][lane] += __ldg(src + lane);
                    if (c1_ok) s_acc[warp][q][lane + 32] += __ldg(src + lane + 32);
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int64_t row = row_base + warp * 4 + q;
        if (row < n_rows) {
            if (c0_ok) G[row * ldG + cb + lane] = s_acc[warp][q][lane];
            if (c1_ok) G[row * ldG + cb + lane + 32] = s_acc[warp][q][lane + 32];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// linear_wgrad: part[chunk][k][f] = sum over the chunk's rows j of g[j][k] * X[row(j)][f]
// ------------------------------------------------------------------------------------------------
constexpr int WG_KT = 64;         // k per CTA (blockIdx.z walks d in steps of 64)
constexpr int WG_SC = 512;        // columns per CTA: 2 KB of every table row it visits
constexpr int WG_RT = 16;         // rows per pipeline stage
constexpr int WG_THREADS = 512;
constexpr size_t WG_SMEM = 2 * WG_RT * WG_SC * sizeof(float) + 2 * WG_RT * WG_KT * sizeof(float);

__global__ void __launch_bounds__(WG_THREADS, 1)
linear_wgrad_kernel(int64_t n, const int64_t* __restrict__ idx, const float* __restrict__ g, int64_t ldg, int d, int d_pad,
                    const float* __restrict__ table, int64_t n_table, int64_t F, int vec, int64_t rows_per_chunk, float* __restrict__ part,
                    float* __restrict__ part_b) {
    extern __shared__ __align__(16) unsigned char wg_smem[];
    float* Xs = reinterpret_cast<float*>(wg_smem);                      // [2][RT][SC]
    float* Gs = Xs + 2 * WG_RT * WG_SC;                                  // [2][RT][KT]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int kg = warp >> 1;                                            // 8 k per thread: kg*8 .. kg*8+7
    const int ca = (warp & 1) * 256 + 4 * lane, cb = ca + 128;           // 8 columns per thread: two float4, conflict-free
    const int64_t col0 = (int64_t)blockIdx.x * WG_SC;
    const int k0 = blockIdx.z * WG_KT;
    const int64_t begin = (int64_t)blockIdx.y * rows_per_chunk;
    const int64_t end = (begin + rows_per_chunk < n) ? begin + rows_per_chunk : n;
    const bool want_b = part_b != nullptr && blockIdx.x == 0 && tid < WG_KT;

    for (int e = tid; e < 2 * WG_RT * WG_SC; e += WG_THREADS) Xs[e] = 0.f;   // columns beyond F are never loaded: keep them finite
    __syncthreads();

    float acc[8][8];
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
    float bacc = 0.f;

    auto stage_load = [&](int buf, int64_t r0) {
        float* xs = Xs + buf * WG_RT * WG_SC;
        float* gs = Gs + buf * WG_RT * WG_KT;
#pragma unroll
        for (int i = 0; i < WG_RT * WG_SC / 4 / WG_THREADS; ++i) {       // 4 x 16 bytes per thread
            const int e = i * WG_THREADS + tid;
            const int r = e >> 7, c4 = e & 127;
            int64_t j = r0 + r;
            if (j >= end) j = end - 1;                                   // a valid row; its g entry is zero below
            int64_t row = idx ? idx[j] : j;
            row = row < 0 ? 0 : (row >= n_table ? n_table - 1 : row);
            const int64_t col = col0 + 4 * c4;
            if (vec) {                                                   // F % 4 == 0, 16-byte aligned table
                if (col < F) cp_async16(xs + r * WG_SC + 4 * c4, table + row * F + col);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) xs[r * WG_SC + 4 * c4 + q] = (col + q < F) ? __ldg(table + row * F + col + q) : 0.f;
            }
        }
#pragma unroll
        for (int i = 0; i < WG_RT * WG_KT / WG_THREADS; ++i) {           // 2 floats per thread
            const int e = i * WG_THREADS + tid;
            const int r = e >> 6, k = e & 63;
            const int64_t j = r0 + r;
            gs[r * WG_KT + k] = (j < end && k0 + k < d) ? __ldg(g + j * ldg + k0 + k) : 0.f;
        }
    };

    if (begin < end) {
        stage_load(0, begin);
        cp_async_commit();
        int cur = 0;
        for (int64_t r0 = begin; r0 < end; r0 += WG_RT, cur ^= 1) {
            cp_async_wait_all();
            __syncthreads();                                             // stage `cur` complete; everyone is done with `cur ^ 1`
            if (r0 + WG_RT < end) stage_load(cur ^ 1, r0 + WG_RT);
            cp_async_commit();
            const float* xs = Xs + cur * WG_RT * WG_SC;
            const float* gs = Gs + cur * WG_RT * WG_KT;
#pragma unroll 4
            for (int r = 0; r < WG_RT; ++r) {
                const float4 g0 = *reinterpret_cast<const float4*>(gs + r * WG_KT + kg * 8);
                const float4 g1 = *reinterpret_cast<const float4*>(gs + r * WG_KT + kg * 8 + 4);
                const float4 x0 = *reinterpret_cast<const float4*>(xs + r * WG_SC + ca);
                const float4 x1 = *reinterpret_cast<const float4*>(xs + r * WG_SC + cb);
                const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                const float xv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int a = 0; a < 8; ++a)
#pragma unroll
                    for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(gv[a], xv[b], acc[a][b]);
                if (want_b) bacc += gs[r * WG_KT + tid];
            }
        }
    }
    float* dst = part + ((int64_t)blockIdx.y * d_pad + k0 + kg * 8) * F;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
        if (vec) {
            if (col0 + ca < F) *reinterpret_cast<float4*>(dst + a * F + col0 + ca) = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
            if (col0 + cb < F) *reinterpret_cast<float4*>(dst + a * F + col0 + cb) = make_float4(acc[a][4], acc[a][5], acc[a][6], acc[a][7]);
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (col0 + ca + q < F) dst[a * F + col0 + ca + q] = acc[a][q];
                if (col0 + cb + q < F) dst[a * F + col0 + cb + q] = acc[a][4 + q];
            }
        }
    }
    if (want_b) part_b[(int64_t)blockIdx.y * d_pad + k0 + tid] = bacc;
}

// dW[k][f] = sum_s part[s][k][f] (s ascending), db[k] = sum_s part_b[s][k]
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(int n_chunks, int d, int d_pad, int64_t F, int vec, const float* __restrict__ part,
                                                           const float* __restrict__ part_b, float* __restrict__ dW, float* __restrict__ db) {
    if (vec) {
        const int64_t n4 = (int64_t)d * (F / 4);
        for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < n4; e += (int64_t)gridDim.x * 256) {
            const int64_t k = e / (F / 4), c4 = e - k * (F / 4);
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int c = 0; c < n_chunks; ++c) {
                const float4 v = ldg4(part + ((int64_t)c * d_pad + k) * F + 4 * c4);
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
            *reinterpret_cast<float4*>(dW + k * F + 4 * c4) = s;
        }
    } else {
        const int64_t n1 = (int64_t)d * F;
        for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < n1; e += (int64_t)gridDim.x * 256) {
            const int64_t k = e / F, f = e - k * F;
            float s = 0.f;
            for (int c = 0; c < n_chunks; ++c) s += __ldg(part + ((int64_t)c * d_pad + k) * F + f);
            dW[e] = s;
        }
    }
    if (db && blockIdx.x == 0) {
        for (int k = threadIdx.x; k < d; k += 256) {
            float s = 0.f;
            for (int c = 0; c < n_chunks; ++c) s += part_b[(int64_t)c * d_pad + k];
            db[k] = s;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// linear_dgrad: T[i][f] = sum_k G[i][k] W[k][f], epilogue = store | Adam step of the table
// ------------------------------------------------------------------------------------------------
struct AdamScalars {
    float w1, beta2, w2, eps, weight_decay, step_size, bc2_sqrt;   // w1 = 1 - beta1, w2 = 1 - beta2, rounded from double as torch does
};
static AdamScalars adam_scalars(double beta1, double beta2, double eps, double weight_decay, double step_size, double bc2_sqrt) {
    return AdamScalars{(float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, (float)weight_decay, (float)step_size, (float)bc2_sqrt};
}

// torch/optim/adam.py `_multi_tensor_adam` (the form torch.optim.Adam takes on CUDA tensors), one element, with the
// roundings of ATen's foreach kernels (oracle.adam_foreach_f32 restates them; tests/test_gpu_exact_arith.py compares bits):
//   grad = fma(weight_decay, param, grad);  exp_avg = fma(1 - beta1, grad - exp_avg, exp_avg)        (_foreach_lerp_)
//   exp_avg_sq = fma(1 - beta2, grad * grad, exp_avg_sq * beta2)   (_foreach_mul_, then _foreach_addcmul_: fma(value, t1 t2, x))
//   denom = sqrt(exp_avg_sq) / sqrt(1 - beta2^t) + eps;  param = fma(-(lr / (1 - beta1^t)), exp_avg / denom, param)
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float gr, const AdamScalars& a) {
    if (a.weight_decay != 0.f) gr = fmaf(a.weight_decay, p, gr);
    m = fmaf(a.w1, gr - m, m);
    v = fmaf(a.w2, gr * gr, v * a.beta2);
    const float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
    p = fmaf(a.step_size, m / denom, p);          // step_size = -lr / (1 - beta1^t): negative
}

enum { DG_STORE = 0, DG_ADAM = 1, DG_STORE_ANY = 2 };   // STORE: 16-byte stores, no accumulation; STORE_ANY: run-time vec / accum

template <int KT, int SC>
struct DgradShape {
    static constexpr int CG = SC / 4;            // column groups (float4 per thread)
    static constexpr int RG = 256 / CG;          // row groups of 8 rows
    static constexpr int RT = RG * 8;            // rows per tile
    static constexpr size_t SMEM = (size_t)KT * SC * sizeof(float) + 2 * (size_t)KT * RT * sizeof(float);
};

template <int KT, int SC, int MODE>
__global__ void __launch_bounds__(256, 1)
linear_dgrad_kernel(int64_t n_rows, const float* __restrict__ G, int64_t ldG, int d, const float* __restrict__ W, int64_t F, int vec, int accum,
                    float* out, float* P, float* M, float* V, AdamScalars as) {
    using S = DgradShape<KT, SC>;
    constexpr int CG = S::CG, RT = S::RT;
    extern __shared__ __align__(16) unsigned char dg_smem[];
    float* Ws = reinterpret_cast<float*>(dg_smem);                       // [KT][SC]
    float* Gs = Ws + KT * SC;                                            // [2][KT][RT]  (k-major: the 8 rows of a thread are contiguous)
    const int tid = threadIdx.x;
    const int cg = tid % CG, rg = tid / CG;
    const int64_t col = (int64_t)blockIdx.x * SC + 4 * cg;
    const bool col_ok = col < F;
    const int64_t n_tiles = (n_rows + RT - 1) / RT;

    for (int e = tid; e < KT * (SC / 4); e += 256) {                      // this CTA's column strip of W, resident for its lifetime
        const int k = e / (SC / 4), c4 = e - k * (SC / 4);
        const int64_t c = (int64_t)blockIdx.x * SC + 4 * c4;
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < d && c < F) {
            const float* src = W + (int64_t)k * F + c;
            if (vec) w = ldg4(src);
            else { w.x = __ldg(src); if (c + 1 < F) w.y = __ldg(src + 1); if (c + 2 < F) w.z = __ldg(src + 2); if (c + 3 < F) w.w = __ldg(src + 3); }
        }
        *reinterpret_cast<float4*>(Ws + k * SC + 4 * c4) = w;
    }
    constexpr int GQ = KT * RT / 256;                                     // G tile elements per thread
    auto g_elem = [&](int64_t tile, int i) -> float {                    // element e = i*256 + tid: r fastest (conflict-free stores)
        const int e = i * 256 + tid;
        const int r = e % RT, k = e / RT;
        const int64_t row = tile * RT + r;
        return (row < n_rows && k < d) ? __ldg(G + row * ldG + k) : 0.f;
    };
    float4 pp[8], pm[8], pv[8];
    auto prefetch = [&](int64_t tile) {
        if constexpr (MODE == DG_ADAM) {
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int64_t row = tile * RT + rg * 8 + r;
                if (col_ok && row < n_rows) {
                    pp[r] = *reinterpret_cast<const float4*>(P + row * F + col);
                    pm[r] = *reinterpret_cast<const float4*>(M + row * F + col);
                    pv[r] = *reinterpret_cast<const float4*>(V + row * F + col);
                }
            }
        }
    };

    int64_t tile = blockIdx.y;
    if (tile < n_tiles) {
#pragma unroll
        for (int i = 0; i < GQ; ++i) Gs[(i * 256 + tid)] = g_elem(tile, i);   // layout [k][r] == element order e = k*RT + r
        prefetch(tile);
    }
    __syncthreads();

    for (int buf = 0; tile < n_tiles; tile += gridDim.y, buf ^= 1) {
        const int64_t next = tile + gridDim.y;
        float gq[GQ];
#pragma unroll
        for (int i = 0; i < GQ; ++i) gq[i] = next < n_tiles ? g_elem(next, i) : 0.f;

        float acc[8][4];
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
        const float* gs = Gs + buf * KT * RT + rg * 8;
        const float* ws = Ws + 4 * cg;
#pragma unroll 16
        for (int k = 0; k < KT; ++k) {
            const float4 w = *reinterpret_cast<const float4*>(ws + k * SC);
            const float4 g0 = *reinterpret_cast<const float4*>(gs + k * RT);
            const float4 g1 = *reinterpret_cast<const float4*>(gs + k * RT + 4);
            const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                acc[r][0] = fmaf(gv[r], w.x, acc[r][0]);
                acc[r][1] = fmaf(gv[r], w.y, acc[r][1]);
                acc[r][2] = fmaf(gv[r], w.z, acc[r][2]);
                acc[r][3] = fmaf(gv[r], w.w, acc[r][3]);
            }
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int64_t row = tile * RT + rg * 8 + r;
            if (!(col_ok && row < n_rows)) continue;
            if (MODE == DG_STORE) {
                *reinterpret_cast<float4*>(out + row * F + col) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
            } else if (MODE == DG_STORE_ANY) {
                float* o = out + row * F + col;
                if (vec) {
                    float4 t = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
                    if (accum) { const float4 q = *reinterpret_cast<const float4*>(o); t.x += q.x; t.y += q.y; t.z += q.z; t.w += q.w; }
                    *reinterpret_cast<float4*>(o) = t;
                } else {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (col + q < F) o[q] = accum ? o[q] + acc[r][q] : acc[r][q];
                }
            } else {
                float4 p = pp[r], m = pm[r], v = pv[r];
                adam_update(p.x, m.x, v.x, acc[r][0], as);
                adam_update(p.y, m.y, v.y, acc[r][1], as);
                adam_update(p.z, m.z, v.z, acc[r][2], as);
                adam_update(p.w, m.w, v.w, acc[r][3], as);
                *reinterpret_cast<float4*>(P + row * F + col) = p;
                *reinterpret_cast<float4*>(M + row * F + col) = m;
                *reinterpret_cast<float4*>(V + row * F + col) = v;
            }
        }
        if (next < n_tiles) prefetch(next);                               // in flight during the next tile's k loop
        float* gn = Gs + (buf ^ 1) * KT * RT;
#pragma unroll
        for (int i = 0; i < GQ; ++i) gn[i * 256 + tid] = gq[i];
        __syncthreads();
    }
}

template <int KT, int SC, int MODE>
static int launch_dgrad(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, int vec, int accum, float* out, float* P,
                        float* M, float* V, const AdamScalars& as, cudaStream_t stream) {
    using S = DgradShape<KT, SC>;
    auto kern = linear_dgrad_kernel<KT, SC, MODE>;
    MMREC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::SMEM));   // per device: set every time
    const int64_t strips = (F + SC - 1) / SC;
    const int64_t n_tiles = (n_rows + S::RT - 1) / S::RT;
    int64_t chunks = sm_count() / strips;
    if (chunks < 1) chunks = 1;
    if (chunks > n_tiles) chunks = n_tiles;
    dim3 grid((unsigned)strips, (unsigned)chunks);
    kern<<<grid, 256, S::SMEM, stream>>>(n_rows, G, ldG, d, W, F, vec, accum, out, P, M, V, as);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

template <int MODE>
static int dispatch_dgrad(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, int vec, float* out, float* P,
                          float* M, float* V, const AdamScalars& as, cudaStream_t stream) {
    if (d <= 64) return launch_dgrad<64, 512, MODE>(n_rows, G, ldG, d, W, F, vec, 0, out, P, M, V, as, stream);
    // wider layers: 128 k at a time; the store form accumulates over the k chunks (Adam needs the whole sum at once: d <= 128)
    for (int k0 = 0; k0 < d; k0 += 128) {
        const int dk = d - k0 < 128 ? d - k0 : 128;
        const int rc = launch_dgrad<128, 256, MODE>(n_rows, G + k0, ldG, dk, W + (int64_t)k0 * F, F, vec, k0 > 0, out, P, M, V, as, stream);
        if (rc != MMREC_OK) return rc;
    }
    return MMREC_OK;
}

// ------------------------------------------------------------------------------------------------
// adam_multi
// ------------------------------------------------------------------------------------------------
constexpr int ADAM_MAX = 24;
constexpr int ADAM_BLOCK_ELEMS = 256 * 16;      // 4 float4 per thread
struct AdamEntry {
    float* p; const float* g; float* m; float* v;
    long long n;
    float step_size, bc2_sqrt;
    int first_block, pad;
};
struct AdamBatch {
    AdamEntry t[ADAM_MAX];
    int n_tensors;
    float w1, beta2, w2, eps, weight_decay;
};

__global__ void __launch_bounds__(256) adam_multi_kernel(const __grid_constant__ AdamBatch b) {
    int ti = 0;
    while (ti + 1 < b.n_tensors && (int)blockIdx.x >= b.t[ti + 1].first_block) ++ti;
    const AdamEntry& t = b.t[ti];
    AdamScalars as{b.w1, b.beta2, b.w2, b.eps, b.weight_decay, t.step_size, t.bc2_sqrt};
    const long long base = (long long)(blockIdx.x - t.first_block) * ADAM_BLOCK_ELEMS;
    const bool vec = ((((uintptr_t)t.p | (uintptr_t)t.g | (uintptr_t)t.m | (uintptr_t)t.v) & 15) == 0);
    if (vec && base + ADAM_BLOCK_ELEMS <= t.n) {
        float4 p[4], g[4], m[4], v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const long long e = base + 4 * (i * 256 + threadIdx.x);
            p[i] = *reinterpret_cast<const float4*>(t.p + e);
            g[i] = ldg4(t.g + e);
            m[i] = *reinterpret_cast<const float4*>(t.m + e);
            v[i] = *reinterpret_cast<const float4*>(t.v + e);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const long long e = base + 4 * (i * 256 + threadIdx.x);
            adam_update(p[i].x, m[i].x, v[i].x, g[i].x, as);
            adam_update(p[i].y, m[i].y, v[i].y, g[i].y, as);
            adam_update(p[i].z, m[i].z, v[i].z, g[i].z, as);
            adam_update(p[i].w, m[i].w, v[i].w, g[i].w, as);
            *reinterpret_cast<float4*>(t.p + e) = p[i];
            *reinterpret_cast<float4*>(t.m + e) = m[i];
            *reinterpret_cast<float4*>(t.v + e) = v[i];
        }
    } else {
        for (int i = threadIdx.x; i < ADAM_BLOCK_ELEMS; i += 256) {
            const long long e = base + i;
            if (e >= t.n) break;
            float p = t.p[e], m = t.m[e], v = t.v[e];
            adam_update(p, m, v, t.g[e], as);
            t.p[e] = p; t.m[e] = m; t.v[e] = v;
        }
    }
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_index_sum_rows_f32(int64_t n_idx, const int64_t* idx, const float* g, int64_t ldg, int d, int64_t n_rows, float* G,
                                        int64_t ldG, void* stream_) {
    MMREC_CHECK_ARG(n_idx >= 0 && n_rows >= 0 && d >= 1 && d <= 65535 * ISR_COLS, "index_sum_rows: bad sizes");
    if (n_rows == 0) return MMREC_OK;
    MMREC_CHECK_ARG(G && ldG >= d && (n_idx == 0 || (idx && g && ldg >= d)), "index_sum_rows: null pointer or bad leading dimension");
    dim3 grid((unsigned)((n_rows + ISR_ROWS - 1) / ISR_ROWS), (unsigned)((d + ISR_COLS - 1) / ISR_COLS));
    index_sum_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>(n_idx, idx, g, ldg, d, n_rows, G, ldG);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

static void wgrad_shape(int64_t n, int64_t F, int d, int64_t* strips, int* ktiles, int64_t* chunks, int64_t* rows_per_chunk) {
    *strips = (F + WG_SC - 1) / WG_SC;
    *ktiles = (d + WG_KT - 1) / WG_KT;
    int64_t c = sm_count() / (*strips * *ktiles);
    const int64_t stages = (n + WG_RT - 1) / WG_RT;
    if (c > stages) c = stages;
    if (c < 1) c = 1;
    int64_t rpc = (stages + c - 1) / c * WG_RT;
    c = (n + rpc - 1) / rpc;
    if (c < 1) c = 1;
    *chunks = c;
    *rows_per_chunk = rpc;
}

extern "C" size_t mmrec_linear_wgrad_workspace_bytes(int64_t n, int64_t F, int d) {
    if (n <= 0 || F < 1 || d < 1) return 256;
    int64_t strips, chunks, rpc; int kt;
    wgrad_shape(n, F, d, &strips, &kt, &chunks, &rpc);        // depends on the SM count of the current device, like the launch
    const size_t d_pad = (size_t)kt * WG_KT;
    return align_up((size_t)chunks * d_pad * (size_t)F * sizeof(float), 256) + align_up((size_t)chunks * d_pad * sizeof(float), 256);
}

extern "C" int mmrec_linear_wgrad_f32(int64_t n, const int64_t* idx, const float* g, int64_t ldg, int d, const float* table, int64_t n_table,
                                      int64_t F, float* dW, float* db, void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(n >= 0 && d >= 1 && F >= 1 && n_table >= 0, "linear_wgrad: bad sizes");
    MMREC_CHECK_ARG(dW && (n == 0 || (g && table && ldg >= d && n_table >= 1)), "linear_wgrad: null pointer or bad leading dimension");
    const int vec = (F & 3) == 0 && (((uintptr_t)table | (uintptr_t)dW | (uintptr_t)ws) & 15) == 0;   // else: 4-byte accesses
    if (n == 0) {
        MMREC_CUDA(cudaMemsetAsync(dW, 0, (size_t)d * F * sizeof(float), stream));
        if (db) MMREC_CUDA(cudaMemsetAsync(db, 0, (size_t)d * sizeof(float), stream));
        return MMREC_OK;
    }
    int64_t strips, chunks, rpc; int kt;
    wgrad_shape(n, F, d, &strips, &kt, &chunks, &rpc);
    const int d_pad = kt * WG_KT;
    const size_t part_bytes = align_up((size_t)chunks * d_pad * (size_t)F * sizeof(float), 256);
    const size_t need = part_bytes + align_up((size_t)chunks * d_pad * sizeof(float), 256);
    if (!ws || ws_bytes < need) {
        set_error("linear_wgrad: workspace of %zu bytes needed, %zu given", need, ws_bytes);
        return MMREC_EWORKSPACE;
    }
    float* part = reinterpret_cast<float*>(ws);
    float* part_b = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(ws) + part_bytes);
    MMREC_CUDA(cudaFuncSetAttribute(linear_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM));
    dim3 grid((unsigned)strips, (unsigned)chunks, (unsigned)kt);
    linear_wgrad_kernel<<<grid, WG_THREADS, WG_SMEM, stream>>>(n, idx, g, ldg, d, d_pad, table, n_table, F, vec, rpc, part, db ? part_b : nullptr);
    MMREC_LAUNCH_CHECK();
    const int64_t n_el = vec ? (int64_t)d * (F / 4) : (int64_t)d * F;
    int64_t blocks = (n_el + 255) / 256;
    if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
    wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, stream>>>((int)chunks, d, d_pad, F, vec, part, part_b, dW, db);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

static int dgrad_args(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, const char* who) {
    MMREC_CHECK_ARG(n_rows >= 0 && d >= 1 && F >= 1, "%s: bad sizes", who);
    MMREC_CHECK_ARG(n_rows == 0 || (G && W && ldG >= d), "%s: null pointer or bad leading dimension", who);
    return MMREC_OK;
}

extern "C" int mmrec_linear_dgrad_f32(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, float* dX, void* stream_) {
    const int rc = dgrad_args(n_rows, G, ldG, d, W, F, "linear_dgrad");
    if (rc != MMREC_OK) return rc;
    if (n_rows == 0) return MMREC_OK;
    MMREC_CHECK_ARG(dX, "linear_dgrad: dX is null");
    const int vec = (F & 3) == 0 && (((uintptr_t)W | (uintptr_t)dX) & 15) == 0;       // else: 4-byte accesses
    AdamScalars as{};
    if (vec && d <= 128) return dispatch_dgrad<DG_STORE>(n_rows, G, ldG, d, W, F, 1, dX, nullptr, nullptr, nullptr, as, (cudaStream_t)stream_);
    return dispatch_dgrad<DG_STORE_ANY>(n_rows, G, ldG, d, W, F, vec, dX, nullptr, nullptr, nullptr, as, (cudaStream_t)stream_);
}

extern "C" int mmrec_linear_dgrad_adam_f32(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, float* param,
                                           float* exp_avg, float* exp_avg_sq, double beta1, double beta2, double eps, double weight_decay,
                                           double step_size, double bc2_sqrt, void* stream_) {
    const int rc = dgrad_args(n_rows, G, ldG, d, W, F, "linear_dgrad_adam");
    if (rc != MMREC_OK) return rc;
    if (d > 128 || (F & 3) != 0) {
        set_error("linear_dgrad_adam: d = %d, F = %lld has no fused kernel (d <= 128, F a multiple of 4)", d, (long long)F);
        return MMREC_EUNSUPPORTED;
    }
    if (n_rows == 0) return MMREC_OK;
    MMREC_CHECK_ARG(param && exp_avg && exp_avg_sq && (((uintptr_t)param | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq | (uintptr_t)W) & 15) == 0,
                    "linear_dgrad_adam: pointers null or not 16-byte aligned");
    MMREC_CHECK_ARG(bc2_sqrt > 0.0, "linear_dgrad_adam: bc2_sqrt must be positive");
    const AdamScalars as = adam_scalars(beta1, beta2, eps, weight_decay, step_size, bc2_sqrt);
    return dispatch_dgrad<DG_ADAM>(n_rows, G, ldG, d, W, F, 1, nullptr, param, exp_avg, exp_avg_sq, as, (cudaStream_t)stream_);
}

extern "C" int mmrec_adam_f32(int n_tensors, const mmrec_adam_tensor* tensors, double beta1, double beta2, double eps, double weight_decay,
                              void* stream_) {
    MMREC_CHECK_ARG(n_tensors >= 0 && (n_tensors == 0 || tensors), "adam: bad tensor list");
    for (int i = 0; i < n_tensors; ++i) {
        MMREC_CHECK_ARG(tensors[i].n >= 0 && (tensors[i].n == 0 || (tensors[i].param && tensors[i].grad && tensors[i].exp_avg && tensors[i].exp_avg_sq)),
                        "adam: tensor %d has a null pointer", i);
        MMREC_CHECK_ARG(tensors[i].bc2_sqrt > 0.0, "adam: tensor %d: bc2_sqrt must be positive", i);
    }
    int i = 0;
    while (i < n_tensors) {
        AdamBatch b;
        const AdamScalars hs = adam_scalars(beta1, beta2, eps, weight_decay, 0.0, 1.0);
        b.n_tensors = 0; b.w1 = hs.w1; b.beta2 = hs.beta2; b.w2 = hs.w2; b.eps = hs.eps; b.weight_decay = hs.weight_decay;
        long long blocks = 0;
        while (i < n_tensors && b.n_tensors < ADAM_MAX) {
            const mmrec_adam_tensor& s = tensors[i++];
            if (s.n == 0) continue;
            const long long nb = (s.n + ADAM_BLOCK_ELEMS - 1) / ADAM_BLOCK_ELEMS;
            if (blocks + nb > 0x7fffffffLL) { --i; break; }
            AdamEntry& e = b.t[b.n_tensors++];
            e.p = s.param; e.g = s.grad; e.m = s.exp_avg; e.v = s.exp_avg_sq; e.n = s.n;
            e.step_size = (float)s.step_size; e.bc2_sqrt = (float)s.bc2_sqrt; e.first_block = (int)blocks; e.pad = 0;
            blocks += nb;
        }
        if (b.n_tensors == 0) continue;
        adam_multi_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream_>>>(b);
        MMREC_LAUNCH_CHECK();
    }
    return MMREC_OK;
}
