// n12: GRCN's edge attention (src/models/grcn.py:46-77, 158-166) as one pass over the rows of a CSR, forward and backward.
//
// Rows are target nodes, entries e = (i, j) the edges j -> i of the symmetric interaction list, each interaction its own
// entry (PyG's `x_i` / `x_j` with the default flow).  Forward, for each row i:
//   s_e = <X[i], X[j]>,  m = max_e s_e,  den = sum_e expf(s_e - m) + 1e-16f,  alpha_e = expf(s_e - m) / den,
//   Y[i] = base[i] + sum_e alpha_e X[j]
// (`torch_geometric.utils.softmax` grouped by the target, then the 'add' aggregation and `x + x_hat_1`).  Backward:
//   da_e = <gY[i], X[j]> + g_alpha[e],  c_i = sum_e alpha_e da_e,  ds_e = alpha_e (da_e - c_i),  dXt[i] = sum_e ds_e X[j].
// The source-side terms of dX (alpha_e gY[i] + ds_e X[i] summed over the entries with column j) are K1 products on the
// transposed pattern; ops.edge_attention adds them.  No [nnz, d] tensor is formed.
//
// Each row runs in passes over its entries, with the per-entry scalars parked in the output array (`alpha` / `ds`)
// between passes, so a row of any length needs no shared memory of its own:
//   P1  entry dots (a group of G lanes per entry, fixed xor butterfly), parked; forward also the row max;
//   P2  the row's reduction (forward: sum of expf(s - m); backward: sum of alpha da), lane-strided then a butterfly;
//   P3a the parked scalars become the weights (alpha / ds) in place;
//   P3b Y / dXt = sum of weight X[j], each group in ascending entry order, groups and warps combined in a fixed order.
// Rows of at most `light_max` entries are run by one warp; longer rows (listed in `heavy_rows`, longest first) by the
// EA_WARPS warps of a CTA, each warp taking one contiguous share of the entries, the shares combined through shared
// memory in warp order.  Every CTA takes the heavy rows b, b + grid, ... first, then its warps deal the light rows.  No
// atomics: every sum runs in an order fixed by the row's length and d, so two runs give the same bits.
#include <math.h>

#include "common.cuh"

namespace mmrec {

constexpr int EA_WARPS = 16;     // warps of a CTA (a heavy row's team)

// G lanes per entry, V floats per lane; VEC: d == G * V exactly (d = 64: 16 x 4, d = 128: 32 x 4), the row operand held in
// registers.  Otherwise G = 32, V = 1 and the lanes stride over d.
template <int G, int V, bool VEC>
struct EaCfg {
    static constexpr int NG = 32 / G;    // entries in flight per warp
    static constexpr int CW = G * V;     // columns of one P3b chunk
    static constexpr int U = VEC ? 4 : 2;  // entries in flight per group in P1 / P3b (2 keeps the strided loops spill-free)
};

template <int V>
__device__ __forceinline__ void ld_row(float (&r)[V], const float* p) {
    if constexpr (V == 4) {
        const float4 t = ldg4(p);
        r[0] = t.x; r[1] = t.y; r[2] = t.z; r[3] = t.w;
    } else {
#pragma unroll
        for (int v = 0; v < V; ++v) r[v] = __ldg(p + v);
    }
}

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct EaShared {
    float red[EA_WARPS];
    float part[EA_WARPS][128];
};

// One row [beg, end) by a team of nw warps (tw = this warp's index in the team; nw = 1: no shared memory, no barrier).
// BWD = false: q = X[row], park = alpha, out = Y (+ base).  BWD = true: q = gY[row], park = ds, ga = g_alpha (or null),
// al = alpha, out = dXt.
template <int G, int V, bool VEC, bool BWD>
__device__ void ea_row(int64_t row, int64_t beg, int64_t end, int nw, int tw, EaShared* sh, const int32_t* __restrict__ colidx,
                       const float* __restrict__ X, int64_t ldx, const float* __restrict__ q, int d,
                       const float* __restrict__ base, int64_t ldb, const float* __restrict__ al, const float* __restrict__ ga,
                       float* __restrict__ park, float* __restrict__ out, int64_t ldo) {
    using C = EaCfg<G, V, VEC>;
    const int lane = threadIdx.x & 31, grp = lane / G, j = lane % G;
    const int64_t n = end - beg;
    const int64_t share = (n + nw - 1) / nw;
    const int64_t lo = beg + (int64_t)tw * share < end ? beg + (int64_t)tw * share : end;
    const int64_t hi = lo + share < end ? lo + share : end;

    float qr[VEC ? V : 1];
    if constexpr (VEC) ld_row<V>(qr, q + j * V);

    // P1: entry dots
    float mx = -INFINITY;
    for (int64_t e0 = lo; e0 < hi; e0 += C::NG * C::U) {      // warp-uniform trip count
        float acc[C::U];
#pragma unroll
        for (int u = 0; u < C::U; ++u) {
            const int64_t e = e0 + u * C::NG + grp;
            acc[u] = 0.f;
            if (e < hi) {
                const float* x = X + (int64_t)__ldg(colidx + e) * ldx;
                if constexpr (VEC) {
                    float xr[V];
                    ld_row<V>(xr, x + j * V);
#pragma unroll
                    for (int v = 0; v < V; ++v) acc[u] = fmaf(qr[v], xr[v], acc[u]);
                } else {
                    for (int k = j; k < d; k += G) acc[u] = fmaf(__ldg(q + k), __ldg(x + k), acc[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < C::U; ++u) {
            const float s = group_sum<G>(acc[u]);
            const int64_t e = e0 + u * C::NG + grp;
            if (e < hi && j == 0) {
                if constexpr (BWD) {
                    park[e] = ga ? s + ga[e] : s;
                } else {
                    park[e] = s;
                    mx = fmaxf(mx, s);
                }
            }
        }
    }
    __syncwarp();
    if constexpr (!BWD) {
        mx = warp_max(mx);
        if (nw > 1) {
            if (lane == 0) sh->red[tw] = mx;
            __syncthreads();
            mx = -INFINITY;
            for (int w = 0; w < nw; ++w) mx = fmaxf(mx, sh->red[w]);
            __syncthreads();
        }
    }

    // P2: the row's reduction
    float t = 0.f;
    for (int64_t e = lo + lane; e < hi; e += 32) {
        if constexpr (BWD) t = fmaf(al[e], park[e], t);
        else t += expf(park[e] - mx);
    }
    t = warp_sum(t);
    if (nw > 1) {
        if (lane == 0) sh->red[tw] = t;
        __syncthreads();
        t = 0.f;
        for (int w = 0; w < nw; ++w) t += sh->red[w];
    }
    if constexpr (!BWD) t += 1e-16f;

    // P3a: the weights, in place
    for (int64_t e = lo + lane; e < hi; e += 32) {
        if constexpr (BWD) park[e] = al[e] * (park[e] - t);
        else park[e] = expf(park[e] - mx) / t;
    }
    __syncwarp();

    // P3b: sum of weight * X[j], chunk by chunk of CW columns (one chunk when VEC)
    for (int c0 = 0; c0 < d; c0 += C::CW) {
        float acc[V];
#pragma unroll
        for (int v = 0; v < V; ++v) acc[v] = 0.f;
        const int col = c0 + j * V;
        for (int64_t e0 = lo; e0 < hi; e0 += C::NG * C::U) {
            float xr[C::U][V], w[C::U];
#pragma unroll
            for (int u = 0; u < C::U; ++u) {
                const int64_t e = e0 + u * C::NG + grp;
                w[u] = 0.f;
#pragma unroll
                for (int v = 0; v < V; ++v) xr[u][v] = 0.f;
                if (e < hi) {
                    w[u] = park[e];
                    const float* x = X + (int64_t)__ldg(colidx + e) * ldx;
                    if constexpr (VEC) ld_row<V>(xr[u], x + col);
                    else if (col < d) xr[u][0] = __ldg(x + col);
                }
            }
#pragma unroll
            for (int u = 0; u < C::U; ++u) {
                if (e0 + u * C::NG + grp < hi) {
#pragma unroll
                    for (int v = 0; v < V; ++v) acc[v] = fmaf(w[u], xr[u][v], acc[v]);
                }
            }
        }
#pragma unroll
        for (int o = G; o < 32; o <<= 1) {                              // the warp's groups, fixed butterfly
#pragma unroll
            for (int v = 0; v < V; ++v) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], o);
        }
        float* y = out + row * ldo;
        const float* b = base ? base + row * ldb : nullptr;
        if (nw == 1) {
            if (grp == 0) {
#pragma unroll
                for (int v = 0; v < V; ++v)
                    if (VEC || col + v < d) y[col + v] = b ? b[col + v] + acc[v] : acc[v];
            }
        } else {
            if (grp == 0) {
#pragma unroll
                for (int v = 0; v < V; ++v) sh->part[tw][j * V + v] = acc[v];
            }
            __syncthreads();
            for (int k = threadIdx.x; k < C::CW && c0 + k < d; k += blockDim.x) {
                float s = 0.f;
                for (int w = 0; w < nw; ++w) s += sh->part[w][k];
                y[c0 + k] = b ? b[c0 + k] + s : s;
            }
            __syncthreads();
        }
    }
}

template <int G, int V, bool VEC, bool BWD>
__global__ void __launch_bounds__(EA_WARPS * 32, 2)
edge_attn_kernel(int64_t n_rows, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float* __restrict__ X,
                 int64_t ldx, int d, const float* __restrict__ Q, int64_t ldq, const float* __restrict__ base, int64_t ldb,
                 const float* __restrict__ al, const float* __restrict__ ga, const int32_t* __restrict__ heavy_rows, int64_t n_heavy,
                 int light_max, float* __restrict__ park, float* __restrict__ out, int64_t ldo) {
    __shared__ EaShared sh;
    const int warp = threadIdx.x >> 5;
    for (int64_t h = blockIdx.x; h < n_heavy; h += gridDim.x) {       // CTA-uniform
        const int64_t r = heavy_rows[h];
        ea_row<G, V, VEC, BWD>(r, rowptr[r], rowptr[r + 1], EA_WARPS, warp, &sh, colidx, X, ldx, Q + r * ldq, d, base, ldb, al, ga,
                               park, out, ldo);
    }
    const int64_t nw = (int64_t)gridDim.x * EA_WARPS;
    for (int64_t r = (int64_t)blockIdx.x * EA_WARPS + warp; r < n_rows; r += nw) {   // warp-uniform
        const int64_t beg = rowptr[r], end = rowptr[r + 1];
        if (end - beg > light_max) continue;
        ea_row<G, V, VEC, BWD>(r, beg, end, 1, 0, nullptr, colidx, X, ldx, Q + r * ldq, d, base, ldb, al, ga, park, out, ldo);
    }
}

template <bool BWD>
static int launch_edge_attn(int64_t n_rows, const int32_t* rowptr, const int32_t* colidx, const float* X, int64_t ldx, int d,
                            const float* Q, int64_t ldq, const float* base, int64_t ldb, const float* al, const float* ga,
                            const int32_t* heavy_rows, int64_t n_heavy, int light_max, float* park, float* out, int64_t ldo,
                            cudaStream_t stream) {
    int64_t grid = (n_rows + EA_WARPS - 1) / EA_WARPS;
    if (grid < n_heavy) grid = n_heavy;
    const int64_t cap = (int64_t)sm_count() * 2;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    const bool aligned = (ldx % 4 == 0) && (ldq % 4 == 0) && ((uintptr_t)X % 16 == 0) && ((uintptr_t)Q % 16 == 0);
#define EA_LAUNCH(G_, V_, VEC_)                                                                                                 \
    edge_attn_kernel<G_, V_, VEC_, BWD><<<(unsigned)grid, EA_WARPS * 32, 0, stream>>>(                                        \
        n_rows, rowptr, colidx, X, ldx, d, Q, ldq, base, ldb, al, ga, heavy_rows, n_heavy, light_max, park, out, ldo)
    if (aligned && d == 64) EA_LAUNCH(16, 4, true);
    else if (aligned && d == 128) EA_LAUNCH(32, 4, true);
    else EA_LAUNCH(32, 1, false);
#undef EA_LAUNCH
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

static int check_edge_attn_args(int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* rowptr, const int32_t* colidx,
                                const float* X, int64_t ldx, int d, const int32_t* heavy_rows, int64_t n_heavy, int light_max,
                                const float* out, int64_t ldo) {
    MMREC_CHECK_ARG(n_rows >= 0 && n_rows < (1ll << 31) && nnz >= 0 && nnz < (1ll << 31), "edge_attn: sizes out of range");
    MMREC_CHECK_ARG(n_cols == n_rows, "edge_attn: the matrix must be square (rows and columns index one table), got %lld x %lld",
                    (long long)n_rows, (long long)n_cols);
    MMREC_CHECK_ARG(d >= 1 && ldx >= d && ldo >= d, "edge_attn: need d >= 1, ldx >= d and ldy >= d");
    MMREC_CHECK_ARG(light_max >= 0, "edge_attn: light_max must be >= 0");
    MMREC_CHECK_ARG(n_heavy >= 0 && n_heavy <= n_rows && (n_heavy == 0 || heavy_rows), "edge_attn: bad heavy row list");
    MMREC_CHECK_ARG(n_rows == 0 || (rowptr && X && out && (nnz == 0 || colidx)), "edge_attn: null pointer");
    return MMREC_OK;
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_edge_attn_f32(int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* rowptr, const int32_t* colidx,
                                   const float* X, int64_t ldx, int d, const float* base, int64_t ldb, const int32_t* heavy_rows,
                                   int64_t n_heavy, int light_max, float* alpha, float* Y, int64_t ldy, void* stream_) {
    const int rc = check_edge_attn_args(n_rows, n_cols, nnz, rowptr, colidx, X, ldx, d, heavy_rows, n_heavy, light_max, Y, ldy);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(!base || ldb >= d, "edge_attn: ldb < d");
    MMREC_CHECK_ARG(nnz == 0 || alpha, "edge_attn: null alpha");
    if (n_rows == 0) return MMREC_OK;
    return launch_edge_attn<false>(n_rows, rowptr, colidx, X, ldx, d, X, ldx, base, ldb, nullptr, nullptr, heavy_rows, n_heavy,
                                   light_max, alpha, Y, ldy, (cudaStream_t)stream_);
}

extern "C" int mmrec_edge_attn_bwd_f32(int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* rowptr, const int32_t* colidx,
                                       const float* X, int64_t ldx, int d, const float* gY, int64_t ldg, const float* alpha,
                                       const float* g_alpha, const int32_t* heavy_rows, int64_t n_heavy, int light_max, float* ds,
                                       float* dXt, int64_t ldo, void* stream_) {
    const int rc = check_edge_attn_args(n_rows, n_cols, nnz, rowptr, colidx, X, ldx, d, heavy_rows, n_heavy, light_max, dXt, ldo);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(ldg >= d && (n_rows == 0 || gY), "edge_attn_bwd: need gY with ldg >= d");
    MMREC_CHECK_ARG(nnz == 0 || (alpha && ds), "edge_attn_bwd: null alpha or ds");
    if (n_rows == 0) return MMREC_OK;
    return launch_edge_attn<true>(n_rows, rowptr, colidx, X, ldx, d, gY, ldg, nullptr, 0, alpha, g_alpha, heavy_rows, n_heavy,
                                  light_max, ds, dXt, ldo, (cudaStream_t)stream_);
}
