// n11: sampled dense-dense product over a CSR pattern, the values gradient of a sparse product.
//
// out[e] = <P[row(e), :], Q[colidx[e], :]> for every stored entry e.  With P = dY and Q = X it is dS of Y = S X restricted to
// S's pattern: the gradient of `torch.mm(item_adj, h)` w.r.t. the learned item graph's values (src/models/lattice.py:162-163),
// which the reference forms as the dense [I, I] product dY X^T.  With P = Q = the normalised features it is the cosine of the
// selected kNN pairs (`build_sim` + `build_knn_neighbourhood`, src/utils/utils.py:119-137) without the [I, I] similarities.
//
// A group of T lanes computes one entry: lane j sums k = j, j + T, j + 2T, ... < d with fmaf in ascending k, then the T
// partial sums meet in a fixed xor butterfly (offsets T/2 .. 1); lane 0 of the group writes.  T depends on d only, so every
// entry's arithmetic is fixed and the result has the same bits on every run.  A warp takes 32 consecutive entries: it finds
// the row of the first by binary search over rowptr, and each group walks forward from there (empty rows are skipped).
#include "common.cuh"

namespace mmrec {

constexpr int SDDMM_CHUNK = 32;   // entries per warp task

template <int T>
__global__ void __launch_bounds__(256) sddmm_kernel(int64_t n_rows, int64_t nnz, const int32_t* __restrict__ rowptr,
                                                    const int32_t* __restrict__ colidx, const float* __restrict__ P, int64_t ldp,
                                                    const float* __restrict__ Q, int64_t ldq, int d, float* __restrict__ out) {
    constexpr int G = 32 / T;                                         // entries in flight per warp
    const int lane = threadIdx.x & 31, grp = lane / T, j = lane % T;
    const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t c0 = warp0 * SDDMM_CHUNK; c0 < nnz; c0 += nwarps * SDDMM_CHUNK) {
        int64_t lo = 0, hi = n_rows - 1;                              // the last row r with rowptr[r] <= c0
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) >> 1;
            if (rowptr[mid] <= c0) lo = mid; else hi = mid - 1;
        }
        int64_t row = lo;
        const int64_t c1 = c0 + SDDMM_CHUNK < nnz ? c0 + SDDMM_CHUNK : nnz;
        for (int64_t e0 = c0; e0 < c1; e0 += G) {                    // warp-uniform trip count: the shuffles see every lane
            const int64_t e = e0 + grp;
            const bool valid = e < c1;
            float acc = 0.f;
            if (valid) {
                while (rowptr[row + 1] <= e) ++row;
                const float* p = P + row * ldp;
                const float* q = Q + (int64_t)colidx[e] * ldq;
#pragma unroll 4
                for (int k = j; k < d; k += T) acc = fmaf(__ldg(p + k), __ldg(q + k), acc);
            }
#pragma unroll
            for (int o = T / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (valid && j == 0) out[e] = acc;
        }
    }
}

template <int T>
static int launch_sddmm(int64_t n_rows, int64_t nnz, const int32_t* rowptr, const int32_t* colidx, const float* P, int64_t ldp,
                        const float* Q, int64_t ldq, int d, float* out, cudaStream_t stream) {
    int64_t grid = (nnz + 8 * SDDMM_CHUNK - 1) / (8 * SDDMM_CHUNK);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    sddmm_kernel<T><<<(unsigned)grid, 256, 0, stream>>>(n_rows, nnz, rowptr, colidx, P, ldp, Q, ldq, d, out);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_sddmm_f32(int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* rowptr, const int32_t* colidx,
                               const float* P, int64_t ldp, const float* Q, int64_t ldq, int d, float* out, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(n_rows >= 0 && n_rows < (1ll << 31) && n_cols >= 0 && n_cols < (1ll << 31) && nnz >= 0 && nnz < (1ll << 31),
                    "sddmm: sizes out of range");
    MMREC_CHECK_ARG(d >= 1 && ldp >= d && ldq >= d, "sddmm: need d >= 1, ldp >= d and ldq >= d");
    if (nnz == 0) return MMREC_OK;
    MMREC_CHECK_ARG(n_rows >= 1 && n_cols >= 1, "sddmm: %lld entries in a %lld x %lld matrix", (long long)nnz, (long long)n_rows,
                    (long long)n_cols);
    MMREC_CHECK_ARG(rowptr && colidx && P && Q && out, "sddmm: null pointer");
    if (d <= 32) return launch_sddmm<8>(n_rows, nnz, rowptr, colidx, P, ldp, Q, ldq, d, out, stream);
    if (d <= 64) return launch_sddmm<16>(n_rows, nnz, rowptr, colidx, P, ldp, Q, ldq, d, out, stream);
    return launch_sddmm<32>(n_rows, nnz, rowptr, colidx, P, ldp, Q, ldq, d, out, stream);
}
