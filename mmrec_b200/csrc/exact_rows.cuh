// The exact route on listed rows, run from the host.  The kNN build (K7, knn_cf.cu) and the sparse scoring (K9,
// sparse_score.cu) list the rows their fused kernel cannot serve and read the count back; those rows are then scored
// densely in chunks (the caller's fill), ranked by mmrec_topk_rows_f32 and put in place: bit-identical to the unfused route
// by construction.  (The fused scoring, K3, keeps its exact rows on the device: it never synchronises.)
#pragma once
#include "common.cuh"

namespace mmrec {

// Rows of one chunk's dense score block: <= 256 MB, <= 1024 rows, <= max_rows (>= 1).
inline int64_t exact_block_rows(int64_t n, int64_t max_rows) {
    int64_t r = (256ll << 20) / (4 * n);
    r = r < 1 ? 1 : (r > 1024 ? 1024 : r);
    return r < max_rows ? r : max_rows;
}

// Workspace (256-byte aligned): the score block [s_rows, n] | its top-k indices | values.
inline size_t exact_rows_bytes(int64_t s_rows, int64_t n, int k) {
    return align_up((size_t)s_rows * n * 4, 256) + align_up((size_t)s_rows * k * 8, 256) + (size_t)s_rows * k * 4;
}

// The count a fused kernel bumped once per listed row (synchronises the stream); negative: an error code.
inline int64_t read_count(const int32_t* counter, cudaStream_t stream) {
    int32_t cnt = 0;
    MMREC_CUDA(cudaMemcpyAsync(&cnt, counter, 4, cudaMemcpyDeviceToHost, stream));
    MMREC_CUDA(cudaStreamSynchronize(stream));
    return cnt;
}

// Top-k rows s < c -> output rows pos[s].  Defined in topk.cu.
__global__ void exact_scatter_kernel(int64_t c, int k, const int64_t* __restrict__ pos, const int64_t* __restrict__ ti,
                                     const float* __restrict__ tv, int64_t* __restrict__ out_idx, float* __restrict__ out_val);

// List rows j < cnt: fill(c0, c, S) writes the scores of list rows c0 .. c0 + c - 1 into S [c, n] (returns an error code);
// their top-k goes to output row dst_pos[j], or to row j when dst_pos is NULL.
template <class Fill>
int exact_rows_topk(int64_t cnt, const int64_t* dst_pos, int64_t n, int k, int64_t s_rows, void* ws, int64_t* out_idx, float* out_val,
                    cudaStream_t stream, Fill fill) {
    float* S = (float*)ws;
    int64_t* ti = (int64_t*)((char*)ws + align_up((size_t)s_rows * n * 4, 256));
    float* tv = (float*)((char*)ti + align_up((size_t)s_rows * k * 8, 256));
    for (int64_t c0 = 0; c0 < cnt; c0 += s_rows) {
        const int64_t c = cnt - c0 < s_rows ? cnt - c0 : s_rows;
        int rc = fill(c0, c, S);
        if (!rc) rc = dst_pos ? mmrec_topk_rows_f32(c, n, S, n, k, 0, ti, tv, stream)
                              : mmrec_topk_rows_f32(c, n, S, n, k, 0, out_idx + c0 * k, out_val + c0 * k, stream);
        if (rc) return rc;
        if (dst_pos) {
            exact_scatter_kernel<<<(unsigned)((c * k + 255) / 256), 256, 0, stream>>>(c, k, dst_pos + c0, ti, tv, out_idx, out_val);
            MMREC_LAUNCH_CHECK();
        }
    }
    return MMREC_OK;
}

}  // namespace mmrec
