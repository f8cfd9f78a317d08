// The trainer's mask (entries (rows[j], cols[j]), global item columns) as a CSR over batch rows, for the fused scoring
// (K3, score_cf.cu) and the sparse scoring (K9, sparse_score.cu).  Entries outside rows [0, B) are dropped; an entry holds
// cols[j] - item_offset if that lies in [0, n_items), else -1 (mask_item): it matches no item, as mmrec_mask_f32 ignores
// it, but still counts in its row (K3's need = k + masked entries).  Order inside a row is free.  Three routes:
//   sorted    (the reference's loader emits the mask row-major: src/utils/dataloader.py:370-391) one parallel pass sets the
//             row pointers where the row changes and flags any descent per block (mask_sorted_block; K3 runs it inside its
//             prep kernel), then, for arbitrary order, one CTA counts in shared memory, scans and fills -- it exits at once
//             when no block flagged a descent.  B <= MC_MAX_ROWS, nnz <= MC_MAX_NNZ;
//   large     otherwise: global count, library scan, fill.
#pragma once
#include "common.cuh"

namespace mmrec {

constexpr int MC_MAX_ROWS = 8192;
constexpr int64_t MC_MAX_NNZ = 1ll << 18;
constexpr int MC_SORTED_THREADS = 256;          // threads per block of the sorted pass (entries + one sentinel thread)

__device__ __forceinline__ int32_t mask_item(int64_t col, int64_t item_offset, int64_t n_items) {
    const int64_t v = col - item_offset;
    return (uint64_t)v < (uint64_t)n_items ? (int32_t)v : -1;
}

inline bool mask_small(int64_t B, int64_t nnz) { return B <= MC_MAX_ROWS && nnz <= MC_MAX_NNZ; }
__host__ __device__ inline int64_t mask_sorted_blocks(int64_t nnz) { return (nnz + MC_SORTED_THREADS) / MC_SORTED_THREADS; }

// A mask and its CSR (defined in batch_mask.cu).
struct BatchMask {
    int64_t nnz, B, item_offset, n_items;
    const int64_t *rows, *cols;
    int32_t* ptr;                               // [B + 1]
    int32_t* items;                             // [nnz]
    int32_t* aux;                               // fill cursors (large route), or the sorted pass's per-block descent flags
    void* scan;                                 // library scan scratch (large route)
    size_t scan_bytes, bytes;                   // bytes: the workspace taken
};
// The CSR carved from the 256-byte aligned workspace `ws`; with ws == NULL only the sizes are set.
BatchMask batch_mask(void* ws, int64_t nnz, const int64_t* rows, const int64_t* cols, int64_t B, int64_t item_offset, int64_t n_items);
int batch_mask_unsorted(const BatchMask& M, cudaStream_t stream);       // the CTA after a sorted pass
int batch_mask_large(const BatchMask& M, cudaStream_t stream);
int batch_mask_build(const BatchMask& M, cudaStream_t stream);          // standalone, any route; nnz > 0

// Block `blk` of the sorted pass (blockDim.x == MC_SORTED_THREADS); aux[blk] = 1: a descent, ptr / items are garbage.
__device__ __forceinline__ void mask_sorted_block(int64_t blk, const BatchMask& M) {
    const int64_t j = blk * (int64_t)blockDim.x + threadIdx.x, B = M.B;        // entry j, plus one sentinel thread j == nnz
    int64_t rj = 0, rp = 0;
    if (j <= M.nnz) {
        rj = j < M.nnz ? __ldg(M.rows + j) : B;
        rp = j > 0 ? __ldg(M.rows + j - 1) : -1;
        if (j < M.nnz) M.items[j] = mask_item(__ldg(M.cols + j), M.item_offset, M.n_items);
    }
    // a block that saw a descent writes no pointer: the unsorted route rebuilds them all, and on an unsorted mask the runs
    // between consecutive entries would cost O(B) each
    const int bad = __syncthreads_or(j < M.nnz && rp > rj);
    if (threadIdx.x == 0) M.aux[blk] = bad;
    if (bad || j > M.nnz) return;
    // rows (rp, rj] start at entry j (rows outside [0, B) own no pointer; clamped so that they delimit correctly)
    const int64_t lo = rp < -1 ? -1 : (rp > B ? B : rp), hi = rj < -1 ? -1 : (rj > B ? B : rj);
    for (int64_t r = lo + 1; r <= hi; ++r) M.ptr[r] = (int32_t)j;
}

}  // namespace mmrec
