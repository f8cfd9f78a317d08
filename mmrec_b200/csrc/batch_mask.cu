// The batch mask CSR (batch_mask.cuh): the unsorted and large routes, and the standalone build.
#include <cub/device/device_scan.cuh>

#include "batch_mask.cuh"

namespace mmrec {

constexpr int MC_THREADS = 1024;

__global__ void __launch_bounds__(MC_SORTED_THREADS) mask_sorted_kernel(const BatchMask M) { mask_sorted_block(blockIdx.x, M); }

// Exclusive scan of a[0 .. n) by one CTA of MC_THREADS threads, each owning a contiguous run: the offsets go to ptr[] and
// replace a[] (which becomes the fill cursor).  wtot: 32 words of shared memory.
__device__ __forceinline__ void cta_exclusive_scan(int32_t* a, int n, int32_t* __restrict__ ptr, int32_t* wtot) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int per = (n + MC_THREADS - 1) / MC_THREADS;
    const int r0 = tid * per, r1 = min(n, r0 + per);
    int local = 0;
    for (int r = r0; r < r1; ++r) local += a[r];
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) wtot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int v = wtot[lane], sc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, sc, o);
            if (lane >= o) sc += u;
        }
        wtot[lane] = sc - v;                                         // exclusive warp offsets
    }
    __syncthreads();
    int run = wtot[wid] + incl - local;
    for (int r = r0; r < r1; ++r) {
        const int c = a[r];
        ptr[r] = run;
        a[r] = run;
        run += c;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(MC_THREADS) mask_csr_small_kernel(const BatchMask M) {
    extern __shared__ int32_t mc_sm[];                               // count / cursor [B + 1] | warp totals [32]
    {   // runs only when the sorted pass found the rows out of order (it then left garbage behind)
        int any = 0;
        for (int i = threadIdx.x; i < mask_sorted_blocks(M.nnz); i += MC_THREADS) any |= M.aux[i];
        if (!__syncthreads_or(any)) return;
    }
    const int64_t nnz = M.nnz;
    const int B = (int)M.B;
    int32_t* cnt = mc_sm;
    const int tid = threadIdx.x, lane = tid & 31;
    for (int r = tid; r <= B; r += MC_THREADS) cnt[r] = 0;
    __syncthreads();
    constexpr int MC_U = 8;                                          // loads in flight per thread (the loop is latency-bound)
    for (int64_t jb = 0; jb < nnz; jb += (int64_t)MC_U * MC_THREADS) {        // warp-uniform trip count (match / shfl below)
        const int64_t j0 = jb + tid;
        int64_t r[MC_U];
#pragma unroll
        for (int u = 0; u < MC_U; ++u) {
            const int64_t j = j0 + (int64_t)u * MC_THREADS;
            r[u] = j < nnz ? __ldg(M.rows + j) : -1;
        }
#pragma unroll
        for (int u = 0; u < MC_U; ++u) {
            // one atomic per distinct row of the warp (same-address shared atomics serialise a full round trip each)
            const int rr = (r[u] >= 0 && r[u] < B) ? (int)r[u] : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, rr);
            if (rr >= 0 && lane == __ffs(peers) - 1) atomicAdd(cnt + rr, __popc(peers));
        }
    }
    __syncthreads();
    cta_exclusive_scan(cnt, B + 1, M.ptr, mc_sm + B + 1);
    for (int64_t jb = 0; jb < nnz; jb += (int64_t)MC_U * MC_THREADS) {
        const int64_t j0 = jb + tid;
        int64_t r[MC_U];
        int32_t it[MC_U];
#pragma unroll
        for (int u = 0; u < MC_U; ++u) {
            const int64_t j = j0 + (int64_t)u * MC_THREADS;
            r[u] = j < nnz ? __ldg(M.rows + j) : -1;
            it[u] = j < nnz ? mask_item(__ldg(M.cols + j), M.item_offset, M.n_items) : -1;
        }
#pragma unroll
        for (int u = 0; u < MC_U; ++u) {
            const int rr = (r[u] >= 0 && r[u] < B) ? (int)r[u] : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, rr);
            const int leader = __ffs(peers) - 1;
            int base = 0;
            if (rr >= 0 && lane == leader) base = atomicAdd(cnt + rr, __popc(peers));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (rr >= 0) M.items[base + __popc(peers & ((1u << lane) - 1u))] = it[u];
        }
    }
}

__global__ void mask_count_kernel(const BatchMask M) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = j < M.nnz ? __ldg(M.rows + j) : -1;
    if (r >= 0 && r < M.B) atomicAdd(M.aux + r, 1);
}

__global__ void mask_fill_kernel(const BatchMask M) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = j < M.nnz ? __ldg(M.rows + j) : -1;
    if (r >= 0 && r < M.B) M.items[M.ptr[r] + atomicAdd(M.aux + r, 1)] = mask_item(__ldg(M.cols + j), M.item_offset, M.n_items);
}

BatchMask batch_mask(void* ws, int64_t nnz, const int64_t* rows, const int64_t* cols, int64_t B, int64_t item_offset, int64_t n_items) {
    BatchMask M{nnz, B, item_offset, n_items, rows, cols};
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return ws ? (char*)ws + o : nullptr; };
    M.ptr = (int32_t*)take((size_t)(B + 2) * 4);
    M.aux = (int32_t*)take((size_t)(B + 2 > mask_sorted_blocks(MC_MAX_NNZ) ? B + 2 : mask_sorted_blocks(MC_MAX_NNZ)) * 4);
    M.items = (int32_t*)take((size_t)(nnz > 0 ? nnz : 1) * 4);
    cub::DeviceScan::ExclusiveSum(nullptr, M.scan_bytes, (int32_t*)nullptr, (int32_t*)nullptr, (int64_t)(B + 1));
    M.scan = take(M.scan_bytes);
    M.bytes = off;
    return M;
}

int batch_mask_unsorted(const BatchMask& M, cudaStream_t stream) {
    mask_csr_small_kernel<<<1, MC_THREADS, (size_t)(M.B + 1 + 32) * 4, stream>>>(M);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

int batch_mask_large(const BatchMask& M, cudaStream_t stream) {
    const unsigned g = (unsigned)((M.nnz + 255) / 256);
    MMREC_CUDA(cudaMemsetAsync(M.aux, 0, (size_t)(M.B + 2) * 4, stream));
    mask_count_kernel<<<g, 256, 0, stream>>>(M);
    MMREC_LAUNCH_CHECK();
    size_t tmp = M.scan_bytes;
    MMREC_CUDA(cub::DeviceScan::ExclusiveSum(M.scan, tmp, M.aux, M.ptr, M.B + 1, stream));
    MMREC_CUDA(cudaMemsetAsync(M.aux, 0, (size_t)(M.B + 2) * 4, stream));
    mask_fill_kernel<<<g, 256, 0, stream>>>(M);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

int batch_mask_build(const BatchMask& M, cudaStream_t stream) {
    if (!mask_small(M.B, M.nnz)) return batch_mask_large(M, stream);
    mask_sorted_kernel<<<(unsigned)mask_sorted_blocks(M.nnz), MC_SORTED_THREADS, 0, stream>>>(M);
    MMREC_LAUNCH_CHECK();
    return batch_mask_unsorted(M, stream);
}

}  // namespace mmrec
