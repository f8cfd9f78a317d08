// K3 (part): train-positive mask, exact per-row top-k, the cross-shard top-k merge, and the scatter of the exact route on
// listed rows (exact_rows.cuh).
// Contract (stronger than torch.topk, which leaves tie order open): descending value, equal values in
// ascending item index.  Replaces src/common/trainer.py:307-309.
//
// mmrec_topk_rows_f32: one CTA per row, cta_topk_from_keys (select.cuh): radix select (4 passes x 8 bits over
// order-preserving keys) finds the k-th largest key; everything above it is gathered unordered, the ties on the
// k-th key are taken in index order (block-wide ordered compaction), then a bitonic sort on the composite
// (key, ~index) puts the k winners in contract order.  (A warp-per-row streaming filter with bitonic compaction
// was measured 2.5x slower at 7k items: the compaction sorts dominate.)
#include "exact_rows.cuh"
#include "peer_sync.cuh"
#include "select.cuh"

namespace mmrec {

__global__ void mask_kernel(int64_t nnz, const int64_t* __restrict__ rows, const int64_t* __restrict__ cols, int64_t row0,
                            int64_t B, int64_t n_items, int64_t item_offset, float* __restrict__ S, int64_t ldS) {
    int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= nnz) return;
    int64_t r = rows[j] - row0, c = cols[j] - item_offset;
    if (r >= 0 && r < B && c >= 0 && c < n_items) S[r * ldS + c] = -1e10f;   // trainer.py:307
}

constexpr int TOPK_THREADS = SELECT_THREADS;

__global__ void __launch_bounds__(TOPK_THREADS) topk_rows_kernel(int64_t n_items, const float* __restrict__ S, int64_t ldS,
                                                                 int k, int64_t item_offset, int64_t* __restrict__ out_idx,
                                                                 float* __restrict__ out_val) {
    __shared__ TopkSmem sm;
    const float* row = S + (int64_t)blockIdx.x * ldS;
    cta_topk_from_keys<TOPK_THREADS>([=](int64_t i) { return float_key(row[i]); }, n_items, k, item_offset,
                                     out_idx + (int64_t)blockIdx.x * k, out_val + (int64_t)blockIdx.x * k, sm);
}

// merge `parts` sorted [B,k] lists per row.  Candidates parts*k <= 4096.
__global__ void __launch_bounds__(TOPK_THREADS) topk_merge_kernel(int parts, int64_t B, int k, const float* __restrict__ vals,
                                                                  const int64_t* __restrict__ idx, int64_t* __restrict__ out_idx,
                                                                  float* __restrict__ out_val) {
    extern __shared__ uint64_t cand[];   // n2 composites (value key, ~slot) + n2 int64 indices
    const int n = parts * k;
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    int64_t* cidx = reinterpret_cast<int64_t*>(cand + n2);
    const int64_t b = blockIdx.x;
    // tie rule: equal values -> lower GLOBAL item index.  Indices need 64 bits, so sort on (key, ~rank) where
    // rank is the position of the candidate's index among the candidates; with at most 4096 candidates a
    // direct O(n) rank count per candidate is cheap and keeps the composite in 64 bits.
    for (int t = threadIdx.x; t < n; t += TOPK_THREADS) {
        int part = t / k, j = t % k;
        cidx[t] = idx[((int64_t)part * B + b) * k + j];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < n2; t += TOPK_THREADS) {
        if (t < n) {
            int part = t / k, j = t % k;
            float v = vals[((int64_t)part * B + b) * k + j];
            int64_t me = cidx[t];
            unsigned rank = 0;
            for (int u = 0; u < n; ++u) rank += (cidx[u] < me) || (cidx[u] == me && u < t);
            cand[t] = ((uint64_t)float_key(v) << 32) | (uint32_t)(~rank);
        } else {
            cand[t] = 0;
        }
    }
    __syncthreads();
    // keep rank -> slot map: after sorting we need the index; store slot by rank
    __shared__ int slot_of_rank[4096];
    for (int t = threadIdx.x; t < n; t += TOPK_THREADS) slot_of_rank[(uint32_t)(~(uint32_t)cand[t])] = t;
    __syncthreads();
    bitonic_desc(cand, n2);
    for (int t = threadIdx.x; t < k; t += TOPK_THREADS) {
        uint64_t c = cand[t];
        int slot = slot_of_rank[(uint32_t)(~(uint32_t)c)];
        out_idx[b * k + t] = cidx[slot];
        out_val[b * k + t] = key_float((uint32_t)(c >> 32));
    }
}

// The same merge with the lists left where the ranks wrote them: list `p` is [B, k] behind vals[p] / idx[p] (peer-mapped
// memory in the item-sharded evaluation), and a local item id becomes the global one as idx * idx_mul + p * idx_add
// (round-robin shards: idx_mul = world, idx_add = 1; pass 1, 0 for ids that are global already).  Rows [row0, row0 +
// n_rows) only: in the sharded evaluation every rank merges its own slice of the batch.
//
// One warp per row.  Every list arrives sorted on the composite (value desc, global item asc) -- a list's local order is
// its global order, the relabelling is monotone -- so the rank of an element is the sum over the lists of the number of
// larger composites there, found by binary search: O(parts log k) per element instead of comparing all pairs.
constexpr int MERGE_MAX_PEERS = 16;
constexpr int MERGE_WARPS = 4;
constexpr int MERGE_WARP_CAP = 1024;    // parts * k one warp handles
struct MergePeers { const float* v[MERGE_MAX_PEERS]; const int64_t* i[MERGE_MAX_PEERS]; };

__device__ __forceinline__ void topk_merge_row(int parts, int k, const MergePeers& src, int64_t idx_mul, int64_t idx_add, int64_t b, int64_t r,
                                               uint64_t* comp, int lane, bool fresh, int64_t* __restrict__ out_idx, float* __restrict__ out_val) {
    const int n = parts * k;
    for (int t = lane; t < n; t += 32) {
        const int p = t / k, j = t - p * k;
        // (`fresh`: the lists were written by other GPUs moments ago -- bypass any cached line of an earlier batch)
        const int64_t li = fresh ? __ldcv(src.i[p] + b * k + j) : src.i[p][b * k + j];
        const float lv = fresh ? __ldcv(src.v[p] + b * k + j) : src.v[p][b * k + j];
        const int64_t gi = li * idx_mul + p * idx_add;                                 // < 2^32 (checked by the host)
        comp[t] = ((uint64_t)float_key(lv) << 32) | (uint32_t)(~(uint32_t)gi);
    }
    __syncwarp();
    for (int t = lane; t < n; t += 32) {
        const uint64_t me = comp[t];
        const int p = t / k, j = t - p * k;
        int rank = j;                                                // its own list: the j elements before it
        for (int q = 0; q < parts && rank < k; ++q) {
            if (q == p) continue;
            const uint64_t* lst = comp + q * k;
            int lo = 0, hi = k;                                      // first position whose composite is < me
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (lst[mid] > me) lo = mid + 1; else hi = mid;
            }
            rank += lo;
        }
        if (rank < k) {
            out_idx[r * k + rank] = (int64_t)(uint32_t)(~(uint32_t)me);
            out_val[r * k + rank] = key_float((uint32_t)(me >> 32));
        }
    }
}

__global__ void __launch_bounds__(32 * MERGE_WARPS) topk_merge_peers_kernel(int parts, int64_t B, int k, const MergePeers src, int64_t idx_mul,
                                                                            int64_t idx_add, int64_t row0, int64_t n_rows,
                                                                            int64_t* __restrict__ out_idx, float* __restrict__ out_val,
                                                                            const PeerFlags flags, int* __restrict__ state, int rank) {
    __shared__ uint64_t comp_all[MERGE_WARPS][MERGE_WARP_CAP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // with flags: the wait for "every rank has written its lists" happens here instead of in a barrier launch
    const int epoch = state ? peer_enter(flags, state, rank, parts) : 0;
    const int64_t r = (int64_t)blockIdx.x * MERGE_WARPS + warp;
    if (r < n_rows) topk_merge_row(parts, k, src, idx_mul, idx_add, row0 + r, r, comp_all[warp], lane, state != nullptr, out_idx, out_val);
    if (state) peer_leave(flags, state, rank, parts, epoch, false);
}

}  // namespace mmrec

namespace mmrec {
int mask_apply(int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int64_t row0, int64_t B,
               int64_t n_items, int64_t item_offset, float* S, int64_t ldS, cudaStream_t stream) {
    if (mask_nnz == 0 || B == 0) return MMREC_OK;
    mask_kernel<<<(unsigned)((mask_nnz + 255) / 256), 256, 0, stream>>>(mask_nnz, mask_rows, mask_cols, row0, B, n_items,
                                                                        item_offset, S, ldS);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

__global__ void exact_scatter_kernel(int64_t c, int k, const int64_t* __restrict__ pos, const int64_t* __restrict__ ti,
                                     const float* __restrict__ tv, int64_t* __restrict__ out_idx, float* __restrict__ out_val) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= c * k) return;
    const int64_t s = t / k, j = t - s * k;
    out_idx[pos[s] * k + j] = ti[t];
    out_val[pos[s] * k + j] = tv[t];
}
}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_mask_f32(int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int64_t B,
                              int64_t n_items, int64_t item_offset, float* S, int64_t ldS, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(mask_nnz >= 0 && B >= 0 && n_items >= 0, "mask: bad sizes");
    if (mask_nnz == 0 || B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(mask_rows && mask_cols && S && ldS >= n_items, "mask: null pointer or ldS < n_items");
    return mask_apply(mask_nnz, mask_rows, mask_cols, 0, B, n_items, item_offset, S, ldS, stream);
}

extern "C" int mmrec_topk_rows_f32(int64_t B, int64_t n_items, const float* S, int64_t ldS, int k, int64_t item_offset,
                                   int64_t* out_idx, float* out_val, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(B >= 0 && n_items >= 1 && k >= 1 && k <= TOPK_MAXK && k <= n_items, "topk_rows: need 1 <= k <= min(%d, n_items)", TOPK_MAXK);
    MMREC_CHECK_ARG(n_items < (1ll << 32), "topk_rows: n_items must fit 32 bits");
    if (B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(S && out_idx && out_val && ldS >= n_items, "topk_rows: null pointer or ldS < n_items");
    topk_rows_kernel<<<(unsigned)B, TOPK_THREADS, 0, stream>>>(n_items, S, ldS, k, item_offset, out_idx, out_val);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_topk_merge(int parts, int64_t B, int k, const float* vals, const int64_t* idx, int64_t* out_idx,
                                float* out_val, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(parts >= 1 && B >= 0 && k >= 1 && (int64_t)parts * k <= 4096, "topk_merge: need parts*k <= 4096");
    if (B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(vals && idx && out_idx && out_val, "topk_merge: null pointer");
    int n = parts * k, n2 = 1;
    while (n2 < n) n2 <<= 1;
    size_t smem = (size_t)n2 * 16;
    MMREC_CUDA(cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
    topk_merge_kernel<<<(unsigned)B, TOPK_THREADS, smem, stream>>>(parts, B, k, vals, idx, out_idx, out_val);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_topk_merge_peers(int parts, int64_t B, int k, const void* const* vals, const void* const* idx, int64_t idx_mul,
                                      int64_t idx_add, int64_t row0, int64_t n_rows, int64_t* out_idx, float* out_val,
                                      void* const* flags, int32_t* state, int rank, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(parts >= 1 && parts <= MERGE_MAX_PEERS && B >= 0 && k >= 1 && (int64_t)parts * k <= MERGE_WARP_CAP,
                    "topk_merge_peers: need parts <= 16 and parts*k <= 1024");
    MMREC_CHECK_ARG(row0 >= 0 && n_rows >= 0 && row0 + n_rows <= B, "topk_merge_peers: row range outside the batch");
    MMREC_CHECK_ARG((flags == nullptr) == (state == nullptr) && (!flags || (rank >= 0 && rank < parts)), "topk_merge_peers: flags / state / rank");
    if (B == 0 || (n_rows == 0 && !flags)) return MMREC_OK;
    MMREC_CHECK_ARG(vals && idx && (n_rows == 0 || (out_idx && out_val)), "topk_merge_peers: null pointer");
    MergePeers src;
    PeerFlags F;
    for (int p = 0; p < MERGE_MAX_PEERS; ++p) { src.v[p] = nullptr; src.i[p] = nullptr; F.f[p] = nullptr; }
    for (int p = 0; p < parts; ++p) {
        MMREC_CHECK_ARG(vals[p] && idx[p] && (!flags || flags[p]), "topk_merge_peers: null list / flag pointer");
        src.v[p] = (const float*)vals[p]; src.i[p] = (const int64_t*)idx[p];
        if (flags) F.f[p] = (int*)flags[p];
    }
    int64_t grid = (n_rows + MERGE_WARPS - 1) / MERGE_WARPS;
    if (grid < 1) grid = 1;                                          // (a rank without rows still takes part in the barrier)
    topk_merge_peers_kernel<<<(unsigned)grid, 32 * MERGE_WARPS, 0, stream>>>(parts, B, k, src, idx_mul, idx_add, row0, n_rows, out_idx, out_val,
                                                                           F, state, rank);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
