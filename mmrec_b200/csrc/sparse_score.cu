// K9: user scores from two sparse operands, `scores_matrix = torch.mm(R, item_sim)` of ItemKNNCBF
// (src/models/itemknncbf.py:54, gathered per batch at :107-111), without the dense [I, I] graph or the dense [U, I] scores.
//
//   R  the training interactions, CSR [U, I] with the dataset's values (columns ascending within a row);
//   S  the item kNN graph, CSR [I, I], knn_k entries per row (distinct columns).
//
// THE arithmetic: score[u, j] = sum over the entries i of R(u), in ascending column order, of R[u, i] * S[i, j], one
// fmaf(r, s, acc) per entry from acc = +0.0.  Items that no S row of R(u) reaches stay +0.0.  (With r = 1 that is acc + s,
// the dense product's sum.)  Every value this file returns is that chain.
//
//   sparse_scores_kernel  mmrec_sparse_scores_f32, the dense [B, I] rows of full_sort_predict: the rows are zero-filled, then
//                         one warp per batch row walks R(u) in order and its lanes add the entries of each S row (distinct
//                         columns: no two lanes touch one element; __syncwarp orders the S rows).  No atomics: deterministic.
//   sparse_topk_kernel    mmrec_sparse_score_topk_f32, one CTA per batch row, nothing dense written:
//                         1. gather the products of R(u) x S as (column, slot) keys, slot = their position in R order, with
//                            (r, s) beside them in shared memory;
//                         2. bitonic sort (select.cuh) on (column, slot): each column's products in R order;
//                         3. one thread per column sums its products in that order -- the same fmaf chain as the dense row;
//                         4. the row's masked items (batch mask CSR, batch_mask.cuh) are sorted; each is looked up by binary
//                            search among the summed columns;
//                         5. rank.  The dense row is +0.0 everywhere except at the "exceptions": masked items (-1e10) and
//                            unmasked columns whose sum is not +0.0 (bit pattern).  The exceptions are sorted on (float_key,
//                            ~index); the output is the exceptions above +0.0, then the +0.0 items in ascending index
//                            (every item that is not an exception), then the remaining exceptions.
//                         This is the order of mmrec_topk_rows_f32 (values descending, equal values by ascending index) on
//                         the dense row after mmrec_mask_f32: -0.0 sorts below +0.0, masked items are -1e10, and k beyond
//                         the unmasked items runs into them.
//   exact route           rows with more than SP_CAP products, more than SP_MCAP masked items or a non-finite sum are listed;
//                         the host then runs the unfused route on them (exact_rows.cuh) -- the same row kernel, the same mask
//                         value, mmrec_topk_rows_f32 -- and scatters the results.  Bit-identical by construction.
#include "batch_mask.cuh"
#include "exact_rows.cuh"
#include "select.cuh"

namespace mmrec {

constexpr int SP_THREADS = 256;
constexpr int SP_CAP = 2048;            // products (and exceptions) one CTA holds per row
constexpr int SP_MCAP = 2048;           // masked items one CTA sorts per row
constexpr size_t SP_SMEM = (size_t)SP_CAP * 8 + (size_t)SP_MCAP * 8 + (size_t)SP_CAP * 12;

struct SpCsr {
    const int32_t* ptr;
    const int32_t* col;
    const float* val;
};

// One warp: the dense score row of user u into out (zero-filled by the caller).
__device__ __forceinline__ void sparse_score_row(int64_t u, const SpCsr& R, const SpCsr& S, float* __restrict__ out, int lane) {
    const int p1 = __ldg(R.ptr + u + 1);
    for (int p = __ldg(R.ptr + u); p < p1; ++p) {
        const int i = __ldg(R.col + p);
        const float r = __ldg(R.val + p);
        const int e1 = __ldg(S.ptr + i + 1);
        for (int e = __ldg(S.ptr + i) + lane; e < e1; e += 32) {
            const int c = __ldg(S.col + e);
            out[c] = fmaf(r, __ldg(S.val + e), out[c]);
        }
        __syncwarp();
    }
}

// rows j < nb: user users[pos ? pos[j] : j] (or that batch row itself when users is NULL) into out + j * ldo
__global__ void __launch_bounds__(256) sparse_scores_kernel(int64_t nb, const int64_t* __restrict__ users, const int64_t* __restrict__ pos,
                                                            SpCsr R, SpCsr S, float* __restrict__ out, int64_t ldo) {
    const int64_t j = blockIdx.x * 8ll + (threadIdx.x >> 5);
    if (j >= nb) return;
    const int64_t b = pos ? pos[j] : j;
    sparse_score_row(users ? users[b] : b, R, S, out + j * ldo, threadIdx.x & 31);
}

// ---- the fused row -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SP_THREADS) sparse_topk_kernel(int64_t n_items, const int64_t* __restrict__ users, SpCsr R, SpCsr S,
                                                                 const int32_t* __restrict__ mptr, const int32_t* __restrict__ mitems, int k,
                                                                 int32_t* __restrict__ counter, int64_t* __restrict__ fb_pos,
                                                                 int64_t* __restrict__ out_idx, float* __restrict__ out_val) {
    extern __shared__ __align__(16) uint8_t sp_sm[];
    uint64_t* keyA = reinterpret_cast<uint64_t*>(sp_sm);          // (column, slot) keys, later the exceptions' composites
    uint64_t* keyB = keyA + SP_CAP;                                // masked items, ascending after the sort
    float* rr = reinterpret_cast<float*>(keyB + SP_MCAP);          // r per slot; later the sum per head slot, then masked flags
    float* ss = rr + SP_CAP;                                       // s per slot; later the sum per column
    int32_t* segcol = reinterpret_cast<int32_t*>(ss + SP_CAP);     // summed columns, ascending
    __shared__ unsigned long long s_base;
    __shared__ unsigned s_bad, s_ns, s_ne, s_nm;
    __shared__ unsigned wtot[SP_THREADS / 32];
    const int64_t b = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int64_t u = users ? users[b] : b;
    const int p0 = __ldg(R.ptr + u), L = __ldg(R.ptr + u + 1) - p0;
    const int m0 = mptr ? mptr[b] : 0, M = mptr ? mptr[b + 1] - m0 : 0;
    if (tid == 0) { s_base = 0; s_bad = M > SP_MCAP; s_ns = 0; s_ne = 0; s_nm = 0; }
    __syncthreads();
    auto to_exact = [&]() {
        if (tid == 0) fb_pos[atomicAdd(counter, 1)] = b;
    };
    if (s_bad) { to_exact(); return; }
    // 1. gather: slot = products of the earlier entries of R(u) + the position in this S row
    for (int t0 = 0; t0 < L; t0 += SP_THREADS) {
        const int t = t0 + tid;
        int len = 0, i = 0;
        float r = 0.f;
        if (t < L) {
            i = __ldg(R.col + p0 + t);
            r = __ldg(R.val + p0 + t);
            len = __ldg(S.ptr + i + 1) - __ldg(S.ptr + i);
        }
        int incl = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wtot[wid] = (unsigned)incl;
        __syncthreads();
        unsigned long long off = s_base + (unsigned)(incl - len);
        for (int w = 0; w < wid; ++w) off += wtot[w];
        if (t < L) {
            const int e0 = __ldg(S.ptr + i);
            for (int j = 0; j < len && off + j < (unsigned long long)SP_CAP; ++j) {
                const uint32_t slot = (uint32_t)(off + j);
                keyA[slot] = ~(((uint64_t)(uint32_t)__ldg(S.col + e0 + j) << 32) | slot);     // complement: the sort is descending
                rr[slot] = r;
                ss[slot] = __ldg(S.val + e0 + j);
            }
        }
        __syncthreads();
        if (tid == 0) {
            unsigned long long tot = 0;
            for (int w = 0; w < SP_THREADS / 32; ++w) tot += wtot[w];
            s_base += tot;
        }
        __syncthreads();
        if (s_base > (unsigned long long)SP_CAP) break;
    }
    if (s_base > (unsigned long long)SP_CAP) { to_exact(); return; }
    const int n = (int)s_base;
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int c = n + tid; c < n2; c += SP_THREADS) keyA[c] = 0;    // (pads: after every real key)
    bitonic_desc(keyA, n2);                                        // keyA[0 .. n): (column, slot) ascending
    auto col_of = [&](int p) { return (uint32_t)(~keyA[p] >> 32); };
    auto slot_of = [&](int p) { return (uint32_t)~keyA[p]; };
    // 2. one thread per column: its products in R order
    for (int p = tid; p < n; p += SP_THREADS) {
        const uint32_t c = col_of(p);
        if (p > 0 && col_of(p - 1) == c) continue;
        float acc = 0.f;
        for (int q = p; q < n && col_of(q) == c; ++q) {
            const uint32_t sl = slot_of(q);
            acc = fmaf(rr[sl], ss[sl], acc);
        }
        rr[slot_of(p)] = acc;                                      // (the head's slot belongs to this column only)
        if (!(fabsf(acc) < INFINITY)) s_bad = 1;
    }
    __syncthreads();
    if (s_bad) { to_exact(); return; }
    // 3. compact the columns in order: segcol[si], ss[si]
    for (int p0c = 0; p0c < n; p0c += SP_THREADS) {
        const int p = p0c + tid;
        const bool head = p < n && (p == 0 || col_of(p - 1) != col_of(p));
        const unsigned bal = __ballot_sync(0xffffffffu, head);
        if (lane == 0) wtot[wid] = __popc(bal);
        __syncthreads();
        unsigned off = s_ns;
        for (int w = 0; w < wid; ++w) off += wtot[w];
        if (head) {
            const unsigned si = off + __popc(bal & ((1u << lane) - 1u));
            segcol[si] = (int32_t)col_of(p);
            ss[si] = rr[slot_of(p)];
        }
        __syncthreads();
        if (tid == 0) {
            unsigned tot = 0;
            for (int w = 0; w < SP_THREADS / 32; ++w) tot += wtot[w];
            s_ns += tot;
        }
        __syncthreads();
    }
    const int NS = (int)s_ns;
    // 4. the row's masked items, ascending (duplicates adjacent); masked flags of the columns
    for (int j = tid; j < NS; j += SP_THREADS) rr[j] = 0.f;
    int m2 = 1;
    while (m2 < M) m2 <<= 1;
    for (int j = tid; j < m2; j += SP_THREADS) {
        uint64_t v = 0;
        if (j < M) {
            const int32_t it = mitems[m0 + j];
            if (it >= 0 && (int64_t)it < n_items) { v = ~(uint64_t)(uint32_t)it; atomicAdd(&s_nm, 1u); }
        }
        keyB[j] = v;
    }
    bitonic_desc(keyB, m2);
    const int Mv = (int)s_nm;
    const uint64_t KEY_MASKED = (uint64_t)float_key(-1e10f) << 32;   // trainer.py:307's value
    for (int j = tid; j < Mv; j += SP_THREADS) {
        if (j > 0 && keyB[j] == keyB[j - 1]) continue;
        const uint32_t it = (uint32_t)~keyB[j];
        int lo = 0, hi = NS;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)segcol[mid] < it) lo = mid + 1; else hi = mid;
        }
        if (lo < NS && (uint32_t)segcol[lo] == it) rr[lo] = 1.f;
        const unsigned e = atomicAdd(&s_ne, 1u);
        if (e < (unsigned)SP_CAP) keyA[e] = KEY_MASKED | (uint32_t)~it;
    }
    __syncthreads();
    // 5. the unmasked columns whose sum is not +0.0
    for (int si = tid; si < NS; si += SP_THREADS) {
        if (rr[si] == 0.f && __float_as_uint(ss[si]) != 0u) {
            const unsigned e = atomicAdd(&s_ne, 1u);
            if (e < (unsigned)SP_CAP) keyA[e] = ((uint64_t)float_key(ss[si]) << 32) | (uint32_t)~(uint32_t)segcol[si];
        }
    }
    __syncthreads();
    const int NE = (int)s_ne;
    if (NE > SP_CAP) { to_exact(); return; }
    int e2 = 1;
    while (e2 < NE) e2 <<= 1;
    for (int c = NE + tid; c < e2; c += SP_THREADS) keyA[c] = 0;
    bitonic_desc(keyA, e2);
    // 6. the exceptions above +0.0 (A of them), the +0.0 items (Z), the rest of the exceptions
    int lo = 0, hi = NE;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((uint32_t)(keyA[mid] >> 32) > 0x80000000u) lo = mid + 1; else hi = mid;    // float_key(+0.0) = 0x80000000
    }
    const int64_t A = lo, Z = n_items - NE;
    int64_t* oi = out_idx + b * k;
    float* ov = out_val + b * k;
    for (int t = tid; t < k; t += SP_THREADS) {
        if (t < A || t >= A + Z) {
            const uint64_t c = keyA[t < A ? t : t - Z];
            oi[t] = (int64_t)(uint32_t)~(uint32_t)c;
            ov[t] = key_float((uint32_t)(c >> 32));
        }
    }
    if (tid == 0) {
        const int64_t t1 = (int64_t)k < A + Z ? (int64_t)k : A + Z;
        int pc = 0, pm = 0;
        int64_t j = 0;
        for (int64_t t = A; t < t1; ++t, ++j) {
            for (;; ++j) {                                         // the next item that is not an exception
                while (pc < NS && (int64_t)segcol[pc] < j) ++pc;
                while (pm < Mv && (int64_t)(uint32_t)~keyB[pm] < j) ++pm;
                const bool masked = pm < Mv && (int64_t)(uint32_t)~keyB[pm] == j;
                const bool nonzero = pc < NS && (int64_t)segcol[pc] == j && __float_as_uint(ss[pc]) != 0u;
                if (!masked && !nonzero) break;
            }
            oi[t] = j;
            ov[t] = 0.f;
        }
    }
}

__global__ void sp_mask_rows_kernel(int64_t c, const int64_t* __restrict__ pos, const int32_t* __restrict__ mptr,
                                    const int32_t* __restrict__ mitems, int64_t n_items, float* __restrict__ S) {
    const int64_t j = blockIdx.x;
    if (j >= c || !mptr) return;
    const int64_t b = pos[j];
    for (int q = mptr[b] + threadIdx.x; q < mptr[b + 1]; q += blockDim.x) {
        const int32_t it = mitems[q];
        if (it >= 0 && (int64_t)it < n_items) S[j * n_items + it] = -1e10f;              // trainer.py:307
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct SpPlan {
    int64_t s_rows;
    size_t off_mask, off_cnt, off_fb, off_ex, total;
};

static SpPlan sp_plan(int64_t B, int64_t n_items, int64_t mask_nnz, int k) {
    SpPlan P;
    P.s_rows = exact_block_rows(n_items, B > 0 ? B : 1);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes > 0 ? bytes : 1, 256); return o; };
    P.off_mask = take(batch_mask(nullptr, mask_nnz, nullptr, nullptr, B, 0, 0).bytes);
    P.off_cnt = take(4);
    P.off_fb = take((size_t)B * 8);
    P.off_ex = take(exact_rows_bytes(P.s_rows, n_items, k));
    P.total = off + 256;
    return P;
}

static int64_t g_sparse_topk_fallback_rows = -1;

static int sp_scores_rows(int64_t nb, const int64_t* users, const int64_t* pos, const SpCsr& R, const SpCsr& S, int64_t n_items,
                          float* out, int64_t ldo, cudaStream_t stream) {
    MMREC_CUDA(cudaMemset2DAsync(out, (size_t)ldo * 4, 0, (size_t)n_items * 4, (size_t)nb, stream));
    sparse_scores_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, stream>>>(nb, users, pos, R, S, out, ldo);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_sparse_scores_f32(int64_t B, const int64_t* users, int64_t n_items, const int32_t* r_ptr, const int32_t* r_col,
                                       const float* r_val, const int32_t* s_ptr, const int32_t* s_col, const float* s_val, float* out,
                                       int64_t ldo, void* stream_) {
    MMREC_CHECK_ARG(B >= 0 && n_items >= 1 && n_items < (1ll << 31), "sparse_scores: need B >= 0 and 1 <= n_items < 2^31");
    if (B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(r_ptr && r_col && r_val && s_ptr && s_col && s_val && out && ldo >= n_items,
                    "sparse_scores: null pointer or ldo < n_items");
    const SpCsr R{r_ptr, r_col, r_val}, S{s_ptr, s_col, s_val};
    return sp_scores_rows(B, users, nullptr, R, S, n_items, out, ldo, (cudaStream_t)stream_);
}

extern "C" size_t mmrec_sparse_score_topk_workspace_bytes(int64_t B, int64_t n_items, int64_t mask_nnz, int k) {
    if (B < 0 || n_items < 1 || mask_nnz < 0 || k < 1 || k > TOPK_MAXK || k > n_items) return 0;
    return sp_plan(B, n_items, mask_nnz, k).total;
}

extern "C" int64_t mmrec_debug_sparse_topk_fallback_rows(void) { return g_sparse_topk_fallback_rows; }

extern "C" int mmrec_sparse_score_topk_f32(int64_t B, const int64_t* users, int64_t n_items, const int32_t* r_ptr, const int32_t* r_col,
                                           const float* r_val, const int32_t* s_ptr, const int32_t* s_col, const float* s_val,
                                           int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int k,
                                           int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(B >= 0 && n_items >= 1 && n_items < (1ll << 31) && mask_nnz >= 0, "sparse_score_topk: bad sizes");
    MMREC_CHECK_ARG(k >= 1 && k <= TOPK_MAXK && k <= n_items, "sparse_score_topk: need 1 <= k <= min(%d, n_items)", TOPK_MAXK);
    if (B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(r_ptr && r_col && r_val && s_ptr && s_col && s_val && out_idx && out_val, "sparse_score_topk: null pointer");
    MMREC_CHECK_ARG(mask_nnz == 0 || (mask_rows && mask_cols), "sparse_score_topk: null mask");
    const SpPlan P = sp_plan(B, n_items, mask_nnz, k);
    char* base = (char*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    if (!ws || ws_bytes < P.total) {
        set_error("sparse_score_topk: workspace %zu < %zu", ws_bytes, P.total);
        return MMREC_EWORKSPACE;
    }
    const BatchMask M = batch_mask(base + P.off_mask, mask_nnz, mask_rows, mask_cols, B, 0, n_items);
    int32_t* counter = (int32_t*)(base + P.off_cnt);
    int64_t* fb = (int64_t*)(base + P.off_fb);
    const SpCsr R{r_ptr, r_col, r_val}, S{s_ptr, s_col, s_val};
    if (mask_nnz > 0) {
        int rc = batch_mask_build(M, stream);
        if (rc) return rc;
    }
    const int32_t* mp = mask_nnz > 0 ? M.ptr : nullptr;
    if (int rc = set_smem_once<sparse_topk_kernel>((int)SP_SMEM)) return rc;
    MMREC_CUDA(cudaMemsetAsync(counter, 0, 4, stream));
    sparse_topk_kernel<<<(unsigned)B, SP_THREADS, SP_SMEM, stream>>>(n_items, users, R, S, mp, M.items, k, counter, fb, out_idx, out_val);
    MMREC_LAUNCH_CHECK();
    const int64_t cnt = read_count(counter, stream);
    if (cnt < 0) return (int)cnt;
    int rc = exact_rows_topk(cnt, fb, n_items, k, P.s_rows, base + P.off_ex, out_idx, out_val, stream, [&](int64_t c0, int64_t c, float* Sd) {
        int rc2 = sp_scores_rows(c, users, fb + c0, R, S, n_items, Sd, n_items, stream);
        if (rc2 || !mp) return rc2;
        sp_mask_rows_kernel<<<(unsigned)c, 256, 0, stream>>>(c, fb + c0, mp, M.items, n_items, Sd);
        MMREC_LAUNCH_CHECK();
        return MMREC_OK;
    });
    if (rc) return rc;
    g_sparse_topk_fallback_rows = cnt;
    return MMREC_OK;
}
