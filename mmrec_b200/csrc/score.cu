// K3: full-catalog scoring  S = U[users] I^T  (src/models/freedom.py:216-220) and its fusion with the
// trainer's mask + top-k (src/common/trainer.py:304-309).
//
// Two arithmetic paths share the entry points:
//   * exact fp32 on CUDA cores (gemm_simt.cuh): one fmaf chain per score, k ascending -- bit-faithful;
//   * wgmma tensor cores with the 3xTF32 split (score_tc.cu) when the shape fits its tiles; selected by
//     mmrec_score_set_path() / env MMREC_SCORE_PATH = "simt" | "tc" (default: tc where supported).
// mmrec_score_topk_f32 processes the users in row blocks whose score block stays L2-resident
// (B_blk x n_items x 4 B <= 64 MiB), so the B x n_items matrix the reference materialises in HBM
// (115 MB per 4096 users at 7k items, 16 GB at 1M items) never exists.
#include <stdlib.h>
#include <string.h>

#include "gemm_simt.cuh"

namespace mmrec {
// implemented in score_tc.cu; returns 1 if it handled the call, 0 if the shape is unsupported, <0 on error
int score_tc(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items, const float* Ie,
             int64_t ldi, int d, float* S, int64_t ldS, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t score_tc_workspace_bytes(int64_t B, int64_t n_items, int d);
// score_cf.cu (certified-filter fused path): 1 handled, 0 unsupported shape / workspace
int score_cf(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items, const float* Ie, int64_t ldi,
             int d, const void* cat, int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int k, int64_t item_offset,
             int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t score_cf_workspace_bytes(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat);
size_t cf_catalog_bytes(int64_t n_items, int d);
int cf_catalog_pack(int64_t n_items, const float* Ie, int64_t ldi, int d, void* cat, size_t cat_bytes, cudaStream_t stream);
int score_cf_timing(float* us, int cap);
int64_t score_cf_fallback_rows(const void* ws, int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat);
int score_cf_scratch(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, bool with_cat, int64_t* out, int cap);

int mask_apply(int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int64_t row0, int64_t B,
               int64_t n_items, int64_t item_offset, float* S, int64_t ldS, cudaStream_t stream);

// -1 unset | 0 simt: exact fp32 CUDA cores | 1 tc: wgmma GEMM -> L2-resident score block -> mask -> streaming top-k
//  2 auto (default): fused wherever its shape rules allow (enough item groups for the certified threshold), else tc
//  3 fused: the certified-filter path of score_cf.cu (wgmma f16 filter + exact fp32 finalists, no score matrix at all)
static int g_score_path = -1;
static int score_path() {
    if (g_score_path < 0) {
        const char* e = getenv("MMREC_SCORE_PATH");
        g_score_path = 2;
        if (e && strcmp(e, "simt") == 0) g_score_path = 0;
        if (e && strcmp(e, "tc") == 0) g_score_path = 1;
        if (e && strcmp(e, "fused") == 0) g_score_path = 3;
    }
    return g_score_path;
}
static bool want_fused(int64_t n_items) { (void)n_items; return score_path() >= 2; }
}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_score_set_path(int path) { g_score_path = path < 0 ? 0 : (path > 3 ? 3 : path); return MMREC_OK; }

extern "C" size_t mmrec_score_workspace_bytes(int64_t B, int64_t n_items, int d) {
    return score_tc_workspace_bytes(B, n_items, d) + 256;
}

extern "C" int mmrec_score_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items,
                               const float* Ie, int64_t ldi, int d, float* S, int64_t ldS, void* ws, size_t ws_bytes,
                               void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(B >= 0 && n_items >= 0 && d >= 1, "score: bad sizes");
    if (B == 0 || n_items == 0) return MMREC_OK;
    MMREC_CHECK_ARG(Ue && Ie && S && ldu >= d && ldi >= d && ldS >= n_items, "score: null pointer or bad leading dimension");
    if (score_path() >= 1) {
        int r = score_tc(B, users, Ue, ldu, n_items, Ie, ldi, d, S, ldS, ws, ws_bytes, stream);
        if (r != 0) return r < 0 ? r : MMREC_OK;
    }
    GemmNT p;
    p.A = Ue; p.lda = ldu; p.a_idx = users; p.M = B;
    p.B = Ie; p.ldb = ldi; p.N = n_items; p.K = d; p.bias = nullptr; p.C = S; p.ldc = ldS; p.l2_normalize = 0;
    return launch_gemm_nt<128, 128, 8, 8>(p, stream);
}

static int64_t score_block_rows(int64_t B, int64_t n_items) {
    const int64_t budget = 64ll << 20;
    int64_t rows = budget / (n_items * 4);
    if (rows < 128) rows = 128;
    rows = rows / 128 * 128;
    return rows < B ? rows : B;
}

extern "C" size_t mmrec_score_topk_workspace_bytes(int64_t B, int64_t n_items, int d, int k) {
    (void)d; (void)k;
    if (B <= 0 || n_items <= 0) return 256;
    const int64_t rows = score_block_rows(B, n_items);
    const size_t unfused = align_up((size_t)rows * (size_t)((n_items + 3) / 4 * 4) * sizeof(float) + 256, 1024) +
                           mmrec_score_workspace_bytes(rows, n_items, d);
    const size_t fused = score_cf_workspace_bytes(B, n_items, d, k, B * 64 + 4096, true);   // mask_nnz is not known here
    return unfused > fused ? unfused : fused;
}

extern "C" size_t mmrec_catalog_bytes(int64_t n_items, int d) { return cf_catalog_bytes(n_items, d); }

extern "C" int mmrec_catalog_pack_f32(int64_t n_items, const float* Ie, int64_t ldi, int d, void* cat, size_t cat_bytes, void* stream_) {
    MMREC_CHECK_ARG(n_items >= 1 && d >= 1 && Ie && ldi >= d, "catalog_pack: bad sizes / null pointer");
    MMREC_CHECK_ARG(cf_catalog_bytes(n_items, d) > 0, "catalog_pack: d > 128 has no tensor-core path");
    return cf_catalog_pack(n_items, Ie, ldi, d, cat, cat_bytes, (cudaStream_t)stream_);
}

extern "C" int mmrec_debug_cf_timing(float* us, int cap) { return score_cf_timing(us, cap); }

extern "C" int64_t mmrec_debug_fused_fallback_rows(const void* ws, int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, int with_cat) {
    return score_cf_fallback_rows(ws, B, n_items, d, k, mask_nnz, with_cat != 0);
}

extern "C" int mmrec_debug_cf_scratch(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, int with_cat, int64_t* out, int cap) {
    MMREC_CHECK_ARG(out != nullptr || cap <= 0, "debug_cf_scratch: null output");
    return score_cf_scratch(B, n_items, d, k, mask_nnz, with_cat != 0, out, cap);
}

extern "C" int mmrec_score_topk_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items,
                                    const float* Ie, int64_t ldi, int d, int64_t mask_nnz, const int64_t* mask_rows,
                                    const int64_t* mask_cols, int k, int64_t item_offset, int64_t* out_idx,
                                    float* out_val, void* ws, size_t ws_bytes, void* stream_) {
    return mmrec_score_topk_cat_f32(B, users, Ue, ldu, n_items, Ie, ldi, d, nullptr, mask_nnz, mask_rows, mask_cols, k, item_offset, out_idx,
                                    out_val, ws, ws_bytes, stream_);
}

extern "C" int mmrec_score_topk_cat_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu, int64_t n_items,
                                        const float* Ie, int64_t ldi, int d, const void* cat, int64_t mask_nnz,
                                        const int64_t* mask_rows, const int64_t* mask_cols, int k, int64_t item_offset,
                                        int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, void* stream_) {
    MMREC_CHECK_ARG(B >= 0 && n_items >= 1 && d >= 1 && k >= 1, "score_topk: bad sizes");
    if (B == 0) return MMREC_OK;
    MMREC_CHECK_ARG(Ue && Ie && out_idx && out_val && ldu >= d && ldi >= d, "score_topk: null pointer or bad leading dimension");
    MMREC_CHECK_ARG(mask_nnz == 0 || (mask_rows && mask_cols), "score_topk: mask pointers missing");
    const size_t need = mmrec_score_topk_workspace_bytes(B, n_items, d, k);
    if (!ws || ws_bytes < need) {
        set_error("score_topk: workspace %zu < %zu", ws_bytes, need);
        return MMREC_EWORKSPACE;
    }
    if (want_fused(n_items)) {
        int r = score_cf(B, users, Ue, ldu, n_items, Ie, ldi, d, cat, mask_nnz, mask_rows, mask_cols, k, item_offset, out_idx,
                         out_val, ws, ws_bytes, (cudaStream_t)stream_);
        if (r != 0) return r < 0 ? r : MMREC_OK;
    }
    float* S = (float*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    const int64_t ldS = (n_items + 3) / 4 * 4;
    const int64_t rows = score_block_rows(B, n_items);
    const size_t s_bytes = align_up((size_t)rows * (size_t)ldS * sizeof(float) + 256, 1024);
    void* ws2 = (char*)ws + s_bytes;
    const size_t ws2_bytes = ws_bytes - s_bytes;
    for (int64_t r0 = 0; r0 < B; r0 += rows) {
        const int64_t nb = (B - r0) < rows ? (B - r0) : rows;
        int rc = mmrec_score_f32(nb, users ? users + r0 : nullptr, users ? Ue : Ue + r0 * ldu, ldu, n_items, Ie, ldi, d, S,
                                 ldS, ws2, ws2_bytes, stream_);
        if (rc) return rc;
        if (mask_nnz > 0) {
            // mask rows are positions in the whole batch: the kernel shifts by r0 and ignores rows outside [0, nb)
            rc = mask_apply(mask_nnz, mask_rows, mask_cols, r0, nb, n_items, item_offset, S, ldS, (cudaStream_t)stream_);
            if (rc) return rc;
        }
        rc = mmrec_topk_rows_f32(nb, n_items, S, ldS, k, item_offset, out_idx + r0 * k, out_val + r0 * k, stream_);
        if (rc) return rc;
    }
    return MMREC_OK;
}
