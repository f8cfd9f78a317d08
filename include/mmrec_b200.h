/* mmrec_b200 -- C ABI of the H100-native hot path of MMRec.
 *
 * The reference (enoche/MMRec, /root/reference) is pure Python on PyTorch; it has no FFI of
 * its own.  Its "plugin boundary" is the model class contract of
 * src/common/abstract_recommender.py:10-52,71-103, and the hot path below that boundary is the
 * set of PyTorch library calls listed next to each entry point.  This header is what a
 * maintainer binds (ctypes stub in INTEGRATION.md) to replace exactly those calls.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (normally a torch tensor); the
 *    library never allocates or frees device memory: scratch is passed in as `ws`, sized by the
 *    matching *_workspace_bytes() call;
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*; 0 = legacy default);
 *  - return value 0 = ok, negative = MMREC_E* below; mmrec_last_error() gives the message
 *    (thread-local);
 *  - all matrices are row-major; floating point is fp32 (the reference computes in fp32),
 *    CSR indices are int32, COO indices / gather indices / result indices are int64 as in the
 *    reference's tensors.
 */
#ifndef MMREC_B200_H
#define MMREC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMREC_OK 0
#define MMREC_EINVAL (-1)      /* bad argument (null pointer, negative size, unsupported d or k) */
#define MMREC_EWORKSPACE (-2)  /* ws_bytes smaller than *_workspace_bytes() */
#define MMREC_ECUDA (-3)       /* a CUDA runtime call failed; see mmrec_last_error() */
#define MMREC_EUNSUPPORTED (-4)/* device is not sm_90 (the library carries sm_90a code only) */

#define MMREC_ABI_VERSION 4

int mmrec_abi_version(void);
const char* mmrec_last_error(void);
/* 0 if the current device can run this library (compute capability 9.x), else MMREC_EUNSUPPORTED */
int mmrec_device_check(void);
/* Kernels of this library launched by the calling process so far (every launch site counts itself; library
 * primitives -- CUB sort/scan, memsets -- are not counted).  bench.py reports the difference over its timed region. */
int64_t mmrec_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * K1c  COO -> CSR.   Replaces the per-call `coalesce()` + COO->CSR conversion hidden inside every
 * `torch.sparse.mm(adj, x)` on the path (src/models/freedom.py:167,172; bm3.py:90;
 * mgcn.py:162,172,176,180,184; layergcn.py:131; lightgcn.py:120; common/encoders.py:99,122).
 * The reference's matrices arrive un-coalesced and, for FREEDOM's mm_adj, with duplicate
 * coordinates that must add (freedom.py:74): duplicates are summed in input order (stable sort),
 * which is what coalesce() does.  Output rows are sorted by column.
 *   row/col  int64[nnz]; val fp32[nnz] or NULL (= all ones)
 *   rowptr   int32[n_rows+1]; colidx int32[nnz]; vals fp32[nnz]  (first nnz_out[0] entries valid)
 *   nnz_out  int64[1] on the device: number of entries after merging duplicates
 * ------------------------------------------------------------------------------------------- */
size_t mmrec_csr_from_coo_workspace_bytes(int64_t nnz, int64_t n_rows);
int mmrec_csr_from_coo(int64_t nnz, const int64_t* row, const int64_t* col, const float* val,
                       int64_t n_rows, int64_t n_cols, int sum_duplicates,
                       int32_t* rowptr, int32_t* colidx, float* vals, int64_t* nnz_out,
                       void* ws, size_t ws_bytes, void* stream);

/* Work plan for mmrec_spmm_run_f32.  A task is a whole row or, for rows longer than `seg` non-zeros, one segment of it.
 * Tasks longer than `light_max` are run by a whole CTA (its lane groups split the task and reduce through shared
 * memory), the others by one lane group each -- the power-law item rows neither serialise on one warp nor sit on
 * the critical path.
 *   tasks      int32[4 * max_tasks]  {row, begin, end, split_id(-1 = whole row)}, sorted longest first, so the
 *                                    CTA-run tasks are the first counts[4] entries
 *   split_rows int32[4 * max_split]  {first_slot, n_seg, row_begin, seg}
 *   counts     int64[8] on the device: {n_tasks, n_split_rows, n_slots, longest_row, n_cta_tasks, 0, 0, 0}
 * max_tasks = n_rows + nnz / seg + 1 and max_split = nnz / seg + 1 are always enough. */
size_t mmrec_spmm_plan_workspace_bytes(int64_t n_rows, int64_t max_tasks);
int mmrec_spmm_plan(int64_t n_rows, const int32_t* rowptr, int seg, int light_max, int64_t max_tasks,
                    int32_t* tasks, int32_t* split_rows, int64_t* counts,
                    void* ws, size_t ws_bytes, void* stream);

/* Per-edge symmetric normalisation of a bipartite edge list, fp32, computed like
 * src/models/freedom.py:145-154 (`_normalize_adj_m`): deg counted exactly, then
 * val[e] = rsqrt(deg_u[u] + eps) * rsqrt(deg_i[i] + eps) with IEEE sqrt and divide.
 *   ws: int32[n_users + n_items] */
size_t mmrec_bipartite_norm_workspace_bytes(int64_t n_users, int64_t n_items);
int mmrec_bipartite_norm_f32(int64_t n_edges, const int64_t* users, const int64_t* items,
                             int64_t n_users, int64_t n_items, float eps, float* vals,
                             void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K1  CSR SpMM with fused layer-combination epilogue.   Replaces `torch.sparse.mm(adj, x)` and the
 * `stack(...).mean(dim=1)` / `+ h` that follow it (src/models/freedom.py:164-178, bm3.py:84-95,
 * lightgcn.py:115-128, mgcn.py:157-185, layergcn.py:125-138); its backward is the same call on the
 * transposed CSR (autograd of torch.sparse.mm, triggered at src/common/trainer.py:185).
 *
 * One mmrec_spmm_op describes one product of the n_rows x n_cols CSR (rowptr, colidx, vals) with X, d columns wide:
 *
 *   y[r,:]   = sum_j w_j * X[colidx[j], :]               j in rowptr[r] .. rowptr[r+1], w_j = vals[j]
 *   if keep_bits: only the entries whose keep bit is set take part, w_j = fl(vals[j] * keep_scale)
 *   if gate_ref:  y[r,:] *= cos(y[r,:], gate_ref[r,:])   (LayerGCN, layergcn.py:132-133)
 *   if Y:         Y[r,:] = y[r,:]  (y_accumulate != 0: Y[r,:] += y[r,:])
 *   if acc_out:   acc_out[r,:] = ((acc_in ? acc_in[r,:] : 0) + y[r,:]) / acc_div
 *                 (+ post[r - post_row0,:] for r >= post_row0 when post is set, after the division)
 *
 *  - acc_in may alias acc_out.  Every matrix is row-major with the leading dimension beside it (in floats, >= d).
 *  - Work plan: tasks/n_tasks/n_cta_tasks/split_rows/counters/partial come from mmrec_spmm_plan (counters:
 *    int32[n_split_rows], zero on entry and zero again on exit; partial: fp32[n_slots * d]); tasks == NULL selects one
 *    warp per row.  Summation order is fixed, so the result is bit-reproducible run to run.
 *  - y_accumulate: for graphs whose X does not fit the L2 the matrix is cut into column panels whose share of X does; the
 *    panels are multiplied one after the other and add up in Y, so every row of X is fetched from HBM once per layer
 *    instead of once per non-zero (ops.PanelCSR).  The running-sum epilogue sees one panel's y only, so the division
 *    belongs to the last panel.  Not with the gate (MMREC_EINVAL).
 *  - keep_bits uint32[ceil(nnz / 32)], bit e (word e / 32, bit e % 32) for CSR position e (mmrec_edge_keep_bits):
 *    `torch.sparse.mm(sparse_dropout(A, rate), X)` of src/common/encoders.py:77-88,99 without building the dropped matrix.
 *    A dropped entry loads nothing and adds nothing, so the result equals the product with the compacted matrix and the
 *    values fl(v * keep_scale), up to the position of the segment boundaries of split rows.  d in {32, 64, 128, 256} and
 *    16-byte aligned operands, and neither the gate nor y_accumulate, else MMREC_EUNSUPPORTED.
 *  - Second row blocks (nullable): X row c is X_hi[c - x_split, :] for c >= x_split, acc_in row r is
 *    acc_in_hi[r - acc_in_split, :] for r >= acc_in_split (acc_in and acc_out must be set) -- layer 1 of a propagation
 *    reads [users; items] straight from the two embedding tables, with the same bits as from their concatenation.
 *
 * mmrec_spmm_run_f32 runs n_ops products in order on `stream`.
 *  - One op without X_hi, acc_in_hi, post or sync_before, cooperative == 0: with keep_bits, the masked kernel.  Otherwise
 *    d in {32, 64, 128, 256} with 16-byte aligned operands runs the vectorised kernel (the lane override applies), as do
 *    d in {96, 192, 384} = 3 x {32, 64, 128} (several d-wide operands side by side, SLMRec's three views: three float4
 *    per lane on the lanes the width d/3 uses; without the gate, every d/3-wide column block of the result is
 *    bit-identical to the width-d/3 product of that block; no lane override).  Any other d >= 1 or alignment runs the
 *    generic kernel.
 *  - Otherwise the ops are the SpMMs of one propagation (src/models/freedom.py:164-178: n_ui_layers products with A_hat,
 *    the item-item product, the layer mean and `+ h`), at most 8, run by the chained kernel: every op needs its work
 *    plan; d in {32, 64, 128, 256}, 16-byte aligned operands, no lane override, no gate, keep bits or y_accumulate --
 *    otherwise MMREC_EUNSUPPORTED and the caller runs the ops one by one.  cooperative != 0: one persistent cooperative
 *    launch, the ops run in order on one resident grid with a grid-wide barrier before every op whose `sync_before` is
 *    set (= it reads what an earlier op wrote).  cooperative == 0: the ops up to the next `sync_before` op share one
 *    ordinary launch (ops that do not read each other's output, such as FREEDOM's item-item product and layer 1 on
 *    A_hat); each `sync_before` op starts a new launch on the stream.  Ops of one launch must not share a work plan's
 *    counters / partial buffer.
 * ------------------------------------------------------------------------------------------- */
/* tuning knob: lanes that cooperate on one row (0 = default min(32, d/4); a power of two, d/(4*lanes) float4 per lane;
 * d in {32, 64, 128, 256} only) */
int mmrec_spmm_set_lanes(int lanes_per_row);
typedef struct {
    int64_t n_rows, n_cols;
    const int32_t* rowptr; const int32_t* colidx; const float* vals;
    const int32_t* tasks; int64_t n_tasks, n_cta_tasks;              /* tasks == NULL: one warp per row */
    const int32_t* split_rows; int32_t* counters; float* partial;
    const float* X; int64_t ldx;
    const float* X_hi; int64_t ldx_hi, x_split;                      /* nullable: second row block of X */
    float* Y; int64_t ldy; int y_accumulate;                         /* Y nullable */
    const float* acc_in; float* acc_out; int64_t ldacc; float acc_div;
    const float* acc_in_hi; int64_t ldacc_in_hi, acc_in_split;       /* nullable */
    const float* gate_ref; int64_t ldgate;                           /* nullable: LayerGCN's cosine gate */
    const float* post; int64_t ldpost, post_row0;                    /* nullable */
    const uint32_t* keep_bits; float keep_scale;                     /* nullable: edge-keep mask */
    int sync_before;
} mmrec_spmm_op;
int mmrec_spmm_run_f32(int d, int n_ops, const mmrec_spmm_op* ops, int cooperative, void* stream);

/* The keep bits of one `sparse_dropout` draw (src/common/encoders.py:77-88): draw j of `torch.rand(nnz)` belongs to the
 * reference's j-th stored entry, which is CSR position e with draw_of[e] = j.  Position e is kept iff
 * floorf(keep_prob + draws[draw_of[e]]) != 0, one IEEE fp32 add (keep_prob = float32(1 - rate), as torch adds it).
 *   keep_bits   uint32[ceil(nnz / 32)]  the forward's bits, CSR order (mmrec_spmm_op.keep_bits)
 *   mirror      int32[nnz] (nullable)   position of (c, r) for the entry (r, c) of a structurally symmetric CSR
 *   keep_bits_t uint32[ceil(nnz / 32)]  (nullable, needs mirror) bit e = bit mirror[e] of keep_bits: the dropped matrix's
 *                                       transpose on the same CSR when its values are symmetric (the backward)
 * Bits past nnz in the last word are 0. */
int mmrec_edge_keep_bits(int64_t nnz, const float* draws, float keep_prob, const int32_t* draw_of, const int32_t* mirror,
                         uint32_t* keep_bits, uint32_t* keep_bits_t, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K2  fused gather -> linear(+bias) -> optional row L2-normalise.   Replaces
 * `self.image_trs(self.image_embedding.weight)[items]` (src/models/freedom.py:205-209,
 * bm3.py:102-104, mgcn.py:148-150) and `F.normalize(MLP(features))` (mmgcn.py:165-168).
 *   Y[n,:] = table[idx ? idx[n] : n, :] @ W^T + bias      table [n_table, F], W [d, F], bias [d]|NULL
 *   l2_normalize: Y[n,:] /= max(||Y[n,:]||_2, 1e-12)
 * Two arithmetic paths: wgmma 3xTF32 with the table split in-kernel (default when ws is given and d <= 256;
 * ws from mmrec_project_workspace_bytes holds the re-tiled weights and the K-split partials) and exact fp32 on CUDA
 * cores (ws == NULL, or mmrec_project_set_path(0) / env MMREC_PROJECT_PATH=simt).
 * ------------------------------------------------------------------------------------------- */
int mmrec_project_set_path(int tensor_core);
size_t mmrec_project_workspace_bytes(int64_t n_out, int64_t F, int d);
int mmrec_project_f32(int64_t n_out, const int64_t* idx, const float* table, int64_t n_table, int64_t F,
                      const float* W, const float* bias, int d, int l2_normalize,
                      float* Y, int64_t ldy, void* ws, size_t ws_bytes, void* stream);

/* measurement aid (tools/probe_mma.py): cycles of `iters` back-to-back wgmma (one warpgroup, operands in shared memory,
 * K-major no swizzle, M = 64, K = 32 bytes) per CTA, one CTA per SM; kind 0 = tf32, 1 = bf16 */
int mmrec_debug_mma_rate(int kind, int N, int iters, int distinct, long long* cycles_per_cta, void* stream);

/* measurement aid (tools/probe_stream.py): stream a [n_rows, F] fp32 table the way K2 does -- every CTA visits R rows
 * round-robin for burst_bytes contiguous bytes each, R * burst_bytes = 64 KB in flight per CTA -- to see what the DRAM
 * delivers for a given burst length */
int mmrec_debug_stream_probe(const float* table, int64_t n_rows, int64_t F, int R, int burst_bytes, int ctas_per_sm, float* sink,
                             void* stream);

/* ---------------------------------------------------------------------------------------------
 * K3  full-catalog scoring, train-positive mask and per-user top-k.   Replaces
 * `torch.matmul(u_embeddings, restore_item_e.transpose(0, 1))` (src/models/freedom.py:219,
 * bm3.py:153, mgcn.py:262, layergcn.py:185, lightgcn.py:162, mmgcn.py:104) and
 * `scores[mask[0], mask[1]] = -1e10; torch.topk(scores, k)` (src/common/trainer.py:304-309).
 *
 * mmrec_score_f32:    S[b, i] = <Ue[users ? users[b] : b, :], Ie[i, :]>            S [B, ldS]
 *                     ws (mmrec_score_workspace_bytes) holds the re-tiled hi/lo operands of the tensor-core
 *                     path; ws == NULL selects the CUDA-core fp32 path.
 * mmrec_mask_f32:     S[mask_rows[j], mask_cols[j] - item_offset] = -1e10 for columns inside
 *                     [item_offset, item_offset + n_items)
 * mmrec_topk_rows_f32: out_idx/out_val [B, k], descending value, ties -> lower index, index
 *                     reported as column + item_offset.  1 <= k <= 1024, k <= n_items.
 * mmrec_score_topk_f32: all three fused, scores never materialised in HBM (score_cf.cu): the tensor cores compute
 *                     approximate scores (operands rounded to fp16 after a power-of-two scaling: 11 significand bits, as
 *                     tf32) with a proven error bound and only FILTER (per-row certified threshold = the
 *                     (k + masked)-th largest group maximum minus the bound); every candidate that survives is scored
 *                     again in fp32 (fmaf) from the original tables and ranked on that value, ties -> lower index.
 *                     Nothing depends on timing.  ws from mmrec_score_topk_workspace_bytes.
 * mmrec_catalog_pack_f32 / mmrec_score_topk_cat_f32: the same with the item operand prepared once per embedding
 *                     table instead of once per batch (the reference calls full_sort_predict per eval batch of 4096
 *                     users against the same item table, src/common/trainer.py:302-310).  `cat`: 1024-byte aligned
 *                     buffer of mmrec_catalog_bytes(n_items, d) bytes; it must be re-packed whenever Ie changes and
 *                     passed together with the same (n_items, Ie, ldi, d).  cat == NULL packs into ws.
 * mmrec_topk_merge:   merge `parts` sorted lists per user ([parts, B, k] values + indices) into
 *                     one (the per-user top-k reduction across item shards, SURVEY 8e).
 * ------------------------------------------------------------------------------------------- */
/* path of mmrec_score_f32 / mmrec_score_topk_f32 (env MMREC_SCORE_PATH = simt | tc | auto | fused sets the start value):
 *   0 simt   exact fp32 on CUDA cores
 *   1 tc     wgmma 3xTF32 GEMM into an L2-resident score block, then mask + radix-select top-k kernels
 *   2 auto   (default) fused wherever its shape rules allow (k <= 256, d <= 128, at least 2k item groups of 16..128
 *            items), else tc
 *   3 fused  certified-filter path, no score matrix */
int mmrec_score_set_path(int path);
size_t mmrec_score_workspace_bytes(int64_t B, int64_t n_items, int d);
int mmrec_score_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu,
                    int64_t n_items, const float* Ie, int64_t ldi, int d,
                    float* S, int64_t ldS, void* ws, size_t ws_bytes, void* stream);
int mmrec_mask_f32(int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols,
                   int64_t B, int64_t n_items, int64_t item_offset, float* S, int64_t ldS, void* stream);
int mmrec_topk_rows_f32(int64_t B, int64_t n_items, const float* S, int64_t ldS, int k,
                        int64_t item_offset, int64_t* out_idx, float* out_val, void* stream);
size_t mmrec_score_topk_workspace_bytes(int64_t B, int64_t n_items, int d, int k);
int mmrec_score_topk_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu,
                         int64_t n_items, const float* Ie, int64_t ldi, int d,
                         int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols,
                         int k, int64_t item_offset, int64_t* out_idx, float* out_val,
                         void* ws, size_t ws_bytes, void* stream);
size_t mmrec_catalog_bytes(int64_t n_items, int d);
int mmrec_catalog_pack_f32(int64_t n_items, const float* Ie, int64_t ldi, int d,
                           void* cat, size_t cat_bytes, void* stream);
int mmrec_score_topk_cat_f32(int64_t B, const int64_t* users, const float* Ue, int64_t ldu,
                             int64_t n_items, const float* Ie, int64_t ldi, int d, const void* cat,
                             int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols,
                             int k, int64_t item_offset, int64_t* out_idx, float* out_val,
                             void* ws, size_t ws_bytes, void* stream);
/* diagnostic, synchronising: rows of the last row block of the last fused call on `ws` that needed the exact kernel
 * (with_cat: the call packed its catalogue into ws, i.e. cat was NULL) */
int64_t mmrec_debug_fused_fallback_rows(const void* ws, int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, int with_cat);
/* diagnostic, host only (no launch, no synchronisation): the scratch layout of a fused call with these arguments, for
 * reading the filter's intermediate stages back after the call.  Fills out[0 .. min(cap, 16) - 1] with
 *   rows_blk, rows_pad, KP, gw, n_it, G, G_valid,
 *   catalogue offset (-1 when with_cat == 0: the catalogue lives in the caller's buffer), catalogue header bytes (the
 *   fp16 item tiles follow the header), user pack, user row norms, gmax [rows_blk][G], thr, bitmap [rows_blk][n_it] x
 *   16 B, flags [rows_blk] | counter | row_of_slot, total workspace,
 * offsets in bytes from the workspace pointer rounded up to 1024.  Only the last row block's scratch survives a call.
 * Returns the number of entries (16), -1 for a shape the fused path does not take. */
int mmrec_debug_cf_scratch(int64_t B, int64_t n_items, int d, int k, int64_t mask_nnz, int with_cat, int64_t* out, int cap);
/* tuning aid: with env MMREC_CF_TIMING set, device time in microseconds of the stages of the last fused call (host array
 * us[cap]; stages: catalogue pack | prep + mask | pass 1 | threshold | pass 2 | finalists | exact rows); returns the count */
int mmrec_debug_cf_timing(float* us, int cap);

/* K7  item-item cosine kNN of a feature table.   Replaces `sim = torch.mm(context_norm, context_norm.transpose(1, 0));
 * torch.topk(sim, k, dim=-1)` of FREEDOM's `get_knn_adj_mat` (src/models/freedom.py:79-91) and of
 * `build_knn_normalized_graph` (src/utils/utils.py:165-172); the caller passes the L2-normalised rows.
 *
 * mmrec_knn_topk_f32: for query rows j < m (table row rows[j]; rows == NULL means all rows, m == n), the top-k of
 *                     X[rows[j]] . X[i] over all n rows i into out_idx / out_val [m, k]: values descending, equal values by
 *                     ascending index -- the contract of mmrec_topk_rows_f32 -- and bit-identical to mmrec_score_f32 on
 *                     its CUDA-core path followed by mmrec_topk_rows_f32, NaN included.  Tensor cores (fp16 operands,
 *                     proven error bound, knn_cf.cu) only select candidates; every returned value is the exact fp32
 *                     chain.  Rows the certificate cannot serve, and every row of a table holding a non-finite element,
 *                     are computed by that exact route itself.  Synchronises `stream` (once per row block).
 *                     Limits: n >= 1, 1 <= F, 1 <= k <= 1024, k <= n, n < 2^31, rows[j] in [0, n) (not checked);
 *                     violations return MMREC_EINVAL, a workspace below mmrec_knn_topk_workspace_bytes(n, F, m, k)
 *                     MMREC_EWORKSPACE.  m == 0 returns at once.
 * mmrec_knn_topk_workspace_bytes: 0 for arguments outside those limits.  Holds the fp16 pack of X (2 n F bytes) plus
 *                     bounded row-block scratch (<= ~1 GB).
 * mmrec_debug_knn_fallback_rows: rows of the last mmrec_knn_topk_f32 call served by the exact route (all m when the table
 *                     held a non-finite element), -1 before the first call.
 * ------------------------------------------------------------------------------------------- */
size_t mmrec_knn_topk_workspace_bytes(int64_t n, int F, int64_t m, int k);
int mmrec_knn_topk_f32(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k,
                       int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, void* stream);
int64_t mmrec_debug_knn_fallback_rows(void);
/* diagnostic, host only (no launch, no synchronisation): the scratch layout of mmrec_knn_topk_f32 / _shrink_f32 with
 * these arguments.  Fills out[0 .. min(cap, 15) - 1] with
 *   rows_blk, rows_pad, KP, items per group (16), n_it, G, G_valid,
 *   header (words: [0] largest |element| bits, [1] largest row norm bits; shrink route [2] .. [5]), fp16 item tiles,
 *   row norms [n], query pack, gmax [rows_blk][G], thr, flags, total workspace,
 * offsets in bytes from the workspace pointer rounded up to 1024.  Only the last row block's scratch survives a call.
 * Returns the number of entries (15), -1 for arguments mmrec_knn_topk_workspace_bytes refuses. */
int mmrec_debug_knn_scratch(int64_t n, int F, int64_t m, int k, int64_t* out, int cap);
/* mmrec_knn_topk_shrink_f32: the same, ranked by the shrunk similarity of ItemKNNCBF's `build_item_sim_matrix`
 *                     (src/models/itemknncbf.py:56-65): v(q, i) = s(q, i) / ((norms[q] * norms[i]) + shrink), s the exact
 *                     chain above, the denominator two IEEE fp32 roundings (multiply, then add) and an IEEE division.
 *                     `norms` [n] is the caller's (the reference's `torch.norm(X, p=2, dim=-1)`).  Bit-identical to
 *                     mmrec_score_f32 on its CUDA-core path, then that elementwise denominator, then mmrec_topk_rows_f32,
 *                     NaN included.  Uses the workspace of mmrec_knn_topk_workspace_bytes.  Besides the rows the certificate
 *                     cannot serve, every row takes the exact route when the table holds a non-finite element, when a norm
 *                     is not finite, when shrink is negative or not finite, or when shrink is 0 and a norm is 0.
 *                     mmrec_debug_knn_fallback_rows counts them. */
int mmrec_knn_topk_shrink_f32(int64_t n, const float* X, int64_t ldx, int F, int64_t m, const int64_t* rows, int k,
                              const float* norms, float shrink, int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes,
                              void* stream);

/* K9  user scores from the sparse interactions and the sparse item kNN graph.   Replaces `scores_matrix = torch.mm(R,
 * item_sim)` of ItemKNNCBF (src/models/itemknncbf.py:54) and its row gather in full_sort_predict (:107-111) without the
 * dense [I, I] graph or the dense [U, I] scores.  R [n_users, n_items] and S [n_items, n_items] are int32 CSR (rowptr, col,
 * val); R's columns ascend within a row, S's columns are distinct within a row.  score[u, j] = the fmaf(R[u, i], S[i, j],
 * acc) chain over the entries i of R(u) in order, from acc = +0.0; items no S row reaches are +0.0.
 *
 * mmrec_sparse_scores_f32: rows users[b] (users == NULL: row b) of that matrix into out [B, n_items] (row stride ldo),
 *                     overwritten.  Deterministic, no atomics.  Limits: 1 <= n_items < 2^31.
 * mmrec_sparse_score_topk_f32: the same rows, then `scores[mask_rows, mask_cols] = -1e10` (mask entries: batch row, item;
 *                     entries outside [0, B) x [0, n_items) are ignored) and the top-k into out_idx / out_val [B, k], with
 *                     no dense row written.  Bit-identical to mmrec_sparse_scores_f32 + mmrec_mask_f32 +
 *                     mmrec_topk_rows_f32 (values descending, equal values by ascending index).  Rows with more than 2048
 *                     products or masked items, or a non-finite score, run that unfused route inside the call.
 *                     Synchronises `stream`.  Limits: 1 <= k <= min(1024, n_items).
 * mmrec_sparse_score_topk_workspace_bytes: 0 for arguments outside those limits.
 * mmrec_debug_sparse_topk_fallback_rows: rows of the last mmrec_sparse_score_topk_f32 call served by the unfused route,
 *                     -1 before the first call.
 * ------------------------------------------------------------------------------------------- */
int mmrec_sparse_scores_f32(int64_t B, const int64_t* users, int64_t n_items, const int32_t* r_ptr, const int32_t* r_col,
                            const float* r_val, const int32_t* s_ptr, const int32_t* s_col, const float* s_val, float* out,
                            int64_t ldo, void* stream);
size_t mmrec_sparse_score_topk_workspace_bytes(int64_t B, int64_t n_items, int64_t mask_nnz, int k);
int mmrec_sparse_score_topk_f32(int64_t B, const int64_t* users, int64_t n_items, const int32_t* r_ptr, const int32_t* r_col,
                                const float* r_val, const int32_t* s_ptr, const int32_t* s_col, const float* s_val,
                                int64_t mask_nnz, const int64_t* mask_rows, const int64_t* mask_cols, int k,
                                int64_t* out_idx, float* out_val, void* ws, size_t ws_bytes, void* stream);
int64_t mmrec_debug_sparse_topk_fallback_rows(void);

/* K8  full-table exp-sum of LGMRec's hypergraph contrastive loss.   Replaces `ttl_score = torch.exp(torch.matmul(norm_emb1,
 * norm_all_emb.T) / self.tau).sum(dim=1)` of `ssl_triple_loss` (src/models/lgmrec.py:159-166) and its autograd, without the
 * [B, M] matrix: wgmma 3xTF32, exp and the row sums in the accumulator registers (expsum.cu, which derives the error bound).
 *
 * mmrec_expsum_rows_f32:     ttl[b] = sum_{j < M} exp(<Q[b], T[j]> * inv_tau) for b < B.  Q [B, d] (row stride ldq), T [M, d]
 *                            (ldt), fp32 row-major.  No maximum is subtracted: inf where the terms or their sum overflow.
 *                            M == 0 gives ttl = 0; B == 0 returns at once.  Duplicate rows are allowed.
 * mmrec_expsum_rows_bwd_f32: for the upstream gradient g [B]:  dQ[b] = g[b] * inv_tau * sum_j e_bj T[j],
 *                            dT[j] = inv_tau * sum_b g[b] e_bj Q[b]  (e_bj recomputed, never stored).  dQ or dT may be NULL
 *                            to skip it (not both).
 *                            Both: d in {32, 64, 128}, B >= 0, M >= 0, leading dimensions >= d; violations and null pointers
 *                            return MMREC_EINVAL, a workspace below mmrec_expsum_rows_workspace_bytes(B, M, d)
 *                            MMREC_EWORKSPACE.  Results are bit-reproducible (fixed summation order, no atomics); the
 *                            chunking depends on B and M only.
 * mmrec_expsum_rows_workspace_bytes: for either call; O((B + M) d) (at most 32 partial slabs of B or 256 tile rows of M,
 *                            0 when none is needed); 0 also for d outside {32, 64, 128} or negative sizes.
 * ------------------------------------------------------------------------------------------- */
size_t mmrec_expsum_rows_workspace_bytes(int64_t B, int64_t M, int d);
int mmrec_expsum_rows_f32(int64_t B, const float* Q, int64_t ldq, int64_t M, const float* T, int64_t ldt, int d, float inv_tau,
                          float* ttl, void* ws, size_t ws_bytes, void* stream);
int mmrec_expsum_rows_bwd_f32(int64_t B, const float* Q, int64_t ldq, int64_t M, const float* T, int64_t ldt, int d, float inv_tau,
                              const float* g, float* dQ, int64_t lddq, float* dT, int64_t lddt, void* ws, size_t ws_bytes,
                              void* stream);

int mmrec_topk_merge(int parts, int64_t B, int k, const float* vals, const int64_t* idx,
                     int64_t* out_idx, float* out_val, void* stream);
/* the same merge over lists left where each rank wrote them (peer-mapped memory): vals[p] / idx[p] are host
 * arrays of `parts` (<= 16, parts * k <= 1024) device pointers to [B, k] lists, each sorted (value desc, index asc); an
 * index becomes idx * idx_mul + p * idx_add (round-robin item shards: idx_mul = world, idx_add = 1; must stay below
 * 2^32).  Only rows [row0, row0 + n_rows) are merged, into out_idx / out_val [n_rows, k]: in the sharded evaluation
 * every rank merges its own slice of the batch.  The ranks must be synchronised before the lists are read: either by
 * the caller, or inside the kernel when `flags` / `state` / `rank` are given (see mmrec_peer_exchange_f32). */
int mmrec_topk_merge_peers(int parts, int64_t B, int k, const void* const* vals, const void* const* idx,
                           int64_t idx_mul, int64_t idx_add, int64_t row0, int64_t n_rows,
                           int64_t* out_idx, float* out_val,
                           void* const* flags /* nullable */, int32_t* state /* nullable */, int rank, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K4  user-embedding exchange of the item-sharded propagation, over peer memory (no reference counterpart:
 * the reference is single-GPU, src/utils/configurator.py:114-118; the sum it distributes is the user half of
 * `torch.sparse.mm(adj, ego)`, src/models/freedom.py:172, plus the layer mean of freedom.py:175-176).
 *
 * mmrec_peer_sum_f32 (all ranks read all partials; right for world = 2):
 *   parts   host array of `world` device pointers, rank order: partial user sums R_g E_Ig, [n] floats each,
 *           peer-mapped (CUDA IPC / symmetric memory) -- the caller synchronises the ranks before the call
 *   sum_out = sum over ranks in rank order (identical bits on every rank), may be NULL
 *   acc_out = (acc_in + sum) / acc_div, may be NULL (acc_in NULL = 0; in place allowed)
 *   n % 4 == 0, all pointers 16-byte aligned, world <= 16.
 *
 * mmrec_peer_reduce_push_f32 (reduce-scatter + all-gather in one kernel; what scales to 8 GPUs): rank `rank` owns the
 *   slice [rank * per, (rank + 1) * per) of the n / 4 float4 elements, per = ceil(n / 4 / world).  It sums that slice of
 *   all partials in rank order and stores the result into the same slice of every dst[p] (peer-mapped, its own
 *   included): a non-final layer stores the sum and, if acc_in, acc_out = acc_in + sum; the final layer stores
 *   (acc_in + sum) / acc_div.  acc_in / acc_out hold THIS RANK'S SLICE only (per float4, may alias).  The caller
 *   synchronises the ranks before (partials complete) and after (stores visible) the call.
 *
 * mmrec_peer_gather_f32: dst[p * n_each + i] = src[p][i] -- all-gather of a sharded table by peer loads (the item-id
 *   embeddings the item-item layer of the sharded FREEDOM needs, src/models/freedom.py:166-167).
 */
int mmrec_peer_sum_f32(int64_t n, int world, const void* const* parts, const float* acc_in,
                       float* acc_out, float acc_div, float* sum_out, void* stream);
int mmrec_peer_reduce_push_f32(int64_t n, int world, int rank, const void* const* parts, void* const* dst,
                               const float* acc_in, float* acc_out, float acc_div, int final_layer, void* stream);
int mmrec_peer_gather_f32(int64_t n_each, int world, const void* const* src, float* dst, void* stream);
/* The same with both synchronisations INSIDE the kernel -- one launch per layer: wait until every rank's partial is
 * complete, reduce my slice, store it to every rank, wait until every rank's stores have landed.
 *   flags  host array of `world` device pointers to each rank's flag array (int32[2 * world], peer-mapped, zero at start)
 *   state  this rank's int32[4] in ordinary device memory, zero at start: {calls completed, release word, block counter, -}
 * Calls are numbered on the device (state[0]), so the launch can be replayed from a CUDA graph; every rank must issue
 * the same sequence of calls that use the same flags (mmrec_peer_exchange_f32, mmrec_peer_barrier, mmrec_topk_merge_peers
 * with flags).  A rank that never arrives makes the others trap after 4 s instead of hanging. */
int mmrec_peer_exchange_f32(int64_t n, int world, int rank, const void* const* parts, void* const* dst, void* const* flags,
                            int32_t* state, const float* acc_in, float* acc_out, float acc_div, int final_layer, void* stream);
int mmrec_peer_barrier(int world, int rank, void* const* flags, int32_t* state, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f2  evaluator on the device.   Replaces the host loop that builds the hit matrix from `.cpu().numpy()` of the index
 * matrix and the metric functions (src/utils/topk_evaluator.py:70-102, src/utils/metrics.py:12-105).
 *   topk_idx  int64 [n_users, K]  the trainer's index matrix (K = max(topk) <= 128)
 *   pos_ptr   int64 [n_users + 1], pos_items int64 sorted ascending per user: the ground-truth items
 *   disc      float64 [K] = 1 / log2(j + 2);  idcg_all float64 [K] = cumsum(disc)      (computed by the host, as numpy does)
 *   sums      float64 [4, K], ADDED to: per position j the sum over users of recall / ndcg / precision / map at j + 1
 *             (zero it before the first batch; divide by the number of users afterwards)
 * ------------------------------------------------------------------------------------------- */
int mmrec_topk_metrics_f64(int64_t n_users, int K, const int64_t* topk_idx, const int64_t* pos_ptr, const int64_t* pos_items,
                           const double* disc, const double* idcg_all, double* sums, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f1  feature-table gradient path and optimiser step.   Replaces, per training batch and modality, the backward of
 * `self.image_trs(self.image_embedding.weight)` (src/models/freedom.py:58-62,205-209; bm3.py:102-104; mgcn.py:148-150:
 * the tables are `nn.Embedding.from_pretrained(.., freeze=False)`, i.e. trainable [n_items, F] parameters) -- cuBLAS
 * GEMMs dW = g^T X, dX = g W plus a dense [n_items, F] gradient -- and `torch.optim.Adam.step` over it
 * (src/common/trainer.py:117-118,185-189).  IEEE fp32 on CUDA cores, operation order of torch's `_multi_tensor_adam`.
 *
 * mmrec_index_sum_rows_f32     G[i,:] = sum over j ascending with idx[j] == i of g[j,:]    G [n_rows, ldG], g [n_idx, ldg];
 *                              rows nobody points at become zero; indices outside [0, n_rows) are ignored.
 *                              The gradient of a gathered projection `Linear(table)[idx]` w.r.t. the table is G W.
 * mmrec_linear_wgrad_f32       dW[k,f] = sum_j g[j,k] table[idx ? idx[j] : j, f]   dW [d, F];   db[k] = sum_j g[j,k]  (db nullable)
 *                              ws from mmrec_linear_wgrad_workspace_bytes (per-CTA partials, reduced in a fixed order:
 *                              bit-reproducible).  16-byte accesses when F % 4 == 0 and table / dW / ws are aligned, else 4-byte.
 * mmrec_linear_dgrad_f32       dX = G W   dX [n_rows, F] (leading dimension F), G [n_rows, ldG], W [d, F]; any d (128 k at a
 *                              time), any F.
 * mmrec_linear_dgrad_adam_f32  one Adam step of `param` [n_rows, F] whose gradient is G W, WITHOUT materialising it:
 *                                grad = G W (+ weight_decay * param);  exp_avg += (1 - beta1)(grad - exp_avg);
 *                                exp_avg_sq = beta2 exp_avg_sq + (1 - beta2) grad^2;
 *                                param += step_size * exp_avg / (sqrt(exp_avg_sq) / bc2_sqrt + eps)
 *                              with step_size = -lr / (1 - beta1^t) and bc2_sqrt = sqrt(1 - beta2^t) computed by the caller in
 *                              double, as torch/optim/adam.py does.  W must still hold the values the forward used.
 *                              d <= 128, F % 4 == 0, 16-byte aligned pointers (else MMREC_EUNSUPPORTED / MMREC_EINVAL).
 * mmrec_adam_f32               the same update for `n_tensors` ordinary (param, grad) pairs, one launch per 24 tensors;
 *                              `tensors` is a HOST array.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    float* param; const float* grad; float* exp_avg; float* exp_avg_sq;
    int64_t n;
    double step_size, bc2_sqrt;
} mmrec_adam_tensor;
int mmrec_index_sum_rows_f32(int64_t n_idx, const int64_t* idx, const float* g, int64_t ldg, int d, int64_t n_rows, float* G,
                             int64_t ldG, void* stream);
size_t mmrec_linear_wgrad_workspace_bytes(int64_t n, int64_t F, int d);
int mmrec_linear_wgrad_f32(int64_t n, const int64_t* idx, const float* g, int64_t ldg, int d, const float* table, int64_t n_table,
                           int64_t F, float* dW, float* db, void* ws, size_t ws_bytes, void* stream);
int mmrec_linear_dgrad_f32(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, float* dX, void* stream);
int mmrec_linear_dgrad_adam_f32(int64_t n_rows, const float* G, int64_t ldG, int d, const float* W, int64_t F, float* param,
                                float* exp_avg, float* exp_avg_sq, double beta1, double beta2, double eps, double weight_decay,
                                double step_size, double bc2_sqrt, void* stream);
int mmrec_adam_f32(int n_tensors, const mmrec_adam_tensor* tensors, double beta1, double beta2, double eps, double weight_decay,
                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * a5b  MGCN's row-wise fusion (src/models/mgcn.py:153-154 purifier gates, :187-201 two-view attention, preference gates,
 * side + content), inference form.  d in {32, 64, 128}; all matrices row-major with leading dimension d; W are
 * `nn.Linear` weights [d, d] (y = x W^T + b), biases nullable.
 * mmrec_gate_rows_f32   out[n,:] = mul[n,:] * sigmoid(X[n,:] W^T + b)                  (mul nullable: the gate alone)
 * mmrec_mgcn_fuse_f32   a_v = wq2 . tanh(Wq img + bq), a_t likewise on txt; (w0, w1) = softmax(a_v, a_t);
 *                       common = w0 img + w1 txt; sep_v = sigmoid(Wgi content + bgi) (img - common), sep_t likewise;
 *                       side = (sep_v + sep_t + common) / 3 (stored if side != NULL); out = content + side
 * ------------------------------------------------------------------------------------------- */
int mmrec_gate_rows_f32(int64_t n, int d, const float* X, const float* W, const float* b, const float* mul, float* out, void* stream);
int mmrec_mgcn_fuse_f32(int64_t n, int d, const float* img, const float* txt, const float* content, const float* Wq, const float* bq,
                        const float* wq2, const float* Wgi, const float* bgi, const float* Wgt, const float* bgt, float* out,
                        float* side, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMREC_B200_H */
