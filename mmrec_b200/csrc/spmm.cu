// K1: CSR SpMM  y = A X  with the layer-combination epilogue fused (running sum / mean, "+h", LayerGCN's
// cosine gate).  L2/HBM-bound gather kernel: no tensor cores (0.25-0.5 flop/byte).
//
// Mapping (D = embedding width, a multiple of 32 floats):
//   * a task is a whole row or, for rows longer than the plan's segment length, one segment of it
//     (mmrec_spmm_plan; tasks arrive sorted longest-first) -- the power-law item rows would otherwise
//     serialise on one warp;
//   * T lanes (default D/4: one float4 per lane) own one task, a warp runs 32/T tasks side by side; each lane
//     holds V = D/(4T) float4 of the row, so one row of X is V coalesced T*16-byte requests; UNR rows of X are
//     in flight per lane group before the first FMA;
//   * every lane loads the (column, value) pairs it needs itself -- the T lanes of a group read the same
//     address, one broadcast transaction, no shuffles in the gather loop; the next batch's indices, the next
//     task's descriptor and the running-sum row of the epilogue are requested while the gather is in flight;
//   * the longest tasks (plan: n_cta_tasks) are run by a whole CTA each, reduced through shared memory in
//     lane-group order; the rest one lane group each, warps walking the sorted list boustrophedon;
//   * split rows: each segment writes its partial sum to scratch, the LAST segment to arrive (per-row
//     counter) adds the partials in segment order -> the summation order never depends on scheduling, so
//     results are bit-reproducible.
// Grid: persistent, (SM count x resident CTAs) CTAs of 8 warps striding over the task list.
#include <cooperative_groups.h>

#include "common.cuh"

namespace mmrec {

struct SpmmParams {
    int64_t n_rows, n_cols;
    const int32_t* rowptr; const int32_t* colidx; const float* vals;
    const int4* tasks; int64_t n_tasks, n_heavy; const int4* split_rows; int32_t* counters; float* partial;
    const float* X; int64_t ldx;
    float* Y; int64_t ldy;
    const float* acc_in; float* acc_out; int64_t ldacc; float acc_div;
    const float* gate_ref; int64_t ldgate;
    int y_acc;                         // Y[r,:] += y[r,:] instead of = (column-panelled products: the panels of one matrix add up in Y)
    const float* post; int64_t post_row0; uint32_t spost;   // acc_out[r,:] += post[r - post_row0, :] for r >= post_row0 (after the division)
    int d;
    uint32_t sx, sy, sacc, sgate;      // the leading dimensions as byte strides (vector kernel: one IMAD.WIDE per row address)
    // Two-block operands (chained kernel only, mmrec_spmm_op.X_hi): row c of X is X_hi[c - x_split] for c >= x_split, row r of
    // acc_in is acc_in_hi[r - acc_split] for r >= acc_split -- [users; items] straight from the two embedding tables, no copy.
    // One block: X_hi = X, x_split = n_cols, acc_in_hi = acc_in, acc_split = n_rows.
    const float* X_hi; const float* acc_in_hi;
    int x_split, acc_split;
    uint32_t sx_hi, sacc_hi;
};

// T lanes cooperate on one task (row or row segment); a warp runs 32/T tasks at once.  Fewer lanes per row
// means more rows in flight per SM -- the kernel is bound by dependent-load latency (task descriptor -> column
// indices -> rows of X), not by bytes, so rows in flight is what buys throughput at Amazon-scale graphs.

// Row `r`, float4 number `f4` of a matrix with byte stride `stride`: 32 x 32 -> 64-bit multiply-add, one instruction.
__device__ __forceinline__ const float4* row_f4(const float* base, uint32_t stride, int r, int f4) {
    return reinterpret_cast<const float4*>(reinterpret_cast<const char*>(base) + (uint64_t)(uint32_t)r * stride) + f4;
}
__device__ __forceinline__ float4* row_f4(float* base, uint32_t stride, int r, int f4) {
    return reinterpret_cast<float4*>(reinterpret_cast<char*>(base) + (uint64_t)(uint32_t)r * stride) + f4;
}

// Row `r` of acc_in; TWO: from the block the row falls in (a select, not a branch: the lane groups of a warp may straddle the split).
template <bool TWO>
__device__ __forceinline__ float4 acc_in_f4(const SpmmParams& p, int r, int f4) {
    const bool hi = TWO && r >= p.acc_split;
    return *row_f4(hi ? p.acc_in_hi : p.acc_in, hi ? p.sacc_hi : p.sacc, hi ? r - p.acc_split : r, f4);
}

template <int D, int T>
struct VecCfg {
    static_assert(D % (4 * T) == 0, "row must split into float4 per lane");
    static constexpr int V = D / (4 * T);              // float4 per lane per row of X
    static constexpr int GPW = 32 / T;                 // tasks per warp
    // rows of X in flight per lane group.  V = 3 (the width-3d instances): 4 rows, 12 float4 per lane -- 86 registers, no
    // spills, 2 CTAs of 256 threads per SM; 8 would be 24 float4 and ~102 registers, 2 would be 80 registers and 3 CTAs but
    // fewer rows in flight per SM (DESIGN.md section 4, K1)
    static constexpr int UNR = (V >= 4) ? 2 : (V == 3 ? 4 : (V == 2 ? 4 : 8));
};

template <int D, int T>
__device__ __forceinline__ void spmm_epilogue(const SpmmParams& p, bool on, int row, int l, float4 (&y)[VecCfg<D, T>::V],
                                              const float4 (&accin)[VecCfg<D, T>::V]) {
    using C = VecCfg<D, T>;
    // Called by ALL 32 lanes (warp-uniform control flow); `on` predicates the memory traffic of this lane group.
    // Lane l of the group owns floats [(v*T + l)*4, +4) of the row: each v is one coalesced T*16-byte request.
    if (p.gate_ref) {
        float dot = 0.f, ny = 0.f, nr = 0.f;
        if (on) {
#pragma unroll
            for (int v = 0; v < C::V; ++v) {
                float4 r = __ldg(row_f4(p.gate_ref, p.sgate, row, v * T + l));
                dot += y[v].x * r.x + y[v].y * r.y + y[v].z * r.z + y[v].w * r.w;
                ny += y[v].x * y[v].x + y[v].y * y[v].y + y[v].z * y[v].z + y[v].w * y[v].w;
                nr += r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
            }
        }
#pragma unroll
        for (int o = T / 2; o > 0; o >>= 1) {       // xor distances < T stay inside the lane group
            dot += __shfl_xor_sync(0xffffffffu, dot, o);
            ny += __shfl_xor_sync(0xffffffffu, ny, o);
            nr += __shfl_xor_sync(0xffffffffu, nr, o);
        }
        // F.cosine_similarity(eps=1e-8): <x/max(|x|,eps), y/max(|y|,eps)>  (layergcn.py:132)
        float c = dot / (fmaxf(sqrtf(ny), 1e-8f) * fmaxf(sqrtf(nr), 1e-8f));
#pragma unroll
        for (int v = 0; v < C::V; ++v) { y[v].x *= c; y[v].y *= c; y[v].z *= c; y[v].w *= c; }
    }
    if (!on) return;
    if (p.Y) {
#pragma unroll
        for (int v = 0; v < C::V; ++v) {
            float4 o = y[v];
            if (p.y_acc) {
                const float4 q = *row_f4(p.Y, p.sy, row, v * T + l);
                o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
            }
            *row_f4(p.Y, p.sy, row, v * T + l) = o;
        }
    }
    if (p.acc_out) {
#pragma unroll
        for (int v = 0; v < C::V; ++v) {
            float4 a = y[v];
            if (p.acc_in) { a.x += accin[v].x; a.y += accin[v].y; a.z += accin[v].z; a.w += accin[v].w; }
            if (p.acc_div != 1.0f) {
                a.x = __fdiv_rn(a.x, p.acc_div); a.y = __fdiv_rn(a.y, p.acc_div);
                a.z = __fdiv_rn(a.z, p.acc_div); a.w = __fdiv_rn(a.w, p.acc_div);
            }
            if (p.post && row >= p.post_row0) {
                const float4 q = *row_f4(p.post, p.spost, row - (int)p.post_row0, v * T + l);
                a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
            }
            *row_f4(p.acc_out, p.sacc, row, v * T + l) = a;
        }
    }
}

// Gather of one task range [b, b + len) by one lane group: UNR rows of X in flight, the next batch's indices
// travel while they are.  `maxlen` is the trip bound shared by every group that runs in lock step with this one.
// TWO: each gathered row is read from the block of X it falls in; the products and their order are the same as from the
// concatenation, so the result is bit-identical.
// DROP: entry e (CSR position) takes part iff bit e of `dk.keep` is set, with weight fl(vals[e] * dk.scale); a dropped entry
// is a padding slot (no load of its row of X, weight 0), so the kept entries are summed in the order of the compacted row.
struct DropKeep { const uint32_t* keep; float scale; };

__device__ __forceinline__ bool keep_bit(const uint32_t* keep, int pos) {
    return (__ldg(keep + (pos >> 5)) >> (pos & 31)) & 1u;
}

template <int D, int T, bool TWO, bool DROP = false>
__device__ __forceinline__ void spmm_gather(const SpmmParams& p, int b, int len, int maxlen, int l, float4 (&acc)[VecCfg<D, T>::V],
                                            const DropKeep dk = DropKeep{nullptr, 1.f}) {
    using C = VecCfg<D, T>;
    int cj[C::UNR]; float wj[C::UNR]; bool kj[C::UNR];
    const int32_t* cp = p.colidx + b;                                // walked with immediate offsets: no per-load address math
    const float* vp = p.vals + b;
    const float* xl = p.X + l * 4;
    const float* xh = TWO ? p.X_hi + l * 4 : xl;
#pragma unroll
    for (int u = 0; u < C::UNR; ++u) {
        const bool ok = u < len;
        cj[u] = ok ? __ldg(cp + u) : 0;
        wj[u] = ok ? __ldg(vp + u) : 0.f;
        if constexpr (DROP) {
            kj[u] = ok && keep_bit(dk.keep, b + u);
            wj[u] = kj[u] ? __fmul_rn(wj[u], dk.scale) : 0.f;
        }
    }
    for (int j0 = 0; j0 < maxlen; j0 += C::UNR, cp += C::UNR, vp += C::UNR) {
        float4 x[C::UNR][C::V];
#pragma unroll
        for (int u = 0; u < C::UNR; ++u) {
            const bool ok = DROP ? kj[u] : j0 + u < len;
            const bool hi = TWO && cj[u] >= p.x_split;
            const float* xb = hi ? xh : xl;
            const uint32_t sb = hi ? p.sx_hi : p.sx;
            const int rb = hi ? cj[u] - p.x_split : cj[u];
#pragma unroll
            for (int v = 0; v < C::V; ++v)
                x[u][v] = ok ? __ldg(row_f4(xb, sb, rb, v * T)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float wc[C::UNR];
#pragma unroll
        for (int u = 0; u < C::UNR; ++u) wc[u] = wj[u];
#pragma unroll
        for (int u = 0; u < C::UNR; ++u) {
            const bool ok = j0 + C::UNR + u < len;
            cj[u] = ok ? __ldg(cp + C::UNR + u) : 0;
            wj[u] = ok ? __ldg(vp + C::UNR + u) : 0.f;
            if constexpr (DROP) {
                kj[u] = ok && keep_bit(dk.keep, b + j0 + C::UNR + u);
                wj[u] = kj[u] ? __fmul_rn(wj[u], dk.scale) : 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < C::UNR; ++u) {
#pragma unroll
            for (int v = 0; v < C::V; ++v) {
                acc[v].x = fmaf(wc[u], x[u][v].x, acc[v].x);
                acc[v].y = fmaf(wc[u], x[u][v].y, acc[v].y);
                acc[v].z = fmaf(wc[u], x[u][v].z, acc[v].z);
                acc[v].w = fmaf(wc[u], x[u][v].w, acc[v].w);
            }
        }
    }
}

// A finished task of a split row: publish the partial, and if this is the last segment of the row to arrive, add
// the partials in segment order and return true (the caller then runs the epilogue).  Warp-collective (full mask);
// `split` marks the lane groups that hold such a task.
template <int D, int T, bool TWO>
__device__ __forceinline__ bool spmm_split_finish(const SpmmParams& p, bool split, int row, int b, int sid, int l,
                                                  float4 (&acc)[VecCfg<D, T>::V], float4 (&accin)[VecCfg<D, T>::V]) {
    using C = VecCfg<D, T>;
    int4 sr = make_int4(0, 1, 0, 1);
    int old = -1;
    bool last = false;
    if (split) {
        sr = __ldg(p.split_rows + sid);                     // {first_slot, n_seg, row_begin, seg_len}
        const int seg = (b - sr.z) / sr.w;
        float* slot = p.partial + ((int64_t)sr.x + seg) * D;
#pragma unroll
        for (int v = 0; v < C::V; ++v) *reinterpret_cast<float4*>(slot + (v * T + l) * 4) = acc[v];
        __threadfence();
    }
    __syncwarp();
    if (split && l == 0) old = atomicAdd(p.counters + sid, 1);
    old = __shfl_sync(0xffffffffu, old, 0, T);
    if (split && old == sr.y - 1) {
        __threadfence();
#pragma unroll
        for (int v = 0; v < C::V; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        constexpr int RB = 8;                               // partials in flight; the order of the adds stays fixed
        for (int s2 = 0; s2 < sr.y; s2 += RB) {
            float4 q[RB][C::V];
#pragma unroll
            for (int r = 0; r < RB; ++r) {
                const float* ps = p.partial + ((int64_t)sr.x + s2 + r) * D;
#pragma unroll
                for (int v = 0; v < C::V; ++v)
                    q[r][v] = (s2 + r < sr.y) ? __ldcg(reinterpret_cast<const float4*>(ps + (v * T + l) * 4))
                                              : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int r = 0; r < RB; ++r) {
#pragma unroll
                for (int v = 0; v < C::V; ++v) {
                    acc[v].x += q[r][v].x; acc[v].y += q[r][v].y; acc[v].z += q[r][v].z; acc[v].w += q[r][v].w;
                }
            }
        }
        if (p.acc_in) {
#pragma unroll
            for (int v = 0; v < C::V; ++v)
                accin[v] = acc_in_f4<TWO>(p, row, v * T + l);
        }
        if (l == 0) p.counters[sid] = 0;                    // self-cleaning for the next launch
        last = true;
    }
    __syncwarp();
    return last;
}

// Phase 1: the n_heavy longest tasks, one CTA each -- its 256/T lane groups split the task evenly, reduce through
// shared memory in group order, warp 0 finishes the row.  A 5,000-nnz item row becomes ~10 CTA tasks of one or two
// load batches per group instead of a chain of dozens of dependent batches on one warp.
// Phase 2: the remaining (short) tasks, one lane group each, 32/T per warp in lock step: warp-uniform control flow
// (trip count = longest task of the warp; the plan sorts by length so neighbours are alike), everything per-group
// predicated, no shuffles in the gather loop (the T lanes of a group read the same (col, val) address = one
// broadcast transaction).  Warps walk the sorted list boustrophedon, so whoever got the longest tasks in one sweep
// gets the shortest in the next.
template <int D, int T, bool TWO, bool DROP = false>
__device__ __forceinline__ void spmm_vec_body(const SpmmParams& p, float* __restrict__ red, const DropKeep dk = DropKeep{nullptr, 1.f}) {
    using C = VecCfg<D, T>;
    constexpr int G = 256 / T;                              // lane groups per CTA
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane / T, l = lane % T;
    const int64_t n_work = p.tasks ? p.n_tasks : p.n_rows;
    const int64_t n_heavy = p.tasks ? p.n_heavy : 0;

    // ---------------- phase 1: CTA-cooperative tasks
    for (int64_t ct = blockIdx.x; ct < n_heavy; ct += gridDim.x) {
        const int4 tk = __ldg(p.tasks + ct);
        const int row = tk.x, sid = tk.w;
        const int len = tk.z - tk.y;
        const int chunk = (len + G - 1) / G;
        const int gi = warp * C::GPW + g;
        const int mb = tk.y + gi * chunk;
        int mylen = tk.z - mb;
        mylen = mylen < 0 ? 0 : (mylen > chunk ? chunk : mylen);
        float4 accin[C::V];
#pragma unroll
        for (int v = 0; v < C::V; ++v) accin[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (warp == 0 && g == 0 && p.acc_in && sid < 0) {
#pragma unroll
            for (int v = 0; v < C::V; ++v)
                accin[v] = acc_in_f4<TWO>(p, row, v * T + l);
        }
        float4 acc[C::V];
#pragma unroll
        for (int v = 0; v < C::V; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        spmm_gather<D, T, TWO, DROP>(p, mb, mylen, chunk, l, acc, dk);
#pragma unroll
        for (int v = 0; v < C::V; ++v) *reinterpret_cast<float4*>(red + gi * D + (v * T + l) * 4) = acc[v];
        __syncthreads();
        if (warp == 0) {
#pragma unroll
            for (int v = 0; v < C::V; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g == 0) {
                for (int q = 0; q < G; ++q) {               // group order: fixed summation order
#pragma unroll
                    for (int v = 0; v < C::V; ++v) {
                        const float4 r4 = *reinterpret_cast<const float4*>(red + q * D + (v * T + l) * 4);
                        acc[v].x += r4.x; acc[v].y += r4.y; acc[v].z += r4.z; acc[v].w += r4.w;
                    }
                }
            }
            bool do_epi = g == 0 && sid < 0;
            if (sid >= 0) do_epi = spmm_split_finish<D, T, TWO>(p, g == 0, row, tk.y, sid, l, acc, accin);
            spmm_epilogue<D, T>(p, do_epi, row, l, acc, accin);
        }
        __syncthreads();
    }

    // ---------------- phase 2: one lane group per task
    const int64_t W = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    const int64_t n_light = n_work - n_heavy;
    auto slot_of = [&](int64_t it) -> int64_t { return it * W + ((it & 1) ? (W - 1 - w) : w); };   // boustrophedon
    auto fetch = [&](int64_t slot) -> int4 {
        const int64_t t = slot * C::GPW + g;
        if (t >= n_light) return make_int4(-1, 0, 0, -1);
        if (p.tasks) return __ldg(p.tasks + n_heavy + t);
        return make_int4((int)t, __ldg(p.rowptr + t), __ldg(p.rowptr + t + 1), -1);
    };
    const int64_t n_slots = (n_light + C::GPW - 1) / C::GPW;
    const int64_t n_iter = (n_slots + W - 1) / W;                   // the same for every warp of the grid
    int4 nxt = fetch(slot_of(0));
    for (int64_t it = 0; it < n_iter; ++it) {
        const int row = nxt.x, b = nxt.y, sid = nxt.w;
        const int len = nxt.z - nxt.y;
        const bool valid = row >= 0;
        nxt = fetch(slot_of(it + 1));                               // next task's descriptor: in flight during the gather
        const int maxlen = __reduce_max_sync(0xffffffffu, valid ? len : 0);
        float4 accin[C::V];
#pragma unroll
        for (int v = 0; v < C::V; ++v) accin[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid && p.acc_in && sid < 0) {                         // epilogue operand does not depend on the gather
#pragma unroll
            for (int v = 0; v < C::V; ++v)
                accin[v] = acc_in_f4<TWO>(p, row, v * T + l);
        }
        float4 acc[C::V];
#pragma unroll
        for (int v = 0; v < C::V; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        spmm_gather<D, T, TWO, DROP>(p, b, valid ? len : 0, maxlen, l, acc, dk);
        bool do_epi = valid && sid < 0;
        const bool split = valid && sid >= 0;
        if (__any_sync(0xffffffffu, split)) {
            if (spmm_split_finish<D, T, TWO>(p, split, row, b, sid, l, acc, accin)) do_epi = true;
        }
        spmm_epilogue<D, T>(p, do_epi, row, l, acc, accin);
    }
}

template <int D, int T>
__global__ void __launch_bounds__(256) spmm_vec_kernel(const SpmmParams p) {
    __shared__ __align__(16) float red[(256 / T) * D];
    spmm_vec_body<D, T, false>(p, red);
}

// K1 with an edge-keep mask (mmrec_spmm_op.keep_bits): the same plan, split rows, segment-order reduction and epilogues, over
// the entries whose keep bit is set, each weighted fl(v * scale) -- SelfCF's per-batch `sparse_dropout` of the normalised
// adjacency (encoders.py:77-88) without rebuilding the matrix.
template <int D, int T>
__global__ void __launch_bounds__(256) spmm_drop_kernel(const SpmmParams p, const uint32_t* __restrict__ keep, float scale) {
    __shared__ __align__(16) float red[(256 / T) * D];
    spmm_vec_body<D, T, false, true>(p, red, DropKeep{keep, scale});
}

// The keep bits of one dropout draw (mmrec_edge_keep_bits): CSR position e is kept iff floor(keep_prob + draws[draw_of[e]])
// != 0 in fp32, and its mirror bit (the transpose's position e) is the bit of position mirror[e].  One thread per position,
// a warp per 32-bit word: the words are assembled by ballot, no atomics.
__global__ void __launch_bounds__(256) edge_keep_bits_kernel(int64_t nnz, const float* __restrict__ draws, float keep_prob,
                                                             const int32_t* __restrict__ draw_of, const int32_t* __restrict__ mirror,
                                                             uint32_t* __restrict__ keep, uint32_t* __restrict__ keep_t) {
    const int64_t n_words = (nnz + 31) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    auto kept = [&](int64_t e) { return floorf(__fadd_rn(keep_prob, __ldg(draws + __ldg(draw_of + e)))) != 0.f; };
    for (int64_t w = w0; w < n_words; w += n_warps) {                // warp-uniform trip count
        const int64_t e = (w << 5) + lane;
        const bool in = e < nnz;
        const uint32_t word = __ballot_sync(0xffffffffu, in && kept(e));
        const uint32_t word_t = keep_t ? __ballot_sync(0xffffffffu, in && kept(__ldg(mirror + e))) : 0u;
        if (lane == 0) {
            keep[w] = word;
            if (keep_t) keep_t[w] = word_t;
        }
    }
}

// Several SpMMs in one persistent launch: the steps run in order on the same grid, a CTA that is done with one step starts
// the next, so the tail of one step overlaps the work of the next.  COOP (a cooperative launch, every CTA resident): a
// grid-wide barrier before every step of `sync_mask` (it reads what an earlier step wrote), so a whole propagation is one
// launch.  Without COOP the steps of one launch must be independent -- FREEDOM's item-item product beside layer 1 on A_hat.
constexpr int SPMM_CHAIN_MAX = 8;
struct SpmmChain { SpmmParams step[SPMM_CHAIN_MAX]; int n; unsigned sync_mask; };

template <int D, int T, bool COOP>
__global__ void __launch_bounds__(256, 3) spmm_chain_kernel(const SpmmChain c) {
    __shared__ __align__(16) float red[(256 / T) * D];
    for (int i = 0; i < c.n; ++i) {
        if (COOP && ((c.sync_mask >> i) & 1u)) { __threadfence(); cooperative_groups::this_grid().sync(); }
        spmm_vec_body<D, T, true>(c.step[i], red);
    }
}

// Any d: 32 columns at a time, scalar loads.  Correctness path for odd widths, not tuned.
__global__ void __launch_bounds__(256) spmm_generic_kernel(const SpmmParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = warp0; row < p.n_rows; row += nwarps) {
        const int b = p.rowptr[row], e = p.rowptr[row + 1];
        float dot = 0.f, ny = 0.f, nr = 0.f;
        if (p.gate_ref) {
            for (int k0 = 0; k0 < p.d; k0 += 32) {
                const int k = k0 + lane;
                float acc = 0.f;
                if (k < p.d)
                    for (int j = b; j < e; ++j) acc = fmaf(p.vals[j], p.X[(int64_t)p.colidx[j] * p.ldx + k], acc);
                float r = k < p.d ? p.gate_ref[row * p.ldgate + k] : 0.f;
                dot += acc * r; ny += acc * acc; nr += r * r;
            }
            dot = warp_sum(dot); ny = warp_sum(ny); nr = warp_sum(nr);
        }
        const float c = p.gate_ref ? dot / (fmaxf(sqrtf(ny), 1e-8f) * fmaxf(sqrtf(nr), 1e-8f)) : 1.f;
        for (int k0 = 0; k0 < p.d; k0 += 32) {
            const int k = k0 + lane;
            if (k >= p.d) continue;
            float acc = 0.f;
            for (int j = b; j < e; ++j) acc = fmaf(p.vals[j], p.X[(int64_t)p.colidx[j] * p.ldx + k], acc);
            if (p.gate_ref) acc *= c;
            if (p.Y) p.Y[row * p.ldy + k] = p.y_acc ? p.Y[row * p.ldy + k] + acc : acc;
            if (p.acc_out) {
                float a = acc + (p.acc_in ? p.acc_in[row * p.ldacc + k] : 0.f);
                if (p.acc_div != 1.0f) a = __fdiv_rn(a, p.acc_div);
                if (p.post && row >= p.post_row0) a += p.post[(row - p.post_row0) * (int64_t)(p.spost / 4) + k];
                p.acc_out[row * p.ldacc + k] = a;
            }
        }
    }
}

int g_spmm_lanes = 0;   // 0 = default lanes per task for the width; set by mmrec_spmm_set_lanes (tuning knob)

template <int D, int T, bool DROP = false>
static int launch_vec(const SpmmParams& p, cudaStream_t stream, const DropKeep dk = DropKeep{nullptr, 1.f}) {
    static int blocks_per_sm = 0;
    if (!blocks_per_sm) {
        if constexpr (DROP) MMREC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, spmm_drop_kernel<D, T>, 256, 0));
        else MMREC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, spmm_vec_kernel<D, T>, 256, 0));
        if (blocks_per_sm < 1) blocks_per_sm = 1;
    }
    const int64_t n_work = p.tasks ? p.n_tasks : p.n_rows;
    const int per_block = 8 * (32 / T);
    int64_t grid = (n_work - p.n_heavy + per_block - 1) / per_block;
    if (grid < p.n_heavy) grid = p.n_heavy;
    const int64_t cap = (int64_t)sm_count() * blocks_per_sm;
    if (grid > cap) grid = cap;
    if (grid < 1) return MMREC_OK;
    if constexpr (DROP) spmm_drop_kernel<D, T><<<(unsigned)grid, 256, 0, stream>>>(p, dk.keep, dk.scale);
    else spmm_vec_kernel<D, T><<<(unsigned)grid, 256, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

template <int D>
static int launch_vec_d(const SpmmParams& p, cudaStream_t stream) {
    constexpr int T4 = D / 4 > 32 ? 32 : D / 4;      // 1 float4 per lane
    constexpr int T8 = D / 8 > 32 ? 32 : D / 8;      // 2 float4 per lane
    constexpr int T16 = D / 16 > 32 ? 32 : D / 16;   // 4 float4 per lane
    int T = g_spmm_lanes ? g_spmm_lanes : T4;       // default: one float4 per lane (measured best at d = 64)
    if (T == T4) return launch_vec<D, T4>(p, stream);
    if (T == T16) return launch_vec<D, T16>(p, stream);
    return launch_vec<D, T8>(p, stream);
}

// The widths 3d (d = 32, 64, 128): three float4 per lane, T = D / 12 -- the lane count of the width-d default (one float4
// per lane at d = D / 3).  Lane l owns float4 v * T + l of a row, so float4 block v is column block v, and every lane group,
// CTA reduction, split-row partial and epilogue sums block v exactly as the width-d kernel sums its row: each column block
// of the width-3d product is the width-d product of that block, bit for bit (not under the cosine gate, which reduces over
// the whole row).  The lane override does not apply to these widths.
template <int D>
static int launch_vec_3d(const SpmmParams& p, cudaStream_t stream) {
    static_assert(VecCfg<D, D / 12>::V == 3, "three float4 per lane");
    return launch_vec<D, D / 12>(p, stream);
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_spmm_set_lanes(int lanes_per_row) {
    MMREC_CHECK_ARG(lanes_per_row == 0 || lanes_per_row == 2 || lanes_per_row == 4 || lanes_per_row == 8 ||
                    lanes_per_row == 16 || lanes_per_row == 32, "spmm_set_lanes: 0 (default) or a power of two <= 32");
    g_spmm_lanes = lanes_per_row;
    return MMREC_OK;
}

extern "C" int mmrec_edge_keep_bits(int64_t nnz, const float* draws, float keep_prob, const int32_t* draw_of, const int32_t* mirror,
                                    uint32_t* keep_bits, uint32_t* keep_bits_t, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(nnz >= 0 && nnz < (1ll << 31), "edge_keep_bits: nnz out of range");
    if (nnz == 0) return MMREC_OK;
    MMREC_CHECK_ARG(draws && draw_of && keep_bits && (!keep_bits_t || mirror), "edge_keep_bits: null pointer");
    const int64_t n_words = (nnz + 31) / 32;
    int64_t grid = (n_words + 7) / 8;                 // 8 warps per block, one word per warp
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    edge_keep_bits_kernel<<<(unsigned)grid, 256, 0, stream>>>(nnz, draws, keep_prob, draw_of, mirror, keep_bits, keep_bits_t);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

namespace mmrec {
// One launch of the chained kernel; COOP: cooperative, so that every CTA is resident for the grid barriers.
template <int D, bool COOP>
static int launch_chain(const SpmmChain& c, cudaStream_t stream) {
    constexpr int T = D / 4 > 32 ? 32 : D / 4;                       // one float4 per lane, as the single-step default
    static int blocks_per_sm = 0;
    if (!blocks_per_sm) {
        MMREC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, spmm_chain_kernel<D, T, COOP>, 256, 0));
        if (blocks_per_sm < 1) blocks_per_sm = 1;
    }
    int64_t max_work = 1;
    for (int i = 0; i < c.n; ++i) {
        const int64_t work = c.step[i].n_tasks > c.step[i].n_heavy ? c.step[i].n_tasks : c.step[i].n_heavy * 8;
        if (work > max_work) max_work = work;
    }
    const int per_block = 8 * (32 / T);
    int64_t grid = (max_work + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count() * blocks_per_sm;         // every block resident (the grid barrier needs it)
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    if (COOP) {
        void* args[] = {(void*)&c};
        MMREC_CUDA(cudaLaunchCooperativeKernel((const void*)spmm_chain_kernel<D, T, true>, dim3((unsigned)grid), dim3(256), args, 0, stream));
        ++g_launches;
    } else {
        spmm_chain_kernel<D, T, false><<<(unsigned)grid, 256, 0, stream>>>(c);
        MMREC_LAUNCH_CHECK();
    }
    return MMREC_OK;
}

// Without the cooperative launch, each run of steps up to the next `sync_before` is one ordinary launch; a run of one step
// with one-block operands is the single-SpMM kernel (the chained kernel reads its parameters by a run-time step index).
template <int D>
static int launch_steps(const SpmmChain& c, int cooperative, cudaStream_t stream) {
    if (cooperative) return launch_chain<D, true>(c, stream);
    constexpr int T = D / 4 > 32 ? 32 : D / 4;
    for (int i = 0; i < c.n;) {
        int j = i + 1;
        while (j < c.n && !((c.sync_mask >> j) & 1u)) ++j;
        const SpmmParams& p = c.step[i];
        int rc;
        if (j == i + 1 && p.x_split == p.n_cols && p.acc_split == p.n_rows) {
            rc = launch_vec<D, T>(p, stream);
        } else {
            SpmmChain run;
            run.n = j - i; run.sync_mask = 0;
            for (int k = 0; k < run.n; ++k) run.step[k] = c.step[i + k];
            rc = launch_chain<D, false>(run, stream);
        }
        if (rc != MMREC_OK) return rc;
        i = j;
    }
    return MMREC_OK;
}

// The checks of one op and its parameter block.  chain: the chained kernel's limits (every op needs its work plan).  Sets
// vec_ok when the operands are 16-byte aligned (the vector kernels' float4 rows).
static int spmm_op_params(const mmrec_spmm_op& o, int i, int d, bool chain, SpmmParams& p, bool& vec_ok) {
    MMREC_CHECK_ARG(o.n_rows >= 0 && o.n_cols >= 0 && o.rowptr && o.X && (o.Y || o.acc_out), "spmm: op %d: null pointer / bad sizes", i);
    MMREC_CHECK_ARG(o.tasks ? (o.n_tasks >= 0 && o.n_cta_tasks >= 0 && o.n_cta_tasks <= o.n_tasks && o.split_rows && o.counters && o.partial)
                            : !chain,
                    "spmm: op %d: work plan pointers missing (the chained kernel needs the plan of mmrec_spmm_plan)", i);
    MMREC_CHECK_ARG(o.ldx >= d && (!o.Y || o.ldy >= d) && (!o.acc_out || o.ldacc >= d) && (!o.gate_ref || o.ldgate >= d) &&
                    (!o.post || o.ldpost >= d) && o.acc_div != 0.0f, "spmm: op %d: leading dimension < d or acc_div == 0", i);
    MMREC_CHECK_ARG(!(o.y_accumulate && o.gate_ref), "spmm: y_accumulate does not combine with the cosine gate");
    MMREC_CHECK_ARG(o.ldx < (1ll << 30) && o.ldy < (1ll << 30) && o.ldacc < (1ll << 30) && o.ldgate < (1ll << 30) && o.ldpost < (1ll << 30) &&
                    o.n_cols < (1ll << 31) && o.n_rows < (1ll << 31), "spmm: op %d: leading dimension / size out of range", i);
    MMREC_CHECK_ARG(!o.X_hi || (o.x_split >= 0 && o.x_split <= o.n_cols && o.ldx_hi >= d && o.ldx_hi < (1ll << 30)),
                    "spmm: op %d: X_hi needs 0 <= x_split <= n_cols and d <= ldx_hi < 2^30", i);
    MMREC_CHECK_ARG(!o.acc_in_hi || (o.acc_in && o.acc_out && o.acc_in_split >= 0 && o.acc_in_split <= o.n_rows && o.ldacc_in_hi >= d &&
                                     o.ldacc_in_hi < (1ll << 30)),
                    "spmm: op %d: acc_in_hi needs acc_in, acc_out, 0 <= acc_in_split <= n_rows and d <= ldacc_in_hi < 2^30", i);
    p.n_rows = o.n_rows; p.n_cols = o.n_cols; p.rowptr = o.rowptr; p.colidx = o.colidx; p.vals = o.vals;
    p.tasks = (const int4*)o.tasks; p.n_tasks = o.n_tasks; p.n_heavy = o.tasks ? o.n_cta_tasks : 0; p.split_rows = (const int4*)o.split_rows;
    p.counters = o.counters; p.partial = o.partial; p.X = o.X; p.ldx = o.ldx; p.Y = o.Y; p.ldy = o.ldy; p.y_acc = o.y_accumulate != 0;
    p.acc_in = o.acc_in; p.acc_out = o.acc_out; p.ldacc = o.ldacc; p.acc_div = o.acc_div; p.gate_ref = o.gate_ref; p.ldgate = o.ldgate;
    p.post = o.post; p.post_row0 = o.post_row0; p.d = d;
    p.sx = (uint32_t)(o.ldx * 4); p.sy = (uint32_t)(o.ldy * 4); p.sacc = (uint32_t)(o.ldacc * 4); p.sgate = (uint32_t)(o.ldgate * 4);
    p.spost = (uint32_t)(o.ldpost * 4);
    p.X_hi = o.X_hi ? o.X_hi : o.X;
    p.x_split = (int)(o.X_hi ? o.x_split : o.n_cols);
    p.sx_hi = (uint32_t)((o.X_hi ? o.ldx_hi : o.ldx) * 4);
    p.acc_in_hi = o.acc_in_hi ? o.acc_in_hi : o.acc_in;
    p.acc_split = (int)(o.acc_in_hi ? o.acc_in_split : o.n_rows);
    p.sacc_hi = (uint32_t)((o.acc_in_hi ? o.ldacc_in_hi : o.ldacc) * 4);
    auto al16 = [](const void* q, int64_t ld) { return q == nullptr || ((((uintptr_t)q) & 15) == 0 && (ld & 3) == 0); };
    vec_ok = al16(o.X, o.ldx) && al16(o.Y, o.ldy) && al16(o.acc_in, o.ldacc) && al16(o.acc_out, o.ldacc) && al16(o.gate_ref, o.ldgate) &&
             al16(o.post, o.ldpost) && al16(o.partial, 4) && al16(o.X_hi, o.ldx_hi) && al16(o.acc_in_hi, o.ldacc_in_hi);
    return MMREC_OK;
}
}  // namespace mmrec

extern "C" int mmrec_spmm_run_f32(int d, int n_ops, const mmrec_spmm_op* ops, int cooperative, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(n_ops >= 1 && n_ops <= SPMM_CHAIN_MAX && ops, "spmm: 1 <= n_ops <= %d", SPMM_CHAIN_MAX);
    const bool vec_d = d == 32 || d == 64 || d == 128 || d == 256;
    bool chain = n_ops > 1 || cooperative;
    for (int i = 0; i < n_ops; ++i) chain = chain || ops[i].X_hi || ops[i].acc_in_hi || ops[i].post || ops[i].sync_before;
    if (chain) {
        if (!vec_d || g_spmm_lanes) {
            set_error("spmm: d = %d (or a lane override) has no chained kernel; run the ops one by one", d);
            return MMREC_EUNSUPPORTED;
        }
        SpmmChain c;
        c.n = n_ops; c.sync_mask = 0;
        for (int i = 0; i < n_ops; ++i) {
            const mmrec_spmm_op& o = ops[i];
            if (o.gate_ref || o.keep_bits || o.y_accumulate) {
                set_error("spmm: op %d: the chained kernel has no cosine gate, edge-keep mask or accumulating Y", i);
                return MMREC_EUNSUPPORTED;
            }
            bool vec_ok = false;
            const int rc = spmm_op_params(o, i, d, true, c.step[i], vec_ok);
            if (rc != MMREC_OK) return rc;
            if (!vec_ok) {
                set_error("spmm: op %d: operands not 16-byte aligned; run the ops one by one", i);
                return MMREC_EUNSUPPORTED;
            }
            if (o.sync_before && i > 0) c.sync_mask |= 1u << i;
        }
        switch (d) {
            case 32: return launch_steps<32>(c, cooperative, stream);
            case 64: return launch_steps<64>(c, cooperative, stream);
            case 128: return launch_steps<128>(c, cooperative, stream);
            default: return launch_steps<256>(c, cooperative, stream);
        }
    }
    const mmrec_spmm_op& o = ops[0];
    MMREC_CHECK_ARG(o.n_rows >= 0 && o.n_cols >= 0 && d >= 1, "spmm: bad sizes");
    if (o.n_rows == 0) return MMREC_OK;
    if (o.keep_bits && (o.gate_ref || o.y_accumulate)) {
        set_error("spmm: the edge-keep mask does not combine with the cosine gate or an accumulating Y");
        return MMREC_EUNSUPPORTED;
    }
    SpmmParams p;
    bool vec_ok = false;
    const int rc = spmm_op_params(o, 0, d, false, p, vec_ok);
    if (rc != MMREC_OK) return rc;
    if (o.keep_bits) {
        if (!vec_ok || !vec_d) {
            set_error("spmm: d = %d or unaligned operands: the masked kernel is built for 16-byte aligned d in {32, 64, 128, 256}", d);
            return MMREC_EUNSUPPORTED;
        }
        const DropKeep dk{o.keep_bits, o.keep_scale};
        switch (d) {                                      // one float4 per lane, the default of the unmasked kernel
            case 32: return launch_vec<32, 8, true>(p, stream, dk);
            case 64: return launch_vec<64, 16, true>(p, stream, dk);
            case 128: return launch_vec<128, 32, true>(p, stream, dk);
            default: return launch_vec<256, 32, true>(p, stream, dk);
        }
    }
    if (vec_ok) {
        switch (d) {
            case 32: return launch_vec_d<32>(p, stream);
            case 64: return launch_vec_d<64>(p, stream);
            case 128: return launch_vec_d<128>(p, stream);
            case 256: return launch_vec_d<256>(p, stream);
            case 96: return launch_vec_3d<96>(p, stream);
            case 192: return launch_vec_3d<192>(p, stream);
            case 384: return launch_vec_3d<384>(p, stream);
            default: break;
        }
    }
    p.tasks = nullptr;   // the generic kernel walks whole rows
    int64_t grid = (o.n_rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    spmm_generic_kernel<<<(unsigned)grid, 256, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
