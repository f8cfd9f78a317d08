// n14 -- PGL's loss after the tables (src/models/pgl.py:227-259) as one row kernel each way plus a one-CTA finish, instead
// of the torch chain of three gathers, two row dots, logsigmoid, four dropouts, four F.normalize, two positive dots, the
// InfoNCE element-wise steps and their autograd (about forty small launches each way):
//
//   x_b   = <u_b, p_b> - <u_b, n_b>,  u_b = UA[users[b]], p_b = IA[pos[b]], n_b = IA[neg[b]]
//   mf    = -(sum_b logsigmoid(x_b)) / B
//   a, b, c, d = drop(u; m0), drop(u; m1), drop(p; m2), drop(p; m3)      drop(s; m) = (s * m) * scale, as ATen's fused dropout
//   InfoNCE(v, w) = (sum_b -log(exp(<v^_b, w^_b> / 0.2) / ttl_b)) / B,  ttl_b = sum_j exp(<v^_b, w^_j> / 0.2),  v^ = F.normalize(v)
//   loss  = mf + reg_weight * ((InfoNCE(a, b) + InfoNCE(c, d)) / 2)
//
// The B x B sums ttl are K8's (ops.expsum_rows, forward and backward): the row kernel writes the four normalised views it
// reads, and the finish kernel combines K8's two [B] sums with the rows' terms.  A warp owns one row, lane j the columns
// j*V .. j*V + V-1 of each 32*V-column chunk (V = 4 at d = 128, 2 at d = 64, 1 at other widths).  Every element-wise step
// is torch's on the device, one IEEE rounding per step (__fadd_rn / __fmul_rn / __fdiv_rn: nothing is contracted):
//  - logsigmoid is ATen's `min(0, x) - log1p(exp(-|x|))`, its backward `g * (max_deriv - sign * (z / (1 + z)))`;
//  - a division by a Python number (`/ 0.2`, `/ 2`, the means' `/ B`) is a multiplication by its fp32 reciprocal, forward
//    and backward (BinaryDivTrueKernel);
//  - F.normalize is `x / clamp_min(||x||, 1e-12)`; its backward is the division's two gradients, the sum over the row of
//    the denominator's, clamp_min's `where(norm >= eps, g, 0)` and the norm's `g * (x / norm)` (0 where norm == 0);
//  - dropout's backward is `(g * m) * scale` with the backward's own scale, fp32(1 / (1 - p)) (native_dropout_backward);
//  - a row's gradients add in autograd's order: the two InfoNCE views first, then the negative and the positive BPR term.
// The dots, sums of squares and the normaliser's row sum run in this kernel's own order (lane-strided fmaf, then a fixed
// xor butterfly), so where they are exact every per-row result equals the torch expression's bits.  The batch sums are one
// CTA's, in a fixed order: no atomics, the same bits on every run.  reg_weight == 0 (PGL's default): the views, K8 and
// the InfoNCE arithmetic are skipped -- `0 * cl` and its gradient add exact zeros while every input is finite.
#include <cuda_runtime.h>

#include "common.cuh"

namespace mmrec {

constexpr int PG_WARPS = 8;
constexpr int PG_FIN_THREADS = 512;

struct PglParams {
    int64_t B;
    int d;
    const float *UA, *IA;
    const int64_t *users, *pos, *neg;
    const uint8_t* m[4];                // bool masks [B, d] of the views a, b, c, d; all null: keep every entry
    float scale;                        // the dropout's forward scale (the backward recomputes the views with it)
    float scale_bwd;                    // backward: the dropout backward's scale
    float* x;                           // [B]
    float* v[4];                        // forward: the normalised views [B, d]; all null without the InfoNCE terms
    float* vnorm;                       // [4, B]: ||view||, before clamp_min
    float* pd;                          // [2, B]: <a^, b^>, <c^, d^>
    const float* gx;                    // backward: [B]
    const float* gpd;                   // backward: [2, B]
    const float* gv[4];                 // backward: K8's gradients of the views; all null without the InfoNCE terms
    float *gU, *gI;                     // backward: [B, d], [2B, d] ([pos rows; neg rows])
};

template <int V>
__device__ __forceinline__ void pg_load(float (&r)[V], const float* __restrict__ p) {
    if constexpr (V == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p));
        r[0] = t.x; r[1] = t.y; r[2] = t.z; r[3] = t.w;
    } else if constexpr (V == 2) {
        const float2 t = __ldg(reinterpret_cast<const float2*>(p));
        r[0] = t.x; r[1] = t.y;
    } else {
        r[0] = __ldg(p);
    }
}

template <int V>
__device__ __forceinline__ void pg_store(float* p, const float (&r)[V]) {
    if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(r[0], r[1], r[2], r[3]);
    else if constexpr (V == 2) *reinterpret_cast<float2*>(p) = make_float2(r[0], r[1]);
    else p[0] = r[0];
}

// V mask bytes as 0.f / 1.f; a null mask keeps everything
template <int V>
__device__ __forceinline__ void pg_mask(float (&r)[V], const uint8_t* m, int64_t off) {
    if (m == nullptr) {
#pragma unroll
        for (int j = 0; j < V; ++j) r[j] = 1.f;
        return;
    }
    if constexpr (V == 4) {
        const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(m + off));
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = ((w >> (8 * j)) & 0xffu) ? 1.f : 0.f;
    } else if constexpr (V == 2) {
        const uint16_t w = __ldg(reinterpret_cast<const unsigned short*>(m + off));
        r[0] = (w & 0xffu) ? 1.f : 0.f;
        r[1] = (w >> 8) ? 1.f : 0.f;
    } else {
        r[0] = __ldg(m + off) ? 1.f : 0.f;
    }
}

__device__ __forceinline__ float pg_eps() { return static_cast<float>(1e-12); }               // F.normalize's eps in fp32
__device__ __forceinline__ float pg_clamp(float n) { return isnan(n) ? n : (n < pg_eps() ? pg_eps() : n); }
__device__ __forceinline__ float pg_inv_tau() { return 5.f; }                                    // fl(1 / fp32(0.2))

// ATen's log_sigmoid forward and the factor of its backward
__device__ __forceinline__ float pg_logsig(float x) {
    const float mn = x < 0.f ? x : 0.f;
    return __fsub_rn(mn, log1pf(expf(-fabsf(x))));
}
__device__ __forceinline__ float pg_logsig_bwd(float x, float g) {
    const float z = expf(-fabsf(x));
    const float t = __fdiv_rn(z, __fadd_rn(1.f, z));
    return __fmul_rn(g, x < 0.f ? __fsub_rn(1.f, t) : t);
}

// the four dropped rows' columns k .. k + V-1: a, b from u, c, d from p
template <int V>
__device__ __forceinline__ void pg_views(float (&w)[4][V], const PglParams& p, const float (&u)[V], const float (&pv)[V], int64_t off) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float m[V];
        pg_mask<V>(m, p.m[q], off);
#pragma unroll
        for (int j = 0; j < V; ++j) w[q][j] = __fmul_rn(__fmul_rn(q < 2 ? u[j] : pv[j], m[j]), p.scale);
    }
}

template <int V>
__global__ void __launch_bounds__(32 * PG_WARPS, 2) pgl_rows_kernel(const PglParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool cl = p.v[0] != nullptr;
    for (int64_t b = (int64_t)blockIdx.x * PG_WARPS + warp; b < p.B; b += (int64_t)gridDim.x * PG_WARPS) {
        const float* urow = p.UA + __ldg(p.users + b) * p.d;
        const float* prow = p.IA + __ldg(p.pos + b) * p.d;
        const float* nrow = p.IA + __ldg(p.neg + b) * p.d;
        float dpos = 0.f, dneg = 0.f, ss[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = lane * V; k < p.d; k += 32 * V) {
            float u[V], pv[V], nv[V];
            pg_load<V>(u, urow + k);
            pg_load<V>(pv, prow + k);
            pg_load<V>(nv, nrow + k);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                dpos = fmaf(u[j], pv[j], dpos);
                dneg = fmaf(u[j], nv[j], dneg);
            }
            if (cl) {
                float w[4][V];
                pg_views<V>(w, p, u, pv, b * p.d + k);
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int j = 0; j < V; ++j) ss[q] = fmaf(w[q][j], w[q][j], ss[q]);
            }
        }
        const float x = __fsub_rn(warp_sum(dpos), warp_sum(dneg));
        if (lane == 0) p.x[b] = x;
        if (!cl) continue;
        float nrm[4], den[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            nrm[q] = sqrtf(warp_sum(ss[q]));
            den[q] = pg_clamp(nrm[q]);
        }
        float d0 = 0.f, d1 = 0.f;
        for (int k = lane * V; k < p.d; k += 32 * V) {
            float u[V], pv[V], w[4][V];
            pg_load<V>(u, urow + k);
            pg_load<V>(pv, prow + k);
            pg_views<V>(w, p, u, pv, b * p.d + k);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
#pragma unroll
                for (int j = 0; j < V; ++j) w[q][j] = __fdiv_rn(w[q][j], den[q]);
                pg_store<V>(p.v[q] + b * p.d + k, w[q]);
            }
#pragma unroll
            for (int j = 0; j < V; ++j) {
                d0 = fmaf(w[0][j], w[1][j], d0);
                d1 = fmaf(w[2][j], w[3][j], d1);
            }
        }
        d0 = warp_sum(d0);
        d1 = warp_sum(d1);
        if (lane == 0) {
#pragma unroll
            for (int q = 0; q < 4; ++q) p.vnorm[q * p.B + b] = nrm[q];
            p.pd[b] = d0;
            p.pd[p.B + b] = d1;
        }
    }
}

// -log(exp(pd / 0.2) / ttl), torch's steps
__device__ __forceinline__ float pg_nce_row(float pd, float ttl) {
    const float pe = expf(__fmul_rn(pd, pg_inv_tau()));
    return -logf(__fdiv_rn(pe, ttl));
}

// one CTA: the three batch sums in a fixed order (thread-strided, then the warps' butterflies, then warp 0 over the warps),
// and the 0-dim loss
__global__ void __launch_bounds__(PG_FIN_THREADS) pgl_finish_kernel(int64_t B, const float* __restrict__ x, const float* __restrict__ pd,
                                                                    const float* __restrict__ ttl1, const float* __restrict__ ttl2,
                                                                    float rw, float inv_b, float* loss) {
    __shared__ float red[PG_FIN_THREADS / 32][3];
    const bool cl = ttl1 != nullptr;
    float s[3] = {0.f, 0.f, 0.f};
    for (int64_t b = threadIdx.x; b < B; b += PG_FIN_THREADS) {
        s[0] = __fadd_rn(s[0], pg_logsig(x[b]));
        if (cl) {
            s[1] = __fadd_rn(s[1], pg_nce_row(pd[b], ttl1[b]));
            s[2] = __fadd_rn(s[2], pg_nce_row(pd[B + b], ttl2[b]));
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int q = 0; q < 3; ++q) s[q] = warp_sum(s[q]);
    if (lane == 0) { red[warp][0] = s[0]; red[warp][1] = s[1]; red[warp][2] = s[2]; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    float t[3] = {0.f, 0.f, 0.f};
    for (int w = 0; w < PG_FIN_THREADS / 32; ++w)
#pragma unroll
        for (int q = 0; q < 3; ++q) t[q] = __fadd_rn(t[q], red[w][q]);
    const float mf = -__fmul_rn(t[0], inv_b);
    const float c = cl ? __fmul_rn(__fadd_rn(__fmul_rn(t[1], inv_b), __fmul_rn(t[2], inv_b)), 0.5f) : 0.f;
    *loss = __fadd_rn(mf, __fmul_rn(rw, c));
}

// per row: the BPR gradient gx, and for each InfoNCE pair the positive dot's gradient gpd and K8's upstream gradient gttl
__global__ void __launch_bounds__(256) pgl_finish_bwd_kernel(int64_t B, const float* __restrict__ x, const float* __restrict__ pd,
                                                             const float* __restrict__ ttl1, const float* __restrict__ ttl2, float rw,
                                                             float inv_b, const float* __restrict__ g, float* gx, float* gpd, float* gttl) {
    const float gl = __ldg(g);
    const float gm = __fmul_rn(-gl, inv_b);                                        // neg, then mean backward
    const float gc = __fmul_rn(__fmul_rn(__fmul_rn(gl, rw), 0.5f), inv_b);         // `reg_weight *`, `/ 2`, mean backward
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        gx[b] = pg_logsig_bwd(x[b], gm);
        if (ttl1 == nullptr) continue;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const float ttl = t ? ttl2[b] : ttl1[b];
            const float pe = expf(__fmul_rn(pd[t * B + b], pg_inv_tau()));
            const float r = __fdiv_rn(pe, ttl);
            const float gr = __fdiv_rn(-gc, r);                                        // neg, then log backward
            const float gpe = __fdiv_rn(gr, ttl);                                      // div backward, numerator
            gttl[t * B + b] = __fmul_rn(-gr, __fdiv_rn(r, ttl));                       // div backward, denominator
            gpd[t * B + b] = __fmul_rn(__fmul_rn(gpe, pe), pg_inv_tau());              // exp backward, `/ 0.2` backward
        }
    }
}

template <int V>
__device__ __forceinline__ void pg_ghat(float (&gh)[4][V], const PglParams& p, const float (&w)[4][V], const float (&den)[4],
                                        float gp0, float gp1, int64_t off) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float k8[V];
        pg_load<V>(k8, p.gv[q] + off);
        const float gpq = q < 2 ? gp0 : gp1;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const float other = __fdiv_rn(w[q ^ 1][j], den[q ^ 1]);                     // the partner view's normalised entry
            gh[q][j] = __fadd_rn(k8[j], __fmul_rn(gpq, other));
        }
    }
}

template <int V>
__global__ void __launch_bounds__(32 * PG_WARPS) pgl_rows_bwd_kernel(const PglParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool cl = p.gv[0] != nullptr;
    for (int64_t b = (int64_t)blockIdx.x * PG_WARPS + warp; b < p.B; b += (int64_t)gridDim.x * PG_WARPS) {
        const float* urow = p.UA + __ldg(p.users + b) * p.d;
        const float* prow = p.IA + __ldg(p.pos + b) * p.d;
        const float* nrow = p.IA + __ldg(p.neg + b) * p.d;
        const float gxb = __ldg(p.gx + b), gy = -gxb;                                 // sub backward: the negative dot's
        float nrm[4], den[4], gnorm[4] = {0.f, 0.f, 0.f, 0.f}, gp0 = 0.f, gp1 = 0.f;
        if (cl) {
            gp0 = __ldg(p.gpd + b);
            gp1 = __ldg(p.gpd + p.B + b);
            float sd[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                nrm[q] = __ldg(p.vnorm + q * p.B + b);
                den[q] = pg_clamp(nrm[q]);
            }
            for (int k = lane * V; k < p.d; k += 32 * V) {                          // the denominators' gradients
                float u[V], pv[V], w[4][V], gh[4][V];
                pg_load<V>(u, urow + k);
                pg_load<V>(pv, prow + k);
                pg_views<V>(w, p, u, pv, b * p.d + k);
                pg_ghat<V>(gh, p, w, den, gp0, gp1, b * p.d + k);
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int j = 0; j < V; ++j)
                        sd[q] = __fadd_rn(sd[q], __fmul_rn(-gh[q][j], __fdiv_rn(__fdiv_rn(w[q][j], den[q]), den[q])));
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float gd = warp_sum(sd[q]);
                gnorm[q] = nrm[q] >= pg_eps() ? gd : 0.f;                                // clamp_min backward
            }
        }
        for (int k = lane * V; k < p.d; k += 32 * V) {
            float u[V], pv[V], nv[V], hu[V], hp[V], hn[V];
            pg_load<V>(u, urow + k);
            pg_load<V>(pv, prow + k);
            pg_load<V>(nv, nrow + k);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                hu[j] = __fadd_rn(__fmul_rn(gy, nv[j]), __fmul_rn(gxb, pv[j]));
                hp[j] = __fmul_rn(gxb, u[j]);
                hn[j] = __fmul_rn(gy, u[j]);
            }
            if (cl) {
                float w[4][V], gh[4][V], gs[4][V];
                pg_views<V>(w, p, u, pv, b * p.d + k);
                pg_ghat<V>(gh, p, w, den, gp0, gp1, b * p.d + k);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float m[V];
                    pg_mask<V>(m, p.m[q], b * p.d + k);
#pragma unroll
                    for (int j = 0; j < V; ++j) {
                        const float qn = nrm[q] == 0.f ? 0.f : __fdiv_rn(w[q][j], nrm[q]);
                        const float gxv = __fadd_rn(__fdiv_rn(gh[q][j], den[q]), __fmul_rn(gnorm[q], qn));
                        gs[q][j] = __fmul_rn(__fmul_rn(gxv, m[j]), p.scale_bwd);             // dropout backward
                    }
                }
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    hu[j] = __fadd_rn(__fadd_rn(__fadd_rn(gs[1][j], gs[0][j]), __fmul_rn(gy, nv[j])), __fmul_rn(gxb, pv[j]));
                    hp[j] = __fadd_rn(__fadd_rn(gs[3][j], gs[2][j]), __fmul_rn(gxb, u[j]));
                }
            }
            pg_store<V>(p.gU + b * p.d + k, hu);
            pg_store<V>(p.gI + b * p.d + k, hp);
            pg_store<V>(p.gI + (p.B + b) * p.d + k, hn);
        }
    }
}

static int64_t pgl_grid(int64_t B) {
    int64_t g = (B + PG_WARPS - 1) / PG_WARPS;
    const int64_t cap = 8 * (int64_t)sm_count();
    return g < 1 ? 1 : (g > cap ? cap : g);
}

static bool pg_aligned(const void* q, int bytes) { return q == nullptr || ((uintptr_t)q % bytes) == 0; }

// 4 at widths of 128k columns, 2 at 64k, else 1
static int pgl_vec(const PglParams& p) {
    for (int V : {4, 2}) {
        const int bytes = 4 * V;
        bool ok = p.d % (32 * V) == 0 && pg_aligned(p.UA, bytes) && pg_aligned(p.IA, bytes) && pg_aligned(p.x, 4);
        for (int q = 0; q < 4; ++q)
            ok = ok && pg_aligned(p.m[q], V) && pg_aligned(p.v[q], bytes) && pg_aligned(p.gv[q], bytes);
        ok = ok && pg_aligned(p.gU, bytes) && pg_aligned(p.gI, bytes);
        if (ok) return V;
    }
    return 1;
}

static int pgl_check(const char* what, int64_t B, int d, const float* UA, const float* IA, const int64_t* users, const int64_t* pos,
                     const int64_t* neg, const uint8_t* const* m) {
    MMREC_CHECK_ARG(B >= 1, "%s: B = %lld, the loss needs at least one row", what, (long long)B);
    MMREC_CHECK_ARG(d >= 1, "%s: d = %d", what, d);
    MMREC_CHECK_ARG(UA && IA && users && pos && neg, "%s: null UA, IA, users, pos or neg", what);
    const bool any = m[0] || m[1] || m[2] || m[3], all = m[0] && m[1] && m[2] && m[3];
    MMREC_CHECK_ARG(!any || all, "%s: give all four masks or none", what);
    return MMREC_OK;
}

static PglParams pgl_params(int64_t B, int d, const float* UA, const float* IA, const int64_t* users, const int64_t* pos,
                            const int64_t* neg, const uint8_t* const* m, float scale) {
    PglParams p{};
    p.B = B;
    p.d = d;
    p.UA = UA;
    p.IA = IA;
    p.users = users;
    p.pos = pos;
    p.neg = neg;
    for (int q = 0; q < 4; ++q) p.m[q] = m[q];
    p.scale = scale;
    return p;
}

}  // namespace mmrec

using namespace mmrec;

extern "C" int mmrec_pgl_rows_f32(int64_t B, int d, const float* UA, const float* IA, const int64_t* users, const int64_t* pos,
                                  const int64_t* neg, const uint8_t* m0, const uint8_t* m1, const uint8_t* m2, const uint8_t* m3,
                                  float scale, float* x, float* va, float* vb, float* vc, float* vd, float* vnorm, float* pd,
                                  void* stream_) {
    const uint8_t* m[4] = {m0, m1, m2, m3};
    int rc = pgl_check("pgl_rows", B, d, UA, IA, users, pos, neg, m);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(x, "pgl_rows: null x");
    const bool any = va || vb || vc || vd || vnorm || pd, all = va && vb && vc && vd && vnorm && pd;
    MMREC_CHECK_ARG(!any || all, "pgl_rows: give all four views, vnorm and pd, or none");
    PglParams p = pgl_params(B, d, UA, IA, users, pos, neg, m, scale);
    p.x = x;
    p.v[0] = va; p.v[1] = vb; p.v[2] = vc; p.v[3] = vd;
    p.vnorm = vnorm;
    p.pd = pd;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)pgl_grid(B);
    const int V = pgl_vec(p);
    if (V == 4) pgl_rows_kernel<4><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    else if (V == 2) pgl_rows_kernel<2><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    else pgl_rows_kernel<1><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_pgl_finish_f32(int64_t B, const float* x, const float* pd, const float* ttl1, const float* ttl2, float reg_weight,
                                    float* loss, void* stream_) {
    MMREC_CHECK_ARG(B >= 1, "pgl_finish: B = %lld, the loss needs at least one row", (long long)B);
    MMREC_CHECK_ARG(x && loss, "pgl_finish: null x or loss");
    MMREC_CHECK_ARG((pd && ttl1 && ttl2) || (!pd && !ttl1 && !ttl2), "pgl_finish: give pd, ttl1 and ttl2, or none");
    pgl_finish_kernel<<<1, PG_FIN_THREADS, 0, (cudaStream_t)stream_>>>(B, x, pd, ttl1, ttl2, reg_weight, 1.f / (float)B, loss);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_pgl_finish_bwd_f32(int64_t B, const float* x, const float* pd, const float* ttl1, const float* ttl2,
                                        float reg_weight, const float* g, float* gx, float* gpd, float* gttl, void* stream_) {
    MMREC_CHECK_ARG(B >= 1, "pgl_finish_bwd: B = %lld, the loss needs at least one row", (long long)B);
    MMREC_CHECK_ARG(x && g && gx, "pgl_finish_bwd: null x, g or gx");
    const bool any = pd || ttl1 || ttl2 || gpd || gttl, all = pd && ttl1 && ttl2 && gpd && gttl;
    MMREC_CHECK_ARG(!any || all, "pgl_finish_bwd: give pd, ttl1, ttl2, gpd and gttl, or none");
    int64_t grid = (B + 255) / 256;
    const int64_t cap = 4 * (int64_t)sm_count();
    grid = grid > cap ? cap : grid;
    pgl_finish_bwd_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream_>>>(B, x, pd, ttl1, ttl2, reg_weight, 1.f / (float)B, g, gx,
                                                                             gpd, gttl);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_pgl_rows_bwd_f32(int64_t B, int d, const float* UA, const float* IA, const int64_t* users, const int64_t* pos,
                                      const int64_t* neg, const uint8_t* m0, const uint8_t* m1, const uint8_t* m2, const uint8_t* m3,
                                      float scale_bwd, float scale, const float* gx, const float* vnorm, const float* gpd,
                                      const float* gva, const float* gvb, const float* gvc, const float* gvd, float* gU, float* gI,
                                      void* stream_) {
    const uint8_t* m[4] = {m0, m1, m2, m3};
    int rc = pgl_check("pgl_rows_bwd", B, d, UA, IA, users, pos, neg, m);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(gx && gU && gI, "pgl_rows_bwd: null gx, gU or gI");
    const bool any = vnorm || gpd || gva || gvb || gvc || gvd, all = vnorm && gpd && gva && gvb && gvc && gvd;
    MMREC_CHECK_ARG(!any || all, "pgl_rows_bwd: give vnorm, gpd and the four view gradients, or none");
    // the views are recomputed with the forward's scale; the dropout's backward multiplies by its own
    PglParams p = pgl_params(B, d, UA, IA, users, pos, neg, m, scale);
    p.scale_bwd = scale_bwd;
    p.gx = gx;
    p.vnorm = const_cast<float*>(vnorm);
    p.gpd = gpd;
    p.gv[0] = gva; p.gv[1] = gvb; p.gv[2] = gvc; p.gv[3] = gvd;
    p.gU = gU;
    p.gI = gI;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)pgl_grid(B);
    const int V = pgl_vec(p);
    if (V == 4) pgl_rows_bwd_kernel<4><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    else if (V == 2) pgl_rows_bwd_kernel<2><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    else pgl_rows_bwd_kernel<1><<<grid, 32 * PG_WARPS, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
