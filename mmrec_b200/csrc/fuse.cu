// a5b -- MGCN's row-wise fusion (src/models/mgcn.py:153-154,187-201) as two kernels instead of ~15 eager element-wise /
// small-GEMM launches over [n_users + n_items, d] tensors:
//
//   gate_rows   out[n,:] = mul[n,:] * sigmoid(X[n,:] W^T + b)              -- `item_id_embedding.weight * gate_v(image_feats)`
//   mgcn_fuse   per row: attention of the two modality views (query_common: Linear -> Tanh -> Linear(d,1), softmax over the
//               two logits), common = w0 img + w1 txt, preference gates on the content embedding, side = (sep_img + sep_txt +
//               common) / 3, out = content + side.
//
// Every row is independent; the d x d weights live in shared memory (transposed, padded), a warp owns 4 rows at a time, a
// lane owns d/32 output features.  Bandwidth-trivial (3 reads + 1 write of [N, d]); the point is the launch count and the
// intermediate tensors that no longer exist.  fp32 fmaf chains, tanhf / expf of the CUDA math library, IEEE division.
#include <cuda_runtime.h>

#include "common.cuh"

namespace mmrec {

constexpr int FR = 4;                 // rows per warp iteration

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// Wt[k * (D + 1) + j] = W[j * D + k]
template <int D>
__device__ __forceinline__ void load_weight_t(float* Wt, const float* __restrict__ W) {
    for (int e = threadIdx.x; e < D * D; e += blockDim.x) {
        const int j = e / D, k = e - j * D;
        Wt[k * (D + 1) + j] = __ldg(W + e);
    }
}

// rows row0 .. row0+3 of X (leading dimension D) -> xs[k * FR + r]; rows beyond n read as zero
template <int D>
__device__ __forceinline__ void stage_rows(float* xs, const float* __restrict__ X, int64_t row0, int64_t n, int lane) {
#pragma unroll
    for (int r = 0; r < FR; ++r)
#pragma unroll
        for (int jt = 0; jt < D / 32; ++jt) {
            const int k = lane + 32 * jt;
            xs[k * FR + r] = (row0 + r < n) ? __ldg(X + (row0 + r) * D + k) : 0.f;
        }
}

template <int D>
__global__ void __launch_bounds__(256) gate_rows_kernel(int64_t n, const float* __restrict__ X, const float* __restrict__ W,
                                                        const float* __restrict__ b, const float* __restrict__ mul, float* __restrict__ out) {
    constexpr int JT = D / 32, LD = D + 1;
    extern __shared__ __align__(16) float fsm[];
    float* Wt = fsm;                               // [D][LD]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    load_weight_t<D>(Wt, W);
    float* xs = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(Wt + D * LD) + 15) & ~uintptr_t(15)) + warp * D * FR;   // 16-byte aligned row tiles
    float bj[JT];
#pragma unroll
    for (int jt = 0; jt < JT; ++jt) bj[jt] = b ? __ldg(b + lane + 32 * jt) : 0.f;
    __syncthreads();
    for (int64_t row0 = ((int64_t)blockIdx.x * n_warps + warp) * FR; row0 < n; row0 += (int64_t)gridDim.x * n_warps * FR) {
        stage_rows<D>(xs, X, row0, n, lane);
        __syncwarp();
        float acc[JT][FR];
#pragma unroll
        for (int jt = 0; jt < JT; ++jt)
#pragma unroll
            for (int r = 0; r < FR; ++r) acc[jt][r] = bj[jt];
#pragma unroll 8
        for (int k = 0; k < D; ++k) {
            const float4 x = *reinterpret_cast<const float4*>(xs + k * FR);
#pragma unroll
            for (int jt = 0; jt < JT; ++jt) {
                const float w = Wt[k * LD + lane + 32 * jt];
                acc[jt][0] = fmaf(w, x.x, acc[jt][0]);
                acc[jt][1] = fmaf(w, x.y, acc[jt][1]);
                acc[jt][2] = fmaf(w, x.z, acc[jt][2]);
                acc[jt][3] = fmaf(w, x.w, acc[jt][3]);
            }
        }
#pragma unroll
        for (int r = 0; r < FR; ++r) {
            if (row0 + r >= n) break;
#pragma unroll
            for (int jt = 0; jt < JT; ++jt) {
                const int64_t o = (row0 + r) * D + lane + 32 * jt;
                const float g = sigmoidf_(acc[jt][r]);
                out[o] = mul ? __ldg(mul + o) * g : g;
            }
        }
        __syncwarp();
    }
}

struct MgcnFuseParams {
    int64_t n;
    const float *img, *txt, *content;
    const float *Wq, *bq, *wq2;      // query_common: Linear(d,d) + Tanh + Linear(d,1,bias=False)
    const float *Wgi, *bgi, *Wgt, *bgt;   // gate_image_prefer / gate_text_prefer: Linear(d,d) + Sigmoid
    float *out, *side;               // side nullable
};

template <int D>
__global__ void __launch_bounds__(256) mgcn_fuse_kernel(const MgcnFuseParams p) {
    constexpr int JT = D / 32, LD = D + 1;
    extern __shared__ __align__(16) float fsm[];
    float* Wq = fsm;
    float* Wi = Wq + D * LD;
    float* Wt = Wi + D * LD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    float* xs = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(Wt + D * LD) + 15) & ~uintptr_t(15)) + warp * 3 * D * FR;
    float* xi = xs;
    float* xt = xs + D * FR;
    float* xc = xs + 2 * D * FR;
    load_weight_t<D>(Wq, p.Wq);
    load_weight_t<D>(Wi, p.Wgi);
    load_weight_t<D>(Wt, p.Wgt);
    float bq[JT], bi[JT], bt[JT], w2[JT];
#pragma unroll
    for (int jt = 0; jt < JT; ++jt) {
        const int j = lane + 32 * jt;
        bq[jt] = p.bq ? __ldg(p.bq + j) : 0.f;
        bi[jt] = p.bgi ? __ldg(p.bgi + j) : 0.f;
        bt[jt] = p.bgt ? __ldg(p.bgt + j) : 0.f;
        w2[jt] = __ldg(p.wq2 + j);
    }
    __syncthreads();
    for (int64_t row0 = ((int64_t)blockIdx.x * n_warps + warp) * FR; row0 < p.n; row0 += (int64_t)gridDim.x * n_warps * FR) {
        stage_rows<D>(xi, p.img, row0, p.n, lane);
        stage_rows<D>(xt, p.txt, row0, p.n, lane);
        stage_rows<D>(xc, p.content, row0, p.n, lane);
        __syncwarp();
        float hi[JT][FR], ht[JT][FR], gi[JT][FR], gt[JT][FR];
#pragma unroll
        for (int jt = 0; jt < JT; ++jt)
#pragma unroll
            for (int r = 0; r < FR; ++r) { hi[jt][r] = bq[jt]; ht[jt][r] = bq[jt]; gi[jt][r] = bi[jt]; gt[jt][r] = bt[jt]; }
#pragma unroll 4
        for (int k = 0; k < D; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(xi + k * FR);
            const float4 b = *reinterpret_cast<const float4*>(xt + k * FR);
            const float4 c = *reinterpret_cast<const float4*>(xc + k * FR);
            const float av[FR] = {a.x, a.y, a.z, a.w}, bv[FR] = {b.x, b.y, b.z, b.w}, cv[FR] = {c.x, c.y, c.z, c.w};
#pragma unroll
            for (int jt = 0; jt < JT; ++jt) {
                const int j = lane + 32 * jt;
                const float wq = Wq[k * LD + j], wi = Wi[k * LD + j], wt = Wt[k * LD + j];
#pragma unroll
                for (int r = 0; r < FR; ++r) {
                    hi[jt][r] = fmaf(wq, av[r], hi[jt][r]);
                    ht[jt][r] = fmaf(wq, bv[r], ht[jt][r]);
                    gi[jt][r] = fmaf(wi, cv[r], gi[jt][r]);
                    gt[jt][r] = fmaf(wt, cv[r], gt[jt][r]);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < FR; ++r) {
            float si = 0.f, st = 0.f;
#pragma unroll
            for (int jt = 0; jt < JT; ++jt) {
                si = fmaf(w2[jt], tanhf(hi[jt][r]), si);
                st = fmaf(w2[jt], tanhf(ht[jt][r]), st);
            }
            si = warp_sum(si);
            st = warp_sum(st);
            const float m = fmaxf(si, st);                              // softmax over the two logits (mgcn.py:189-190)
            const float ei = expf(si - m), et = expf(st - m);
            const float w0 = ei / (ei + et), w1 = et / (ei + et);
            if (row0 + r >= p.n) continue;
#pragma unroll
            for (int jt = 0; jt < JT; ++jt) {
                const int j = lane + 32 * jt;
                const float ximg = xi[j * FR + r], xtxt = xt[j * FR + r], cont = xc[j * FR + r];
                const float common = w0 * ximg + w1 * xtxt;                // mgcn.py:191-192
                const float sep_i = sigmoidf_(gi[jt][r]) * (ximg - common);   // :193-198
                const float sep_t = sigmoidf_(gt[jt][r]) * (xtxt - common);
                const float side = (sep_i + sep_t + common) / 3.f;          // :199
                const int64_t o = (row0 + r) * D + j;
                if (p.side) p.side[o] = side;
                p.out[o] = cont + side;                                     // :201
            }
        }
        __syncwarp();
    }
}

template <int D>
static constexpr int fuse_warps() { return D >= 128 ? 4 : 8; }            // D = 128: three weight matrices take 198 KB of the 227 KB

template <int D>
static size_t fuse_smem(int n_weights, int n_inputs) {
    return (size_t)n_weights * D * (D + 1) * sizeof(float) + 16 + (size_t)fuse_warps<D>() * n_inputs * D * FR * sizeof(float) + 16;
}

static unsigned fuse_grid(int64_t n, int warps) {
    int64_t g = (n + warps * FR - 1) / (warps * FR);
    const int64_t cap = sm_count();                                       // persistent: the weights are loaded once per CTA
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

template <int D>
static int launch_gate(int64_t n, const float* X, const float* W, const float* b, const float* mul, float* out, cudaStream_t stream) {
    const size_t smem = fuse_smem<D>(1, 1);
    MMREC_CUDA(cudaFuncSetAttribute(gate_rows_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gate_rows_kernel<D><<<fuse_grid(n, fuse_warps<D>()), 32 * fuse_warps<D>(), smem, stream>>>(n, X, W, b, mul, out);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

template <int D>
static int launch_fuse(const MgcnFuseParams& p, cudaStream_t stream) {
    const size_t smem = fuse_smem<D>(3, 3);
    MMREC_CUDA(cudaFuncSetAttribute(mgcn_fuse_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mgcn_fuse_kernel<D><<<fuse_grid(p.n, fuse_warps<D>()), 32 * fuse_warps<D>(), smem, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

// n9 -- MMGCF's late fusion (src/models/mmgcf.py:177-254, element-wise modes) as one row kernel forward and one backward:
//
//   out[r] = combine(c_e * n_e(E[idx[r]]), c_m * n_m(M0[r]) [, c_m * n_m(M1[r])])
//
// combine is `torch.stack(ts).sum(0)` or `.mean(0)`; `equal` takes two stages (the modalities first, then the ID row with
// their fusion).  A warp owns one row, lane j the columns j, j + 32, ...  Each torch step is one IEEE rounding here
// (__fadd_rn / __fmul_rn / __fdiv_rn: nothing is contracted into an fma), in torch's order:
//  - sum over k terms: ((t0 + t1) + t2), the order of ATen's CUDA reduction over the stacked dimension.
//  - mean: that sum times fl(1/k).  ATen's CUDA MeanOps multiplies the sum by a factor, numel(out) / numel(in) in fp32,
//    which is fl(1/k) for every d here (k * n * d has at least five trailing zero bits, so it is exact below 2^29); the
//    CPU divides by k instead, so the bits follow the device, not the CPU.
//  - its backward: autograd's mean backward is `grad / k`, which ATen's CUDA division by a scalar runs as grad * fl(1/k)
//    (BinaryDivTrueKernel's reciprocal); the CPU divides.  Again the device's rule.
//  - alpha: e * a and m * (1 - a), a = sigmoid(mm_alpha) read from the device; 1 - a is one fp32 subtraction, as torch's.
//  - normalized: F.normalize = x / max(||x||, 1e-12), the ID row then times n_modalities.  torch's norm is a parallel
//    reduction whose order is its own, so these modes are held to a bound, not to bits (tests/test_gpu_mmgcf.py).
// The backward recomputes the row norms instead of storing them.  Under alpha, d alpha is per-CTA partials (fixed warp
// order) summed by one warp in a fixed order: no atomics, the same bits on every run.
enum { LF_MEAN = 0, LF_SUM = 1 };
enum { LF_EQUAL = 0, LF_ALPHA = 1, LF_NORMALIZED = 2 };
constexpr int LF_WARPS = 8;

struct LateFuseParams {
    int64_t n;
    int fusion, weighting;
    const int64_t* idx;                 // nullable: row r of E is r
    const float *E, *M0, *M1;           // M1 nullable (one modality)
    const float* alpha;                 // weighting == alpha only
    float ce, factor;                   // c_e of `normalized`; fl(1/k) of the final mean
    float* out;                         // forward
    const float* g;                     // backward: upstream gradient [n, d]
    float *dE, *dM0, *dM1, *partial;    // dE per gathered row; partial: 2 floats per CTA (alpha)
};

template <int D>
__device__ __forceinline__ void lf_load(float (&x)[D / 32], const float* __restrict__ row, int lane) {
#pragma unroll
    for (int j = 0; j < D / 32; ++j) x[j] = __ldg(row + lane + 32 * j);
}

template <int D>
__device__ __forceinline__ void lf_store(float* row, const float (&x)[D / 32], int lane) {
#pragma unroll
    for (int j = 0; j < D / 32; ++j) row[lane + 32 * j] = x[j];
}

template <int D>
__device__ __forceinline__ float lf_dot(const float (&x)[D / 32], const float (&y)[D / 32]) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < D / 32; ++j) s = fmaf(x[j], y[j], s);
    return warp_sum(s);
}

// x <- x / max(||x||, 1e-12) (F.normalize); returns the clamped norm, *raw the unclamped one
template <int D>
__device__ __forceinline__ float lf_normalize(float (&x)[D / 32], float* raw) {
    const float nrm = sqrtf(lf_dot<D>(x, x));
    const float c = nrm < 1e-12f ? 1e-12f : nrm;                      // clamp_min keeps a NaN norm, as torch's does
#pragma unroll
    for (int j = 0; j < D / 32; ++j) x[j] = __fdiv_rn(x[j], c);
    *raw = nrm;
    return c;
}

template <int D>
__global__ void __launch_bounds__(32 * LF_WARPS) late_fuse_kernel(const LateFuseParams p) {
    constexpr int J = D / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool two = p.M1 != nullptr, mean = p.fusion == LF_MEAN;
    float al = 0.f, be = 0.f;
    if (p.weighting == LF_ALPHA) { al = __ldg(p.alpha); be = __fsub_rn(1.f, al); }
    for (int64_t r = (int64_t)blockIdx.x * LF_WARPS + warp; r < p.n; r += (int64_t)gridDim.x * LF_WARPS) {
        float e[J], a[J], b[J], raw;
        lf_load<D>(e, p.E + (p.idx ? __ldg(p.idx + r) : r) * D, lane);
        lf_load<D>(a, p.M0 + r * D, lane);
        if (two) lf_load<D>(b, p.M1 + r * D, lane);
        if (p.weighting == LF_NORMALIZED) {
            lf_normalize<D>(e, &raw);
            lf_normalize<D>(a, &raw);
            if (two) lf_normalize<D>(b, &raw);
        }
        bool third = two;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            if (p.weighting == LF_ALPHA) {
                e[j] = __fmul_rn(e[j], al);
                a[j] = __fmul_rn(a[j], be);
                if (two) b[j] = __fmul_rn(b[j], be);
            } else if (p.weighting == LF_NORMALIZED) {
                e[j] = __fmul_rn(e[j], p.ce);
            } else if (two) {                                         // equal, stage 1: the modalities fused first
                a[j] = __fadd_rn(a[j], b[j]);
                if (mean) a[j] = __fmul_rn(a[j], 0.5f);
            }
        }
        if (p.weighting == LF_EQUAL) third = false;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            float s = __fadd_rn(e[j], a[j]);
            if (third) s = __fadd_rn(s, b[j]);
            e[j] = mean ? __fmul_rn(s, p.factor) : s;
        }
        lf_store<D>(p.out + r * D, e, lane);
    }
}

// dx of y = x / max(||x||, eps) for the upstream gy: (gy - y (gy . y)) / n where the clamp is inactive, gy / n where it is
template <int D>
__device__ __forceinline__ void lf_normalize_bwd(float (&gy)[D / 32], const float (&y)[D / 32], float n, float raw) {
    const float gdy = raw >= 1e-12f ? lf_dot<D>(gy, y) : 0.f;
#pragma unroll
    for (int j = 0; j < D / 32; ++j) gy[j] = __fdiv_rn(fmaf(-y[j], gdy, gy[j]), n);
}

template <int D>
__global__ void __launch_bounds__(32 * LF_WARPS) late_fuse_bwd_kernel(const LateFuseParams p) {
    constexpr int J = D / 32;
    __shared__ float red[LF_WARPS][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool two = p.M1 != nullptr, mean = p.fusion == LF_MEAN;
    float al = 0.f, be = 0.f, se = 0.f, sm = 0.f;
    if (p.weighting == LF_ALPHA) { al = __ldg(p.alpha); be = __fsub_rn(1.f, al); }
    for (int64_t r = (int64_t)blockIdx.x * LF_WARPS + warp; r < p.n; r += (int64_t)gridDim.x * LF_WARPS) {
        float h[J], ge[J], ga[J], gb[J];
        lf_load<D>(h, p.g + r * D, lane);
        const float* erow = p.E + (p.idx ? __ldg(p.idx + r) : r) * D;
        if (p.weighting == LF_EQUAL) {
#pragma unroll
            for (int j = 0; j < J; ++j) {
                ge[j] = mean ? __fmul_rn(h[j], 0.5f) : h[j];
                ga[j] = gb[j] = (two && mean) ? __fmul_rn(ge[j], 0.5f) : ge[j];
            }
        } else {
#pragma unroll
            for (int j = 0; j < J; ++j) h[j] = mean ? __fmul_rn(h[j], p.factor) : h[j];
            if (p.weighting == LF_ALPHA) {
                float e[J], a[J], b[J];
                lf_load<D>(e, erow, lane);
                lf_load<D>(a, p.M0 + r * D, lane);
                if (two) lf_load<D>(b, p.M1 + r * D, lane);
#pragma unroll
                for (int j = 0; j < J; ++j) {
                    ge[j] = __fmul_rn(h[j], al);
                    ga[j] = gb[j] = __fmul_rn(h[j], be);
                    se = fmaf(h[j], e[j], se);
                    sm = fmaf(h[j], a[j], sm);
                    if (two) sm = fmaf(h[j], b[j], sm);
                }
            } else {                                                  // normalized
                float e[J], a[J], b[J], re, ra, rb = 0.f, ne, na, nb = 1.f;
                lf_load<D>(e, erow, lane);
                lf_load<D>(a, p.M0 + r * D, lane);
                if (two) lf_load<D>(b, p.M1 + r * D, lane);
                ne = lf_normalize<D>(e, &re);
                na = lf_normalize<D>(a, &ra);
                if (two) nb = lf_normalize<D>(b, &rb);
#pragma unroll
                for (int j = 0; j < J; ++j) { ge[j] = __fmul_rn(h[j], p.ce); ga[j] = gb[j] = h[j]; }
                lf_normalize_bwd<D>(ge, e, ne, re);
                lf_normalize_bwd<D>(ga, a, na, ra);
                if (two) lf_normalize_bwd<D>(gb, b, nb, rb);
            }
        }
        lf_store<D>(p.dE + r * D, ge, lane);
        lf_store<D>(p.dM0 + r * D, ga, lane);
        if (two) lf_store<D>(p.dM1 + r * D, gb, lane);
    }
    if (p.weighting != LF_ALPHA) return;
    se = warp_sum(se);
    sm = warp_sum(sm);
    if (lane == 0) { red[warp][0] = se; red[warp][1] = sm; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float te = 0.f, tm = 0.f;
        for (int w = 0; w < LF_WARPS; ++w) { te = __fadd_rn(te, red[w][0]); tm = __fadd_rn(tm, red[w][1]); }
        p.partial[2 * blockIdx.x] = te;
        p.partial[2 * blockIdx.x + 1] = tm;
    }
}

// d alpha = sum e.h - sum m.h over the CTAs' partials, one warp, a fixed order
__global__ void __launch_bounds__(32) late_fuse_alpha_kernel(int n_parts, const float* __restrict__ partial, float* dalpha) {
    float te = 0.f, tm = 0.f;
    for (int i = threadIdx.x; i < n_parts; i += 32) { te += partial[2 * i]; tm += partial[2 * i + 1]; }
    te = warp_sum(te);
    tm = warp_sum(tm);
    if (threadIdx.x == 0) *dalpha = __fsub_rn(te, tm);
}

static int64_t late_fuse_grid(int64_t n) {
    int64_t g = (n + LF_WARPS - 1) / LF_WARPS;
    const int64_t cap = 8 * (int64_t)sm_count();
    return g < 1 ? 1 : (g > cap ? cap : g);
}

static int late_fuse_check(const char* what, int64_t n, int d, int fusion, int weighting, const float* E, int64_t n_E,
                           const int64_t* idx, const float* V, const float* T, const float* alpha) {
    MMREC_CHECK_ARG(n >= 0 && n_E >= 0, "%s: bad sizes", what);
    MMREC_CHECK_ARG(fusion == LF_MEAN || fusion == LF_SUM, "%s: fusion %d is not mean (0) or sum (1)", what, fusion);
    MMREC_CHECK_ARG(weighting >= LF_EQUAL && weighting <= LF_NORMALIZED, "%s: weighting %d is not equal (0), alpha (1) or normalized (2)",
                    what, weighting);
    MMREC_CHECK_ARG(idx || n <= n_E, "%s: %lld rows without idx, E has %lld", what, (long long)n, (long long)n_E);
    if (d != 32 && d != 64 && d != 128) {
        set_error("%s: d = %d has no kernel (32, 64, 128)", what, d);
        return MMREC_EUNSUPPORTED;
    }
    if (n == 0) return MMREC_OK;
    MMREC_CHECK_ARG(E && (V || T), "%s: null E, or neither modality", what);
    MMREC_CHECK_ARG(weighting != LF_ALPHA || alpha, "%s: alpha weighting without alpha", what);
    return MMREC_OK;
}

static LateFuseParams late_fuse_params(int64_t n, int fusion, int weighting, const int64_t* idx, const float* E, const float* V,
                                       const float* T, const float* alpha) {
    LateFuseParams p{};
    const int n_mod = (V != nullptr) + (T != nullptr);
    p.n = n;
    p.fusion = fusion;
    p.weighting = weighting;
    p.idx = idx;
    p.E = E;
    p.M0 = V ? V : T;
    p.M1 = V ? T : nullptr;
    p.alpha = alpha;
    p.ce = (float)n_mod;
    p.factor = 1.f / (float)(weighting == LF_EQUAL ? 2 : 1 + n_mod);
    return p;
}

template <int D>
static int launch_late_fuse(const LateFuseParams& p, bool backward, float* dalpha, cudaStream_t stream) {
    const unsigned grid = (unsigned)late_fuse_grid(p.n);
    if (!backward) {
        late_fuse_kernel<D><<<grid, 32 * LF_WARPS, 0, stream>>>(p);
        MMREC_LAUNCH_CHECK();
        return MMREC_OK;
    }
    late_fuse_bwd_kernel<D><<<grid, 32 * LF_WARPS, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    if (p.weighting == LF_ALPHA) {
        late_fuse_alpha_kernel<<<1, 32, 0, stream>>>((int)grid, p.partial, dalpha);
        MMREC_LAUNCH_CHECK();
    }
    return MMREC_OK;
}

static int late_fuse_dispatch(int d, const LateFuseParams& p, bool backward, float* dalpha, cudaStream_t stream) {
    if (d == 32) return launch_late_fuse<32>(p, backward, dalpha, stream);
    if (d == 64) return launch_late_fuse<64>(p, backward, dalpha, stream);
    return launch_late_fuse<128>(p, backward, dalpha, stream);
}

}  // namespace mmrec

using namespace mmrec;

extern "C" size_t mmrec_late_fuse_workspace_bytes(int64_t n, int d) {
    if (n < 0 || (d != 32 && d != 64 && d != 128)) return 0;
    return (size_t)late_fuse_grid(n) * 2 * sizeof(float);
}

extern "C" int mmrec_late_fuse_f32(int64_t n, int d, int fusion, int weighting, const int64_t* idx, const float* E, int64_t n_E,
                                   const float* V, const float* T, const float* alpha, float* out, void* stream_) {
    int rc = late_fuse_check("late_fuse", n, d, fusion, weighting, E, n_E, idx, V, T, alpha);
    if (rc != MMREC_OK || n == 0) return rc;
    MMREC_CHECK_ARG(out, "late_fuse: null out");
    LateFuseParams p = late_fuse_params(n, fusion, weighting, idx, E, V, T, alpha);
    p.out = out;
    return late_fuse_dispatch(d, p, false, nullptr, (cudaStream_t)stream_);
}

extern "C" int mmrec_late_fuse_bwd_f32(int64_t n, int d, int fusion, int weighting, const int64_t* idx, const float* E, int64_t n_E,
                                       const float* V, const float* T, const float* alpha, const float* g, float* dE_rows, float* dV,
                                       float* dT, float* dalpha, void* ws, size_t ws_bytes, void* stream_) {
    int rc = late_fuse_check("late_fuse_bwd", n, d, fusion, weighting, E, n_E, idx, V, T, alpha);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(weighting != LF_ALPHA || dalpha, "late_fuse_bwd: alpha weighting without dalpha");
    if (n == 0) {
        if (weighting == LF_ALPHA) MMREC_CUDA(cudaMemsetAsync(dalpha, 0, sizeof(float), (cudaStream_t)stream_));
        return MMREC_OK;
    }
    MMREC_CHECK_ARG(g && dE_rows && (!V || dV) && (!T || dT), "late_fuse_bwd: null g, dE_rows, or the gradient of a given modality");
    if (weighting == LF_ALPHA && (!ws || ws_bytes < mmrec_late_fuse_workspace_bytes(n, d))) {
        set_error("late_fuse_bwd: workspace %zu bytes, needs %zu", ws_bytes, mmrec_late_fuse_workspace_bytes(n, d));
        return MMREC_EWORKSPACE;
    }
    LateFuseParams p = late_fuse_params(n, fusion, weighting, idx, E, V, T, alpha);
    p.g = g;
    p.dE = dE_rows;
    p.dM0 = V ? dV : dT;
    p.dM1 = V ? dT : nullptr;
    p.partial = (float*)ws;
    return late_fuse_dispatch(d, p, true, dalpha, (cudaStream_t)stream_);
}

extern "C" int mmrec_gate_rows_f32(int64_t n, int d, const float* X, const float* W, const float* b, const float* mul, float* out,
                                   void* stream_) {
    MMREC_CHECK_ARG(n >= 0 && d >= 1, "gate_rows: bad sizes");
    if (d != 32 && d != 64 && d != 128) {
        set_error("gate_rows: d = %d has no kernel (32, 64, 128)", d);
        return MMREC_EUNSUPPORTED;
    }
    if (n == 0) return MMREC_OK;
    MMREC_CHECK_ARG(X && W && out, "gate_rows: null pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d == 32) return launch_gate<32>(n, X, W, b, mul, out, stream);
    if (d == 64) return launch_gate<64>(n, X, W, b, mul, out, stream);
    return launch_gate<128>(n, X, W, b, mul, out, stream);
}

extern "C" int mmrec_mgcn_fuse_f32(int64_t n, int d, const float* img, const float* txt, const float* content, const float* Wq,
                                   const float* bq, const float* wq2, const float* Wgi, const float* bgi, const float* Wgt,
                                   const float* bgt, float* out, float* side, void* stream_) {
    MMREC_CHECK_ARG(n >= 0 && d >= 1, "mgcn_fuse: bad sizes");
    if (d != 32 && d != 64 && d != 128) {
        set_error("mgcn_fuse: d = %d has no kernel (32, 64, 128)", d);
        return MMREC_EUNSUPPORTED;
    }
    if (n == 0) return MMREC_OK;
    MMREC_CHECK_ARG(img && txt && content && Wq && wq2 && Wgi && Wgt && out, "mgcn_fuse: null pointer");
    MgcnFuseParams p{n, img, txt, content, Wq, bq, wq2, Wgi, bgi, Wgt, bgt, out, side};
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d == 32) return launch_fuse<32>(p, stream);
    if (d == 64) return launch_fuse<64>(p, stream);
    return launch_fuse<128>(p, stream);
}
