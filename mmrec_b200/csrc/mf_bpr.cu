// n13 -- the matrix-factorisation BPR loss of BPR and VBPR (src/models/bpr.py:62-86, src/models/vbpr.py:69-98 with
// BPRLoss / EmbLoss of src/common/loss.py) as one row kernel forward and one backward, instead of the torch chain of three
// gathers, two row dots, sigmoid / log / mean, three Frobenius norms and their autograd (a few dozen small launches):
//
//   x_b  = <U[users[b]], I(pos[b])> - <U[users[b]], I(neg[b])>,   I(pos[b]) = [A[pos[b]] | P[b]],  I(neg[b]) = [A[neg[b]] | P[B + b]]
//   loss = -(sum_b log(1e-10 + sigmoid(x_b))) / B + reg_weight * (((0 + ||U_b||) + ||Pos_b||) + ||Neg_b||) / B
//
// A warp owns one row, lane j the columns j*V .. j*V + V-1 of each 32*V-column chunk (V = 4 at du = 128, 2 at du = 64,
// 1 at other widths).  The element-wise chain is torch's on the device, one IEEE rounding per step (__fadd_rn /
// __fmul_rn / __fdiv_rn: nothing is contracted into an fma):
//  - sigmoid is 1 / (1 + expf(-x)) (ATen's CUDA kernel), then `1e-10 + s` with the scalar rounded to fp32, then logf;
//  - ATen's CUDA mean is the sum times fl(1/B), and a division of a tensor by a Python number runs as a multiplication by
//    its fp32 reciprocal (BinaryDivTrueKernel), forward and in autograd's backward, so `/ B` is `* fl(1/B)` throughout;
//  - the backward follows autograd: mean backward (-g) * fl(1/B), log backward g / t, sigmoid backward (g * (1 - s)) * s,
//    the norm's `grad * (x / norm).masked_fill_(norm == 0, 0)`, and the user row's three incoming gradients summed in the
//    order autograd's input buffer adds them: ((norm term + neg-dot term) + pos-dot term).
// The dots and the sums of squares run in this kernel's own order (lane-strided fmaf, then a fixed xor butterfly), so on
// inputs where they are exact every result equals the torch expression's bits; elsewhere they are held to a bound
// (tests/test_gpu_vbpr.py).  The batch sums are per-CTA partials (fixed warp order) summed by one warp in a fixed order:
// no atomics, the same bits on every run.
#include <cuda_runtime.h>

#include "common.cuh"

namespace mmrec {

constexpr int BM_WARPS = 8;

struct BprMfParams {
    int64_t B;
    int du, da, dp;
    const float *U, *A, *P;             // P nullable (dp == 0)
    const int64_t *users, *pos, *neg;
    float rw, inv_b;                    // fp32 reg_weight, fl(1/B)
    float* x;                           // [B]: written by the forward, read by the backward
    float* partial;                     // forward: 4 floats per CTA
    const float *norms, *g;             // backward: ||U_b||, ||Pos_b||, ||Neg_b||; the upstream gradient (one fp32)
    float *gU, *gA, *gP;                // backward: [B, du], [2B, da], [2B, dp]
};

template <int V>
__device__ __forceinline__ void bm_load(float (&r)[V], const float* __restrict__ p) {
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
__device__ __forceinline__ void bm_store(float* p, const float (&r)[V]) {
    if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(r[0], r[1], r[2], r[3]);
    else if constexpr (V == 2) *reinterpret_cast<float2*>(p) = make_float2(r[0], r[1]);
    else p[0] = r[0];
}

__device__ __forceinline__ float bm_sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

__device__ __forceinline__ float bm_gamma() { return static_cast<float>(1e-10); }      // BPRLoss's gamma, as ATen rounds it

// one row's item columns k .. k + V-1: the ID table below da, the projected rows above
template <int V>
__device__ __forceinline__ void bm_item(float (&r)[V], const BprMfParams& p, int64_t item, int64_t prow, int k) {
    if (k < p.da) bm_load<V>(r, p.A + item * p.da + k);
    else bm_load<V>(r, p.P + prow * p.dp + (k - p.da));
}

template <int V>
__global__ void __launch_bounds__(32 * BM_WARPS) bpr_mf_kernel(const BprMfParams p) {
    __shared__ float red[BM_WARPS][4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float sl = 0.f, su = 0.f, sp = 0.f, sn = 0.f;
    for (int64_t b = (int64_t)blockIdx.x * BM_WARPS + warp; b < p.B; b += (int64_t)gridDim.x * BM_WARPS) {
        const float* urow = p.U + __ldg(p.users + b) * p.du;
        const int64_t ip = __ldg(p.pos + b), in = __ldg(p.neg + b);
        float dpos = 0.f, dneg = 0.f;
        for (int k = lane * V; k < p.du; k += 32 * V) {
            float u[V], a[V], c[V];
            bm_load<V>(u, urow + k);
            bm_item<V>(a, p, ip, b, k);
            bm_item<V>(c, p, in, p.B + b, k);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                dpos = fmaf(u[j], a[j], dpos);
                dneg = fmaf(u[j], c[j], dneg);
                su = fmaf(u[j], u[j], su);
                sp = fmaf(a[j], a[j], sp);
                sn = fmaf(c[j], c[j], sn);
            }
        }
        const float x = __fsub_rn(warp_sum(dpos), warp_sum(dneg));
        if (lane == 0) {
            p.x[b] = x;
            sl = __fadd_rn(sl, logf(__fadd_rn(bm_gamma(), bm_sigmoid(x))));
        }
    }
    sl = warp_sum(sl);
    su = warp_sum(su);
    sp = warp_sum(sp);
    sn = warp_sum(sn);
    if (lane == 0) { red[warp][0] = sl; red[warp][1] = su; red[warp][2] = sp; red[warp][3] = sn; }
    __syncthreads();
    if (threadIdx.x < 4) {
        float t = 0.f;
        for (int w = 0; w < BM_WARPS; ++w) t = __fadd_rn(t, red[w][threadIdx.x]);
        p.partial[4 * blockIdx.x + threadIdx.x] = t;
    }
}

// the batch sums over the CTAs' partials, one warp in a fixed order; then the norms and the [1] loss
__global__ void __launch_bounds__(32) bpr_mf_finish_kernel(int n_parts, const float* __restrict__ partial, float rw, float inv_b,
                                                           float* loss, float* norms) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = threadIdx.x; i < n_parts; i += 32)
#pragma unroll
        for (int q = 0; q < 4; ++q) s[q] = __fadd_rn(s[q], partial[4 * i + q]);
#pragma unroll
    for (int q = 0; q < 4; ++q) s[q] = warp_sum(s[q]);
    if (threadIdx.x != 0) return;
    const float nu = sqrtf(s[1]), np = sqrtf(s[2]), nn = sqrtf(s[3]);
    norms[0] = nu;
    norms[1] = np;
    norms[2] = nn;
    const float mf = -__fmul_rn(s[0], inv_b);                                          // -(mean of the log terms)
    const float reg = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, nu), np), nn), inv_b);   // EmbLoss
    *loss = __fadd_rn(mf, __fmul_rn(rw, reg));
}

// grad * (x / norm).masked_fill_(norm == 0, 0): autograd's backward of a 2-norm
__device__ __forceinline__ float bm_norm_bwd(float g, float x, float nrm) { return __fmul_rn(g, nrm == 0.f ? 0.f : __fdiv_rn(x, nrm)); }

template <int V>
__global__ void __launch_bounds__(32 * BM_WARPS) bpr_mf_bwd_kernel(const BprMfParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float g = __ldg(p.g);
    const float gl = __fmul_rn(-g, p.inv_b);                                // neg, then mean backward
    const float gn = __fmul_rn(__fmul_rn(g, p.rw), p.inv_b);                // `reg_weight *`, then `/ B`
    const float nu = __ldg(p.norms), np = __ldg(p.norms + 1), nn = __ldg(p.norms + 2);
    for (int64_t b = (int64_t)blockIdx.x * BM_WARPS + warp; b < p.B; b += (int64_t)gridDim.x * BM_WARPS) {
        const float* urow = p.U + __ldg(p.users + b) * p.du;
        const int64_t ip = __ldg(p.pos + b), in = __ldg(p.neg + b);
        const float s = bm_sigmoid(__ldg(p.x + b));
        const float gx = __fmul_rn(__fmul_rn(__fdiv_rn(gl, __fadd_rn(bm_gamma(), s)), __fsub_rn(1.f, s)), s);
        const float gy = -gx;                                                  // sub backward: the neg dot's gradient
        for (int k = lane * V; k < p.du; k += 32 * V) {
            float u[V], a[V], c[V], hu[V], ha[V], hc[V];
            bm_load<V>(u, urow + k);
            bm_item<V>(a, p, ip, b, k);
            bm_item<V>(c, p, in, p.B + b, k);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                hu[j] = __fadd_rn(__fadd_rn(bm_norm_bwd(gn, u[j], nu), __fmul_rn(gy, c[j])), __fmul_rn(gx, a[j]));
                ha[j] = __fadd_rn(bm_norm_bwd(gn, a[j], np), __fmul_rn(gx, u[j]));
                hc[j] = __fadd_rn(bm_norm_bwd(gn, c[j], nn), __fmul_rn(gy, u[j]));
            }
            bm_store<V>(p.gU + b * p.du + k, hu);
            if (k < p.da) {
                bm_store<V>(p.gA + b * p.da + k, ha);
                bm_store<V>(p.gA + (p.B + b) * p.da + k, hc);
            } else {
                bm_store<V>(p.gP + b * p.dp + (k - p.da), ha);
                bm_store<V>(p.gP + (p.B + b) * p.dp + (k - p.da), hc);
            }
        }
    }
}

static int64_t bpr_mf_grid(int64_t B) {
    int64_t g = (B + BM_WARPS - 1) / BM_WARPS;
    const int64_t cap = 8 * (int64_t)sm_count();
    return g < 1 ? 1 : (g > cap ? cap : g);
}

static bool bm_aligned(const void* q, int bytes) { return q == nullptr || ((uintptr_t)q % bytes) == 0; }

// 4 at widths of 128k columns, 2 at 64k, else 1; a vector never straddles the ID / projected boundary
static int bpr_mf_vec(const BprMfParams& p, bool backward) {
    for (int V : {4, 2}) {
        const int bytes = 4 * V;
        bool ok = p.du % (32 * V) == 0 && p.da % V == 0 && bm_aligned(p.U, bytes) && bm_aligned(p.A, bytes) && bm_aligned(p.P, bytes);
        if (backward) ok = ok && bm_aligned(p.gU, bytes) && bm_aligned(p.gA, bytes) && bm_aligned(p.gP, bytes);
        if (ok) return V;
    }
    return 1;
}

static int bpr_mf_check(const char* what, int64_t B, int du, int da, int dp, const float* U, const float* A, const float* P,
                        const int64_t* users, const int64_t* pos, const int64_t* neg, const float* x) {
    MMREC_CHECK_ARG(B >= 1, "%s: B = %lld, the loss needs at least one row", what, (long long)B);
    MMREC_CHECK_ARG(da >= 0 && dp >= 0 && du >= 1 && du == da + dp, "%s: du = %d must be da + dp = %d + %d >= 1", what, du, da, dp);
    MMREC_CHECK_ARG(U && users && pos && neg && x, "%s: null U, users, pos, neg or x", what);
    MMREC_CHECK_ARG(da == 0 || A, "%s: null A with da = %d", what, da);
    MMREC_CHECK_ARG(dp == 0 || P, "%s: null P with dp = %d", what, dp);
    return MMREC_OK;
}

static BprMfParams bpr_mf_params(int64_t B, int du, int da, int dp, const float* U, const float* A, const float* P,
                                 const int64_t* users, const int64_t* pos, const int64_t* neg, float reg_weight) {
    BprMfParams p{};
    p.B = B;
    p.du = du;
    p.da = da;
    p.dp = dp;
    p.U = U;
    p.A = da ? A : nullptr;
    p.P = dp ? P : nullptr;
    p.users = users;
    p.pos = pos;
    p.neg = neg;
    p.rw = reg_weight;
    p.inv_b = 1.f / (float)B;
    return p;
}

}  // namespace mmrec

using namespace mmrec;

extern "C" size_t mmrec_bpr_mf_workspace_bytes(int64_t B) {
    if (B < 1) return 0;
    return (size_t)bpr_mf_grid(B) * 4 * sizeof(float);
}

extern "C" int mmrec_bpr_mf_f32(int64_t B, int du, int da, int dp, const float* U, const float* A, const float* P, const int64_t* users,
                                const int64_t* pos, const int64_t* neg, float reg_weight, float* loss, float* x, float* norms, void* ws,
                                size_t ws_bytes, void* stream_) {
    int rc = bpr_mf_check("bpr_mf", B, du, da, dp, U, A, P, users, pos, neg, x);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(loss && norms, "bpr_mf: null loss or norms");
    if (!ws || ws_bytes < mmrec_bpr_mf_workspace_bytes(B)) {
        set_error("bpr_mf: workspace %zu bytes, needs %zu", ws_bytes, mmrec_bpr_mf_workspace_bytes(B));
        return MMREC_EWORKSPACE;
    }
    BprMfParams p = bpr_mf_params(B, du, da, dp, U, A, P, users, pos, neg, reg_weight);
    p.x = x;
    p.partial = (float*)ws;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)bpr_mf_grid(B);
    const int V = bpr_mf_vec(p, false);
    if (V == 4) bpr_mf_kernel<4><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    else if (V == 2) bpr_mf_kernel<2><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    else bpr_mf_kernel<1><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    bpr_mf_finish_kernel<<<1, 32, 0, stream>>>((int)grid, p.partial, p.rw, p.inv_b, loss, norms);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

extern "C" int mmrec_bpr_mf_bwd_f32(int64_t B, int du, int da, int dp, const float* U, const float* A, const float* P,
                                    const int64_t* users, const int64_t* pos, const int64_t* neg, float reg_weight, const float* x,
                                    const float* norms, const float* g, float* gU, float* gA_rows, float* gP_rows, void* stream_) {
    int rc = bpr_mf_check("bpr_mf_bwd", B, du, da, dp, U, A, P, users, pos, neg, x);
    if (rc != MMREC_OK) return rc;
    MMREC_CHECK_ARG(norms && g && gU, "bpr_mf_bwd: null norms, g or gU");
    MMREC_CHECK_ARG((da == 0 || gA_rows) && (dp == 0 || gP_rows), "bpr_mf_bwd: null gA_rows with da > 0 or gP_rows with dp > 0");
    BprMfParams p = bpr_mf_params(B, du, da, dp, U, A, P, users, pos, neg, reg_weight);
    p.x = const_cast<float*>(x);
    p.norms = norms;
    p.g = g;
    p.gU = gU;
    p.gA = da ? gA_rows : nullptr;
    p.gP = dp ? gP_rows : nullptr;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned grid = (unsigned)bpr_mf_grid(B);
    const int V = bpr_mf_vec(p, true);
    if (V == 4) bpr_mf_bwd_kernel<4><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    else if (V == 2) bpr_mf_bwd_kernel<2><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    else bpr_mf_bwd_kernel<1><<<grid, 32 * BM_WARPS, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
