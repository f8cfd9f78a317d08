// Exact-fp32 CUDA-core NT GEMM with gathered A rows:  C[m, n] = sum_k A[idx[m], k] * B[n, k]  (+ bias[n]).
// This is the bit-faithful fp32 path (one fmaf chain per output, k ascending) used by
//   * mmrec_project_f32  (M = rows to project, N = d, K = F)       -- src/models/freedom.py:205-209
//   * mmrec_score_f32    (M = users, N = items, K = d)             -- src/models/freedom.py:219
// and the yardstick the tensor-core kernels are validated against on the device.
#pragma once
#include "common.cuh"

namespace mmrec {

struct GemmNT {
    const float* A; int64_t lda; const int64_t* a_idx; int64_t M;   // A row m is A[a_idx ? a_idx[m] : m]
    const float* B; int64_t ldb; int64_t N;
    int64_t K;
    const float* bias;       // [N] or null
    float* C; int64_t ldc;
    int l2_normalize;        // needs N <= BN
};

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(256) gemm_nt_kernel(const GemmNT p) {
    constexpr int BK = 32;
    constexpr int TX = BN / TN, TY = BM / TM;
    static_assert(TX * TY == 256, "256 threads");
    static_assert(TX <= 32 && (32 % TX) == 0, "row group inside a warp");
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int64_t m0 = (int64_t)blockIdx.x * BM, n0 = (int64_t)blockIdx.y * BN;
    const bool vecA = ((p.lda & 3) == 0) && ((((uintptr_t)p.A) & 15) == 0);
    const bool vecB = ((p.ldb & 3) == 0) && ((((uintptr_t)p.B) & 15) == 0);

    constexpr int A4 = BM * BK / 4 / 256 > 0 ? BM * BK / 4 / 256 : 1;
    constexpr int B4 = BN * BK / 4 / 256 > 0 ? BN * BK / 4 / 256 : 1;
    float4 ra[A4], rb[B4];
    const float* a_row[A4];
    const float* b_row[B4];
    int a_k4[A4], a_m[A4], b_k4[B4], b_n[B4];
#pragma unroll
    for (int i = 0; i < A4; ++i) {
        int f = tid + i * 256;
        a_m[i] = f / (BK / 4); a_k4[i] = (f % (BK / 4)) * 4;
        int64_t m = m0 + a_m[i];
        a_row[i] = nullptr;
        if (a_m[i] < BM && m < p.M) a_row[i] = p.A + (p.a_idx ? p.a_idx[m] : m) * p.lda;
    }
#pragma unroll
    for (int i = 0; i < B4; ++i) {
        int f = tid + i * 256;
        b_n[i] = f / (BK / 4); b_k4[i] = (f % (BK / 4)) * 4;
        int64_t n = n0 + b_n[i];
        b_row[i] = (b_n[i] < BN && n < p.N) ? p.B + n * p.ldb : nullptr;
    }
    auto load4 = [&](const float* row, int64_t k, bool vec) -> float4 {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!row) return v;
        if (vec && k + 3 < p.K) return ldg4(row + k);
        if (k + 0 < p.K) v.x = __ldg(row + k + 0);
        if (k + 1 < p.K) v.y = __ldg(row + k + 1);
        if (k + 2 < p.K) v.z = __ldg(row + k + 2);
        if (k + 3 < p.K) v.w = __ldg(row + k + 3);
        return v;
    };
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

#pragma unroll
    for (int i = 0; i < A4; ++i) ra[i] = load4(a_row[i], a_k4[i], vecA);
#pragma unroll
    for (int i = 0; i < B4; ++i) rb[i] = load4(b_row[i], b_k4[i], vecB);

    for (int64_t k0 = 0; k0 < p.K; k0 += BK) {
#pragma unroll
        for (int i = 0; i < A4; ++i)
            if (a_m[i] < BM) {
                As[a_k4[i] + 0][a_m[i]] = ra[i].x; As[a_k4[i] + 1][a_m[i]] = ra[i].y;
                As[a_k4[i] + 2][a_m[i]] = ra[i].z; As[a_k4[i] + 3][a_m[i]] = ra[i].w;
            }
#pragma unroll
        for (int i = 0; i < B4; ++i)
            if (b_n[i] < BN) {
                Bs[b_k4[i] + 0][b_n[i]] = rb[i].x; Bs[b_k4[i] + 1][b_n[i]] = rb[i].y;
                Bs[b_k4[i] + 2][b_n[i]] = rb[i].z; Bs[b_k4[i] + 3][b_n[i]] = rb[i].w;
            }
        __syncthreads();
        if (k0 + BK < p.K) {   // prefetch the next K slab while computing this one
#pragma unroll
            for (int i = 0; i < A4; ++i) ra[i] = load4(a_row[i], k0 + BK + a_k4[i], vecA);
#pragma unroll
            for (int i = 0; i < B4; ++i) rb[i] = load4(b_row[i], k0 + BK + b_k4[i], vecB);
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    // epilogue
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t m = m0 + ty * TM + i;
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int64_t n = n0 + tx * TN + j;
            if (p.bias && n < p.N) acc[i][j] += __ldg(p.bias + n);
            if (n < p.N) ss += acc[i][j] * acc[i][j];
        }
        if (p.l2_normalize) {
#pragma unroll
            for (int o = TX / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);   // F.normalize(eps=1e-12)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] *= inv;
        }
        if (m < p.M) {
#pragma unroll
            for (int j = 0; j < TN; ++j) {
                const int64_t n = n0 + tx * TN + j;
                if (n < p.N) p.C[m * p.ldc + n] = acc[i][j];
            }
        }
    }
}

template <int BM, int BN, int TM, int TN>
static inline int launch_gemm_nt(const GemmNT& p, cudaStream_t stream) {
    if (p.M <= 0 || p.N <= 0) return MMREC_OK;
    dim3 grid((unsigned)((p.M + BM - 1) / BM), (unsigned)((p.N + BN - 1) / BN));
    gemm_nt_kernel<BM, BN, TM, TN><<<grid, 256, 0, stream>>>(p);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

}  // namespace mmrec
