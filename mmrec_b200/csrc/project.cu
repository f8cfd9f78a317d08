// K2: fused gather -> linear(+bias) -> optional L2 normalise (exact-fp32 CUDA-core path).
// The tensor-core (wgmma, 3xTF32) variant lives in project_tc.cu; this file is the bit-faithful
// fp32 path and the fallback for widths the tensor-core tiles do not cover.
#include "gemm_simt.cuh"

#include <stdlib.h>
#include <string.h>

using namespace mmrec;

namespace mmrec {
// project_tc.cu
int project_tc(int64_t n_out, const int64_t* idx, const float* table, int64_t F, const float* W, const float* bias, int d,
               int l2_normalize, float* Y, int64_t ldy, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t project_tc_workspace_bytes(int64_t n_out, int64_t F, int d);

static int g_project_path = -1;   // 0 = exact fp32 CUDA cores, 1 = wgmma 3xTF32 (default)
static int project_path() {
    if (g_project_path < 0) {
        const char* e = getenv("MMREC_PROJECT_PATH");
        g_project_path = (e && strcmp(e, "simt") == 0) ? 0 : 1;
    }
    return g_project_path;
}

// any d: one CTA per output row, threads stride over the d outputs (correctness path for odd widths)
__global__ void project_generic_kernel(int64_t n_out, const int64_t* __restrict__ idx, const float* __restrict__ table,
                                       int64_t F, const float* __restrict__ W, const float* __restrict__ bias, int d,
                                       int l2, float* __restrict__ Y, int64_t ldy) {
    extern __shared__ float sh[];   // d floats
    __shared__ float red[32];
    const int64_t n = blockIdx.x;
    const float* x = table + (idx ? idx[n] : n) * F;
    float ss = 0.f;
    for (int c = threadIdx.x; c < d; c += blockDim.x) {
        const float* w = W + (int64_t)c * F;
        float acc = 0.f;
        for (int64_t k = 0; k < F; ++k) acc = fmaf(x[k], w[k], acc);
        if (bias) acc += bias[c];
        sh[c] = acc;
        ss += acc * acc;
    }
    if (l2) {
        ss = warp_sum(ss);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
        __syncthreads();
        if (threadIdx.x < 32) {
            float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
            v = warp_sum(v);
            if (threadIdx.x == 0) red[0] = v;
        }
        __syncthreads();
    } else {
        __syncthreads();
    }
    const float inv = l2 ? 1.0f / fmaxf(sqrtf(red[0]), 1e-12f) : 1.0f;
    for (int c = threadIdx.x; c < d; c += blockDim.x) Y[n * ldy + c] = l2 ? sh[c] * inv : sh[c];
}
}  // namespace mmrec

extern "C" int mmrec_project_set_path(int tensor_core) { g_project_path = tensor_core ? 1 : 0; return MMREC_OK; }

extern "C" size_t mmrec_project_workspace_bytes(int64_t n_out, int64_t F, int d) {
    return project_tc_workspace_bytes(n_out, F, d) + 256;
}

extern "C" int mmrec_project_f32(int64_t n_out, const int64_t* idx, const float* table, int64_t n_table, int64_t F,
                                 const float* W, const float* bias, int d, int l2_normalize, float* Y, int64_t ldy,
                                 void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    MMREC_CHECK_ARG(n_out >= 0 && n_table >= 0 && F >= 1 && d >= 1, "project: bad sizes");
    if (n_out == 0) return MMREC_OK;
    MMREC_CHECK_ARG(table && W && Y && ldy >= d, "project: null pointer or ldy < d");
    if (project_path() == 1 && ws) {
        int r = project_tc(n_out, idx, table, F, W, bias, d, l2_normalize, Y, ldy, ws, ws_bytes, stream);
        if (r != 0) return r < 0 ? r : MMREC_OK;
    }
    GemmNT p;
    p.A = table; p.lda = F; p.a_idx = idx; p.M = n_out;
    p.B = W; p.ldb = F; p.N = d; p.K = F; p.bias = bias; p.C = Y; p.ldc = ldy; p.l2_normalize = l2_normalize;
    if (d <= 32) return launch_gemm_nt<64, 32, 4, 2>(p, stream);
    if (d <= 64) return launch_gemm_nt<32, 64, 2, 4>(p, stream);
    if (d <= 128) return launch_gemm_nt<32, 128, 2, 8>(p, stream);
    if (d <= 256) return launch_gemm_nt<32, 256, 2, 16>(p, stream);
    project_generic_kernel<<<(unsigned)n_out, 128, (size_t)d * sizeof(float), stream>>>(n_out, idx, table, F, W, bias, d,
                                                                                   l2_normalize, Y, ldy);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}

// ---- measurement aid: how fast can a [rows, F] fp32 table be streamed when every CTA visits `R` rows round-robin for
// `burst` contiguous bytes each (R * burst = 64 KB in flight per CTA)?  K2 reads its table in exactly this pattern
// (R = 128, burst = 512 B); the probe tells what longer bursts per row would buy.  Result: bytes summed (so nothing is
// optimised away).
namespace mmrec {
__global__ void __launch_bounds__(256) stream_probe_kernel(const float4* __restrict__ table, int64_t n_rows, int64_t row_f4, int R, int burst_f4,
                                                           float* __restrict__ sink) {
    const int tiles = (int)((n_rows + R - 1) / R);
    float acc = 0.f;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        for (int64_t o = 0; o < row_f4; o += burst_f4) {
            float4 v[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {                          // 256 threads x 16 x 16 B = 64 KB
                const int e = i * 256 + threadIdx.x;                 // element of the (R x burst) visit, burst-major inside a row
                const int r = e / burst_f4, c = e - r * burst_f4;
                const int64_t row = (int64_t)tile * R + r;
                v[i] = (r < R && row < n_rows && o + c < row_f4) ? __ldg(table + row * row_f4 + o + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) acc += v[i].x + v[i].y + v[i].z + v[i].w;
        }
    }
    if (acc == 123.456f) *sink = acc;
}
}  // namespace mmrec

extern "C" int mmrec_debug_stream_probe(const float* table, int64_t n_rows, int64_t F, int R, int burst_bytes, int ctas_per_sm, float* sink,
                                        void* stream_) {
    MMREC_CHECK_ARG(table && sink && (F & 3) == 0 && R >= 1 && burst_bytes >= 16 && (int64_t)R * burst_bytes == 65536 && ctas_per_sm >= 1,
                    "stream_probe: need R * burst_bytes == 65536");
    mmrec::stream_probe_kernel<<<(unsigned)(mmrec::sm_count() * ctas_per_sm), 256, 0, (cudaStream_t)stream_>>>(
        (const float4*)table, n_rows, F / 4, R, burst_bytes / 16, sink);
    MMREC_LAUNCH_CHECK();
    return MMREC_OK;
}
