// fp32 CUDA-core GEMM (parity mode and the GPU-side yardstick for the tensor-core kernels).
//   out[M,N] = epi(A[M,K] . W[N,K]^T + bias)      both operands K-contiguous ("NT")
// Replaces the cuBLAS calls behind vLLM's QKV/O/MLP linears and the LM head
// (SURVEY.md §2.4 K4,K6,K7,K9; call sites vllm_mm_gpt.py:759,687).
#include "kernels.h"

namespace xtts {

thread_local KernelCtx* t_kctx = nullptr;
KernelCtx& kctx_default() { static KernelCtx c; return c; }

namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;   // 256 threads, 4x4 outputs each

template <bool kAligned>
__global__ void __launch_bounds__(256)
gemm_f32_nt_kernel(const float* __restrict__ A, const float* __restrict__ W, const float* __restrict__ bias,
                   const float* resid, float* out, int M, int N, int K, int flags) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Ws[BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tx = tid & 15, ty = tid >> 4;          // tx -> n, ty -> m
    // loader mapping: each thread fetches 4 consecutive k of one row of A and one row of W
    const int lrow = tid >> 2, lk = (tid & 3) * 4;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += BK) {
        float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f), w4 = a4;
        const int gm = m0 + lrow, gn = n0 + lrow, gk = k0 + lk;
        if (kAligned) {
            if (gm < M && gk < K) a4 = *reinterpret_cast<const float4*>(A + (size_t)gm * K + gk);
            if (gn < N && gk < K) w4 = *reinterpret_cast<const float4*>(W + (size_t)gn * K + gk);
        } else {
            if (gm < M) {
                const float* p = A + (size_t)gm * K + gk;
                if (gk + 0 < K) a4.x = p[0];
                if (gk + 1 < K) a4.y = p[1];
                if (gk + 2 < K) a4.z = p[2];
                if (gk + 3 < K) a4.w = p[3];
            }
            if (gn < N) {
                const float* p = W + (size_t)gn * K + gk;
                if (gk + 0 < K) w4.x = p[0];
                if (gk + 1 < K) w4.y = p[1];
                if (gk + 2 < K) w4.z = p[2];
                if (gk + 3 < K) w4.w = p[3];
            }
        }
        __syncthreads();     // previous tile fully consumed
        As[lk + 0][lrow] = a4.x; As[lk + 1][lrow] = a4.y; As[lk + 2][lrow] = a4.z; As[lk + 3][lrow] = a4.w;
        Ws[lk + 0][lrow] = w4.x; Ws[lk + 1][lrow] = w4.y; Ws[lk + 2][lrow] = w4.z; Ws[lk + 3][lrow] = w4.w;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * TM]);
            const float4 wv = *reinterpret_cast<const float4*>(&Ws[k][tx * TN]);
            const float a[4] = {av.x, av.y, av.z, av.w};
            const float w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + ty * TM + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            if (n >= N) continue;
            float v = acc[i][j];
            if (bias) v += bias[n];
            if (flags & GEMM_GELU) v = gelu_new(v);
            if (flags & GEMM_RESID) v += resid[(size_t)m * N + n];
            out[(size_t)m * N + n] = v;
        }
    }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = __float2bfloat16_rn(in[i]);
}

__global__ void gemv_kernel(const float* __restrict__ W, const float* __restrict__ b, const float* __restrict__ g,
                            float* __restrict__ y, int rows, int cols) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s = fmaf(W[(size_t)row * cols + c], g[c], s);
    s = warp_sum(s);
    if (lane == 0) y[row] = s + (b ? b[row] : 0.f);
}

}  // namespace

void launch_gemm_f32(const float* A, const float* W, const float* bias, const float* resid, float* out,
                     int M, int N, int K, int flags, cudaStream_t st) {
    if (M <= 0 || N <= 0) return;
    dim3 grid(ceil_div(N, BN), ceil_div(M, BM));
    const bool aligned = (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
    ProfScope ps(KF_GEMM_F32, st, 2.0 * M * N * K, 4.0 * ((double)M * K + (double)N * K + (double)M * N));
    if (aligned)
        gemm_f32_nt_kernel<true><<<grid, 256, 0, st>>>(A, W, bias, resid, out, M, N, K, flags);
    else
        gemm_f32_nt_kernel<false><<<grid, 256, 0, st>>>(A, W, bias, resid, out, M, N, K, flags);
    COUNT_LAUNCH();
    KERNEL_CHECK();
}

__global__ void f32_to_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = __float2half_rn(in[i]);
}
void launch_f32_to_f16(const float* in, __half* out, size_t n, cudaStream_t st) {
    if (n == 0) return;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
    f32_to_f16_kernel<<<blocks, 256, 0, st>>>(in, out, n);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_f32_to_bf16(const float* in, __nv_bfloat16* out, size_t n, cudaStream_t st) {
    if (n == 0) return;
    int blocks = (int)((n + 255) / 256);
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    ProfScope ps(KF_MISC, st, 0, 6.0 * n);
    f32_to_bf16_kernel<<<blocks, 256, 0, st>>>(in, out, n);
    COUNT_LAUNCH();
    KERNEL_CHECK();
}

void launch_gemv(const float* W, const float* b, const float* g, float* y, int rows, int cols, cudaStream_t st) {
    const int wpb = 8;
    ProfScope ps(KF_MISC, st, 2.0 * rows * cols, 4.0 * rows * cols);
    gemv_kernel<<<ceil_div(rows, wpb), wpb * 32, 0, st>>>(W, b, g, y, rows, cols);
    COUNT_LAUNCH();
    KERNEL_CHECK();
}

}  // namespace xtts
