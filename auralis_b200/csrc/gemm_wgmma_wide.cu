// bf16 / fp16 tensor-core GEMM for prefill-shaped problems (M >= 256):  out[M,N] = epi(A[M,K] . W[N,K]^T + bias)
//
// The one-tile-per-CTA kernel of gemm_wgmma.cu pays its prologue, pipeline ramp and epilogue per 128 x BN tile, and a
// 128 x 128 tile streams 2 operand bytes per 128 flops from shared memory.  This kernel is the large-shape path:
//   * WIDE TILES: 128 (M) x 256 (N) per CTA; each of the two consumer warpgroups issues wgmma m64n256k16 on its 64 rows
//     (128 fp32 accumulator registers per thread), so every A byte staged in shared memory feeds 256 columns;
//   * PERSISTENT: one CTA per SM walks the tile list; barriers and the TMA ring live across tiles, and the producer warp
//     streams the next tile's operands while the consumers run the epilogue of the current one.
// Roles (288 threads): warps 0-7 consumer warpgroups (MMA + epilogue straight from the accumulators), warp 8 TMA producer.
#include "hopper.cuh"
#include "kernels.h"

namespace xtts {
namespace {

using namespace hop;

constexpr int BM = 128, BN = 256, BK = 64, MMA_K = 16;      // BK: the 128-byte rows of tma_encode_bf16_2d
constexpr int kConsumers = 256, kThreads = kConsumers + 32, kConsumerWarps = kConsumers / 32;
constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;      // per 64-wide k-block: 16 KB + 32 KB
__host__ __device__ constexpr size_t smem_for(int stages) { return (size_t)stages * (A_BYTES + B_BYTES) + 1024; }

template <int STAGES>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const float* __restrict__ bias, const float* resid, void* out, int M, int N, int K, int flags) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
    const int total = tiles_m * tiles_n;
    const int num_kb = K / BK;

    if (warp == kConsumerWarps) {
        if (lane == 0) {
            int it = 0;
            for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
                const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
                for (int kb = 0; kb < num_kb; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&empty_bar[s], (uint32_t)(((it / STAGES) & 1) ^ 1));
                    mbar_expect_tx(&full_bar[s], A_BYTES + B_BYTES);       // out-of-range rows are zero-filled and still counted
                    tma_load_2d(sA + s * A_BYTES, &tmA, &full_bar[s], kb * BK, m0);
                    tma_load_2d(sB + s * B_BYTES, &tmB, &full_bar[s], kb * BK, n0);
                }
            }
        }
        return;
    }

    // ---------------- consumer warpgroup wg: rows [m0 + 64*wg, +64) of each tile
    const int wg = warp >> 2;
    const bool f16 = (flags & GEMM_F16) != 0;
    int it = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
        const bool active = m0 + 64 * wg < M;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(&full_bar[s], (uint32_t)((it / STAGES) & 1));
            // issued by both warpgroups unconditionally (see gemm_wgmma.cu consume_ring): rows past M are TMA zero-fill
            const uint32_t a_addr = smem_u32(sA + s * A_BYTES) + (uint32_t)(64 * wg) * 128u, b_addr = smem_u32(sB + s * B_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k)
                Wgmma<BN>::run(acc, desc_sw128(a_addr + k * MMA_K * 2), desc_sw128(b_addr + k * MMA_K * 2), 1, f16);
            wgmma_commit();
            wgmma_wait<1>();
            fence_acc(acc);
            if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
            prev = s;
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        if (!active) continue;
        // ---- epilogue: a lane holds column pairs (c, c+1) of rows r and r + 8; four lanes cover 32 contiguous bytes of a row
        const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            const int col = n0 + 8 * i + 2 * (lane & 3);
            if (col >= N) continue;
            const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                if (row >= M) continue;
                float x0 = acc[4 * i + 2 * h] + b0, x1 = acc[4 * i + 2 * h + 1] + b1;
                if (flags & GEMM_GELU) { x0 = gelu_new(x0); x1 = gelu_new(x1); }
                if (flags & GEMM_RESID) {
                    const float2 t = *reinterpret_cast<const float2*>(resid + (size_t)row * N + col);
                    x0 += t.x; x1 += t.y;
                }
                if (flags & GEMM_OUT_BF16)
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(out) + (size_t)row * N + col) = pack16(x0, x1, f16);
                else
                    *reinterpret_cast<float2*>(reinterpret_cast<float*>(out) + (size_t)row * N + col) = make_float2(x0, x1);
            }
        }
    }
}

}  // namespace

bool gemm_wide_supported(int M, int N, int K) { return M >= 256 && N >= 256 && N % 32 == 0 && K % BK == 0 && K >= BK; }

void launch_gemm_bf16_wide(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, const float* resid, void* out,
                           int M, int N, int K, int flags, cudaStream_t st) {
    if (!gemm_wide_supported(M, N, K)) throw CudaError("gemm_wide: unsupported shape");
    static bool attr[64] = {};
    if (first_on_device(attr)) {
        CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_wide_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_for(2)));
        CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_wide_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_for(3)));
        CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_wide_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_for(4)));
    }
    CUtensorMap tmA, tmB;
    tma_encode_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, BM);
    tma_encode_bf16_2d(&tmB, W, (uint64_t)N, (uint64_t)K, BN);
    const int total = ceil_div(M, BM) * ceil_div(N, BN);
    const dim3 grid(std::min(total, sm_count()));
    ProfScope ps(KF_GEMM_TC, st, 2.0 * M * N * K,
                 2.0 * ((double)M * K + (double)N * K) + ((flags & GEMM_OUT_BF16) ? 2.0 : 4.0) * M * N);
    // g_gemm_wide = the ring depth: 4 stages (192 KB, default), 3 or 2.  Every depth runs the same MMA order per output
    // element, so all give the same bits.
#define XTTS_WIDE(ST) gemm_bf16_wide_kernel<ST><<<grid, dim3(kThreads), smem_for(ST), st>>>(tmA, tmB, bias, resid, out, M, N, K, flags)
    if (g_gemm_wide == 2) XTTS_WIDE(2);
    else if (g_gemm_wide == 3) XTTS_WIDE(3);
    else XTTS_WIDE(4);
#undef XTTS_WIDE
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
