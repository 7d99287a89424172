// bf16 / fp16 tensor-core GEMM for sm_90a:  out[M,N] = epi(A[M,K] . W[N,K]^T + bias)
//   * operands staged by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) into a shared-memory ring guarded by mbarriers
//   * wgmma.mma_async m64nBNk16 from shared memory, fp32 accumulators in registers: two consumer warpgroups, each owning
//     64 rows of the 128-row tile (both always issue their wgmmas; rows past M are computed and never stored)
//   * the consumers' epilogue fuses bias / gelu_new / residual and stores fp32 or 16-bit straight from the accumulators
// Warp roles: warps 0-7 = consumer warpgroups (MMA + epilogue), warp 8 = TMA producer.  Replaces cuBLAS behind vLLM's
// GPT2 linears (SURVEY.md §2.4 K4,K6,K7,K9).
#include "hopper.cuh"
#include "kernels.h"

namespace xtts {
namespace {

using namespace hop;

constexpr int BM = 128, BK = 64, MMA_K = 16;
// ring depth per tile width
// (BN <= 64 rings stay <= 100 KB so that two CTAs fit on an SM: under PDL the next GEMM's CTA can sit beside this one
// and prefetch its weight tiles)
__host__ __device__ constexpr int stages_for(int bn) { return bn >= 128 ? 6 : (bn >= 64 ? 4 : 5); }
constexpr int kConsumers = 256, kThreads = kConsumers + 32;
constexpr int kConsumerWarps = kConsumers / 32;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

// The k-block loop of one consumer warpgroup: acc (+)= A[64 rows at a_row_off] . B^T over `num_kb` ring slots starting at
// ring position `it`.  Slot s is handed back to the producer (one arrive per consumer warp) once the wgmmas that read it
// have retired; the wgmmas of the next slot are issued before that wait, so the tensor cores never drain between slots.
// Both warpgroups always issue their wgmmas, also when one owns no valid rows (M <= 64): a branch around the issue would be
// divergent across the CTA, and ptxas then serialises every wgmma of the kernel.  Rows past M are zero-filled by TMA or
// stale; their accumulators are never stored.
template <int BN, int STAGES>
__device__ __forceinline__ void consume_ring(float (&acc)[BN / 2], const uint8_t* sA, const uint8_t* sB, uint64_t* full_bar,
                                             uint64_t* empty_bar, int it, int num_kb, uint32_t a_row_off, bool f16, int lane) {
    constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full_bar[s], (uint32_t)((it / STAGES) & 1));
        const uint32_t a_addr = smem_u32(sA + s * A_BYTES) + a_row_off, b_addr = smem_u32(sB + s * B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k)
            Wgmma<BN>::run(acc, desc_sw128(a_addr + k * MMA_K * 2), desc_sw128(b_addr + k * MMA_K * 2), 1, f16);
        wgmma_commit();
        wgmma_wait<1>();                             // the previous slot's wgmmas have retired
        fence_acc(acc);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = s;
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
}

template <int BN>
__global__ void __launch_bounds__(kThreads, BN >= 128 ? 1 : 2)
gemm_bf16_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const float* __restrict__ bias, const float* resid, void* out, int M, int N, int K, int flags,
                    int a_box_rows) {
    // (bias / out / flags are re-pointed below for split-K launches)
    constexpr int STAGES = stages_for(BN);
    constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;

    trace_pt(TR_GEMM, 0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
    // split-K: gridDim.z CTAs share one output tile, each owning a contiguous range of k-blocks and writing its raw
    // fp32 partial tile to out + z*M*N (bias/activation/residual are applied by the consumer, deterministically)
    const int total_kb = K / BK;
    const int kb_per = (total_kb + gridDim.z - 1) / gridDim.z;
    const int kb_begin = blockIdx.z * kb_per;
    const int num_kb = max(0, min(total_kb, kb_begin + kb_per) - kb_begin);
    const int flags_in = flags;
    if (gridDim.z > 1) {
        out = reinterpret_cast<float*>(out) + (size_t)blockIdx.z * M * N;
        bias = nullptr; flags = 0;
    }

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    pdl_trigger();                                   // dependents may start their prologue now
    if (warp == kConsumerWarps) {
        if (lane == 0) {
            // weights never depend on the previous kernel: their tiles for the first ring pass are requested BEFORE the
            // dependency wait, the activation tiles right after it
            const int pre = min(num_kb, STAGES);
            for (int kb = 0; kb < pre; ++kb) {
                mbar_expect_tx(&full_bar[kb], (uint32_t)a_box_rows * BK * 2 + B_BYTES);
                tma_load_2d(sB + kb * B_BYTES, &tmB, &full_bar[kb], (kb_begin + kb) * BK, n0);
            }
            pdl_wait();                                  // the activations exist
            trace_pt(TR_GEMM, 1);
            for (int kb = 0; kb < pre; ++kb)
                tma_load_2d(sA + kb * A_BYTES, &tmA, &full_bar[kb], (kb_begin + kb) * BK, m0);
            for (int kb = pre; kb < num_kb; ++kb) {
                const int s = kb % STAGES;
                const uint32_t ph = (kb / STAGES) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                mbar_expect_tx(&full_bar[s], (uint32_t)a_box_rows * BK * 2 + B_BYTES);
                tma_load_2d(sA + s * A_BYTES, &tmA, &full_bar[s], (kb_begin + kb) * BK, m0);
                tma_load_2d(sB + s * B_BYTES, &tmB, &full_bar[s], (kb_begin + kb) * BK, n0);
            }
        }
    } else {
        // ---------------- consumer warpgroup wg: rows [m0 + 64*wg, +64) of the tile
        const int wg = warp >> 2;
        const bool active = m0 + 64 * wg < M;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        consume_ring<BN, STAGES>(acc, sA, sB, full_bar, empty_bar, 0, num_kb, (uint32_t)(64 * wg) * 128u,
                                 (flags_in & GEMM_F16) != 0, lane);
        pdl_wait();                                  // the epilogue reads `resid` and overwrites `out`
        if (active) {
            const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
            const bool f16 = (flags & GEMM_F16) != 0;
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
    trace_pt(TR_GEMM, 2);
}

// rows of the A box: the whole 128-row tile, or (single m-tile problems) just the valid rows rounded up to 8 —
// the rest of the smem tile keeps stale data whose accumulator rows are never stored
inline int a_box_rows_for(int M) { return M >= BM ? BM : ((M + 7) / 8) * 8; }

template <int BN>
constexpr size_t smem_bytes() { return stages_for(BN) * (BM * BK * 2 + BN * BK * 2) + 1024; }

template <int BN>
void launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, const float* resid, void* out, int M,
               int N, int K, int flags, cudaStream_t st, int splits, int a_box_rows, bool pdl) {
    constexpr size_t smem = smem_bytes<BN>();
    static bool attr_set[64] = {};
    if (first_on_device(attr_set))
        CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ceil_div(N, BN), ceil_div(M, BM), splits);
    ProfScope ps(KF_GEMM_TC, st, 2.0 * M * N * K,
                 2.0 * ((double)M * K + (double)N * K) + ((flags & GEMM_OUT_BF16) ? 2.0 : 4.0) * M * N);
    launch_k(gemm_bf16_tc_kernel<BN>, grid, dim3(kThreads), smem, st, pdl, tmA, tmB, bias, resid, out, M, N, K, flags,
             a_box_rows);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace

XTTS_TRACE_SETTER(trace_set_gemm)

void tma_encode_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    if (!g_encode) { std::string err; if (!gemm_tc_init(&err)) throw CudaError(err); }
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {cols * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[160];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu box_rows=%u", (int)r,
                 (unsigned long long)rows, (unsigned long long)cols, box_rows);
        throw CudaError(buf);
    }
}

bool gemm_tc_init(std::string* err) {
    static bool dev_done[64] = {};
    auto per_device = [&] {
        // opt every instantiation into its dynamic shared memory now (never inside a stream capture); per device
        if (!first_on_device(dev_done)) return;
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<128>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<64>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<32>());
        (void)cudaGetLastError();
    };
    if (g_encode) { per_device(); return true; }
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
        if (err) *err = std::string("cuTensorMapEncodeTiled not available: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();
        return false;
    }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    per_device();
    return true;
}

// tile-N heuristic: the largest tile that still gives >= 1 CTA per SM; decode-shaped problems (small M) are
// weight-streaming, so more, narrower CTAs pull more HBM bandwidth
static int pick_bn(int M, int N, int splits) {
    const int mt = ceil_div(M, BM), n_sm = sm_count();
    int bn = 128;
    if (N % 128 != 0 || mt * (N / 128) * splits < n_sm) bn = 64;
    if (bn == 64 && (N % 64 != 0 || mt * (N / 64) * splits < n_sm)) bn = 32;
    if (g_gemm_decode_bn && M <= 256 && N % g_gemm_decode_bn == 0) bn = g_gemm_decode_bn;
    return bn;
}

void launch_gemm_bf16_tc(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, const float* resid,
                         void* out, int M, int N, int K, int flags, cudaStream_t st, bool pdl) {
    if (M <= 0 || N <= 0) return;
    if (K % BK != 0 || N % 32 != 0) throw CudaError("gemm_bf16_tc: need K % 64 == 0 and N % 32 == 0");
    if (g_gemm_wide && !pdl && gemm_wide_supported(M, N, K)) {       // prefill-shaped: persistent wide tiles
        launch_gemm_bf16_wide(A, W, bias, resid, out, M, N, K, flags, st);
        return;
    }
    if (!g_encode) {
        std::string err;
        if (!gemm_tc_init(&err)) throw CudaError(err);
    }
    const int bn = pick_bn(M, N, 1);
    CUtensorMap tmA, tmB;
    const int abox = a_box_rows_for(M);
    tma_encode_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint32_t)abox);
    tma_encode_bf16_2d(&tmB, W, (uint64_t)N, (uint64_t)K, (uint32_t)bn);
    if (bn == 128) launch_bn<128>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl);
    else if (bn == 64) launch_bn<64>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl);
    else launch_bn<32>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl);
}


// split-K variant for the skinny decode GEMMs (N = hidden): partials[z][M][N] = A[:, kz] . W[:, kz]^T, fp32, no epilogue
void launch_gemm_bf16_tc_splitk(const __nv_bfloat16* A, const __nv_bfloat16* W, float* partials, int M, int N, int K,
                                int splits, cudaStream_t st, bool pdl, int flags) {
    flags &= GEMM_F16;
    if (M <= 0 || N <= 0) return;
    if (K % BK != 0 || N % 32 != 0 || splits < 1 || (K / BK) % splits != 0) throw CudaError("gemm_bf16_tc_splitk: bad shape");
    if (!g_encode) { std::string err; if (!gemm_tc_init(&err)) throw CudaError(err); }
    const int bn = pick_bn(M, N, splits);
    CUtensorMap tmA, tmB;
    const int abox = a_box_rows_for(M);
    tma_encode_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint32_t)abox);
    tma_encode_bf16_2d(&tmB, W, (uint64_t)N, (uint64_t)K, (uint32_t)bn);
    if (bn == 128) launch_bn<128>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl);
    else if (bn == 64) launch_bn<64>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl);
    else launch_bn<32>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl);
}


}  // namespace xtts
