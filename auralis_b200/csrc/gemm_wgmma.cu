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

// STAGES = 0: the default ring (stages_for(BN), two CTAs of the narrow tiles fit on an SM); otherwise an explicit depth — the
// "deep" instantiations (engine option "gemm_deep_ring") fill the SM's shared memory with ONE CTA's ring: a decode-shaped GEMM
// is a chain of ring passes that each pay the load latency, and its 16 k-blocks then need 1.6 passes instead of 3.2
template <int BN, int STAGES_ = 0>
__global__ void __launch_bounds__(kThreads, BN >= 128 ? 1 : 2)
gemm_bf16_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const float* __restrict__ bias, const float* resid, void* out, int M, int N, int K, int flags,
                    int a_box_rows, const DepFlag dep) {
    // (bias / out / flags are re-pointed below for split-K launches)
    constexpr int STAGES = STAGES_ > 0 ? STAGES_ : stages_for(BN);
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
            // ... and the weight tiles of the later passes are pulled into L2 meanwhile (engine option gemm_l2_prefetch)
            if (!(flags_in & GEMM_NO_L2PF))
            for (int kb = pre; kb < num_kb; ++kb)
                asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
                             ::"l"(&tmB), "r"((kb_begin + kb) * BK), "r"(n0) : "memory");
            dep_wait(dep);                       // the activations exist (whole predecessor grid, or its counter)
            if (dep.wait) asm volatile("fence.proxy.async;" ::: "memory");     // generic-proxy stores -> TMA (async proxy) reads
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
        if (dep.wait == nullptr) pdl_wait();         // the epilogue reads `resid` and overwrites `out` (with a counter: ordered
                                                     // behind the producer's wait through the full barriers; such launches
                                                     // carry no resid)
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
    dep_arrive(dep, threadIdx.x == 0);               // (fence + CTA barrier inside) this CTA's tile is in global memory
    trace_pt(TR_GEMM, 2);
}

// rows of the A box: the whole 128-row tile, or (single m-tile problems) just the valid rows rounded up to 8 —
// the rest of the smem tile keeps stale data whose accumulator rows are never stored
inline int a_box_rows_for(int M) { return M >= BM ? BM : ((M + 7) / 8) * 8; }

constexpr int deep_stages_for(int bn) { return bn >= 128 ? 6 : (bn >= 64 ? 8 : 10); }
template <int BN, int STAGES_>
constexpr size_t smem_bytes() { return (STAGES_ > 0 ? STAGES_ : stages_for(BN)) * (BM * BK * 2 + BN * BK * 2) + 1024; }

template <int BN, int STAGES_>
int launch_bn_st(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, const float* resid, void* out, int M,
                 int N, int K, int flags, cudaStream_t st, int splits, int a_box_rows, bool pdl, const DepFlag& dep) {
    constexpr size_t smem = smem_bytes<BN, STAGES_>();
    static bool attr_set[64] = {};
    if (first_on_device(attr_set))
        CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_tc_kernel<BN, STAGES_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ceil_div(N, BN), ceil_div(M, BM), splits);
    ProfScope ps(KF_GEMM_TC, st, 2.0 * M * N * K,
                 2.0 * ((double)M * K + (double)N * K) + ((flags & GEMM_OUT_BF16) ? 2.0 : 4.0) * M * N);
    if (dep.wait && (flags & GEMM_RESID)) throw CudaError("gemm_bf16_tc: a counter dependency cannot order a residual read");
    launch_k(gemm_bf16_tc_kernel<BN, STAGES_>, grid, dim3(kThreads), smem, st, pdl, tmA, tmB, bias, resid, out, M, N, K,
             flags | (g_gemm_l2_prefetch ? 0 : GEMM_NO_L2PF), a_box_rows, dep);
    COUNT_LAUNCH(); KERNEL_CHECK();
    return (int)(grid.x * grid.y * grid.z);
}
template <int BN>
int launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, const float* resid, void* out, int M,
              int N, int K, int flags, cudaStream_t st, int splits, int a_box_rows, bool pdl, const DepFlag& dep) {
    // deep ring: only where the whole K range is one CTA's (no split-K: those CTAs have 2-4 k-blocks) and the shape is decode's
    if (g_gemm_deep_ring && BN < 128 && M <= 256 && splits == 1 && K / BK > stages_for(BN))
        return launch_bn_st<BN, deep_stages_for(BN)>(tmA, tmB, bias, resid, out, M, N, K, flags, st, splits, a_box_rows, pdl, dep);
    return launch_bn_st<BN, 0>(tmA, tmB, bias, resid, out, M, N, K, flags, st, splits, a_box_rows, pdl, dep);
}


// =================================================================================================================
// Fused decode "chain" kernel: everything between two attention calls of the decode step in ONE persistent launch
//
//   proj (split-K) -> residual + LayerNorm2 -> fc + gelu -> fc2 (split-K) -> residual + LayerNorm1(next) -> qkv(next)
//
// At decode shapes (M <= 256 rows) every one of those six launches is latency-bound (a 16-k-block main loop between a
// launch, a barrier prologue and an epilogue); here the CTAs stay resident, keep their barriers and smem ring, and separate
// the phases with a device-wide barrier (one atomic + one acquire-poll per CTA).
// One CTA per SM, 288 threads: GEMM phases use the roles of gemm_bf16_tc_kernel (warps 0-7 consumer warpgroups, warp 8
// TMA producer); the reduce + LayerNorm phases use all 9 warps, one row per warp.
// Data written by generic stores in one phase is read by TMA (async proxy) in the next: the barrier is followed by a
// cross-proxy fence.  Co-residency: the grid is <= the SM count, one CTA per SM, and griddepcontrol.launch_dependents is
// only issued after the last device-wide barrier, so no dependent grid can take an SM one of our CTAs still needs.
// =================================================================================================================
constexpr int CH_BN = 64, CH_STAGES = 6, CH_SPLITS = 4;
constexpr int kWarps = kThreads / 32;
enum { EPI_PARTIAL = 0, EPI_BIAS_F32 = 1, EPI_BIAS_GELU_BF16 = 2 };

struct ChainParams {
    int phases, M, H, FF, abox;
    float eps;
    const float* proj_bias; const float* ln2_w; const float* ln2_b;
    const float* fc_bias;
    const float* fc2_bias; const float* ln1_w; const float* ln1_b;     // LayerNorm1 of the NEXT layer (null: residual only)
    const float* qkv_bias;                                              // next layer
    float* X; __nv_bfloat16* Xn; __nv_bfloat16* FFb; float* QKV; float* PART;
    unsigned* sync;                                                     // [0] arrival count, [32] generation (64 words)
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// self-resetting device-wide barrier (all CTAs of the grid are resident: grid <= #SMs, 1 CTA/SM).
// sync[0] = arrival count, sync[32] = generation: separate 128-byte lines, so the pollers do not queue behind the arrivals.
__device__ __forceinline__ void chain_grid_sync(unsigned* sync) {
    asm volatile("fence.proxy.async;" ::: "memory");          // generic writes of this phase -> later async-proxy (TMA) reads
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned* gen_p = sync + 32;
        const unsigned gen = ld_acquire_u32(gen_p);
        __threadfence();
        if (atomicAdd(sync, 1u) == gridDim.x - 1) {
            sync[0] = 0u;
            __threadfence();
            atomicAdd(gen_p, 1u);
        } else {
            const long long t0 = clock64();
            int polls = 0;
            while (ld_acquire_u32(gen_p) == gen) {
                __nanosleep(40);
                if ((++polls & 1023) == 0 && clock64() - t0 > 4000000000LL) __trap();     // watchdog
            }
        }
        __threadfence();
    }
    __syncthreads();
    asm volatile("fence.proxy.async;" ::: "memory");
}

struct ChainSmem {
    uint8_t* sA; uint8_t* sB;
    uint64_t* full_bar; uint64_t* empty_bar;
};

// one GEMM phase: out = epi(A[M,K] . W[N,K]^T); tiles (n-tile, m-tile, k-split) strided over the grid.  `it` = ring position,
// advanced identically by the producer and the consumers.
__device__ __forceinline__ void chain_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int splits,
                                           int epi, const float* __restrict__ bias, void* out, int abox, const ChainSmem& S,
                                           int warp, int lane, int& it) {
    constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = CH_BN * BK * 2;
    const int tiles_n = N / CH_BN, mt = (M + BM - 1) / BM;
    const int kb_per = (K / BK) / splits;
    const int total = tiles_n * mt * splits;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int nt = tile % tiles_n, mi = (tile / tiles_n) % mt, z = tile / (tiles_n * mt);
        const int n0 = nt * CH_BN, m0 = mi * BM, kb0 = z * kb_per;
        if (warp == kConsumerWarps) {
            if (lane == 0) {
                for (int kb = 0; kb < kb_per; ++kb) {
                    const int s = (it + kb) % CH_STAGES;
                    mbar_wait(&S.empty_bar[s], (uint32_t)((((it + kb) / CH_STAGES) & 1) ^ 1));
                    mbar_expect_tx(&S.full_bar[s], (uint32_t)abox * BK * 2 + B_BYTES);
                    tma_load_2d(S.sB + s * B_BYTES, tmB, &S.full_bar[s], (kb0 + kb) * BK, n0);
                    tma_load_2d(S.sA + s * A_BYTES, tmA, &S.full_bar[s], (kb0 + kb) * BK, m0);
                }
            }
        } else {
            const int wg = warp >> 2;
            const bool active = m0 + 64 * wg < M;
            float acc[CH_BN / 2];
#pragma unroll
            for (int i = 0; i < CH_BN / 2; ++i) acc[i] = 0.f;
            consume_ring<CH_BN, CH_STAGES>(acc, S.sA, S.sB, S.full_bar, S.empty_bar, it, kb_per, (uint32_t)(64 * wg) * 128u,
                                           false, lane);
            if (active) {
                const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
                for (int i = 0; i < CH_BN / 8; ++i) {
                    const int col = n0 + 8 * i + 2 * (lane & 3);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r0 + 8 * h;
                        if (row >= M) continue;
                        const float x0 = acc[4 * i + 2 * h], x1 = acc[4 * i + 2 * h + 1];
                        if (epi == EPI_BIAS_GELU_BF16) {
                            const __nv_bfloat162 hv = __floats2bfloat162_rn(gelu_new(x0 + __ldg(bias + col)), gelu_new(x1 + __ldg(bias + col + 1)));
                            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(out) + (size_t)row * N + col) = hv;
                        } else {
                            float* base = reinterpret_cast<float*>(out) + (epi == EPI_PARTIAL ? (size_t)z * M * N : (size_t)0);
                            float2 v = make_float2(x0, x1);
                            if (epi == EPI_BIAS_F32) { v.x += __ldg(bias + col); v.y += __ldg(bias + col + 1); }
                            *reinterpret_cast<float2*>(base + (size_t)row * N + col) = v;
                        }
                    }
                }
            }
        }
        it += kb_per;
    }
}

// X[r] += bias + sum_z PART[z][r] (fixed order: deterministic); optional LayerNorm -> bf16 Xn[r].  One row per warp.
__device__ __forceinline__ void chain_reduce_ln(const ChainParams& P, const float* __restrict__ bias, const float* __restrict__ w,
                                                const float* __restrict__ b, int warp, int lane) {
    const int H = P.H, nj = H / 128;                 // H <= 1024: up to 8 float4 per lane
    const size_t zs = (size_t)P.M * H;
    for (int r = blockIdx.x * kWarps + warp; r < P.M; r += gridDim.x * kWarps) {
        float4 v[8];
        float* x = P.X + (size_t)r * H;
        const float* p = P.PART + (size_t)r * H;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < nj) {
                const int c = j * 128 + lane * 4;
                float4 acc = __ldcg(reinterpret_cast<const float4*>(x + c));
                float4 pz[CH_SPLITS];
#pragma unroll
                for (int z = 0; z < CH_SPLITS; ++z) pz[z] = __ldcg(reinterpret_cast<const float4*>(p + (size_t)z * zs + c));
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
                acc.x += b4.x; acc.y += b4.y; acc.z += b4.z; acc.w += b4.w;
#pragma unroll
                for (int z = 0; z < CH_SPLITS; ++z) { acc.x += pz[z].x; acc.y += pz[z].y; acc.z += pz[z].z; acc.w += pz[z].w; }
                v[j] = acc;
                *reinterpret_cast<float4*>(x + c) = acc;
            }
        }
        if (w == nullptr) continue;
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) if (j < nj) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        const float mean = warp_sum(s) / (float)H;
        float q = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < nj) {
                const float d0 = v[j].x - mean, d1 = v[j].y - mean, d2 = v[j].z - mean, d3 = v[j].w - mean;
                q = fmaf(d0, d0, q); q = fmaf(d1, d1, q); q = fmaf(d2, d2, q); q = fmaf(d3, d3, q);
            }
        const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)H + P.eps);
        __nv_bfloat16* y = P.Xn + (size_t)r * H;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < nj) {
                const int c = j * 128 + lane * 4;
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + c)), b4 = __ldg(reinterpret_cast<const float4*>(b + c));
                __nv_bfloat162 h0 = __floats2bfloat162_rn((v[j].x - mean) * rstd * w4.x + b4.x, (v[j].y - mean) * rstd * w4.y + b4.y);
                __nv_bfloat162 h1 = __floats2bfloat162_rn((v[j].z - mean) * rstd * w4.z + b4.z, (v[j].w - mean) * rstd * w4.w + b4.w);
                uint2 pk;
                pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(y + c) = pk;
            }
    }
}

__global__ void __launch_bounds__(kThreads, 1)
decode_chain_kernel(const __grid_constant__ CUtensorMap tmATT, const __grid_constant__ CUtensorMap tmWo,
                    const __grid_constant__ CUtensorMap tmXn, const __grid_constant__ CUtensorMap tmWfc,
                    const __grid_constant__ CUtensorMap tmFF, const __grid_constant__ CUtensorMap tmWproj,
                    const __grid_constant__ CUtensorMap tmWqkv, const ChainParams P) {
    constexpr uint32_t A_BYTES = BM * BK * 2;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[CH_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[CH_STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmATT) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmXn) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWfc) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmFF) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWproj) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWqkv) : "memory");
        for (int s = 0; s < CH_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    ChainSmem S;
    S.sA = smem; S.sB = smem + CH_STAGES * A_BYTES;
    S.full_bar = full_bar; S.empty_bar = empty_bar;

    pdl_wait();                                    // the attention output (and everything before it) is complete
    int it = 0;
    const int last = 31 - __clz(P.phases);         // index of the last enabled phase
    auto boundary = [&](int bit) {                 // device-wide barrier after every phase but the last; dependents may
        if ((1 << last) == bit) return;            // start launching once the final barrier is behind us
        chain_grid_sync(P.sync);
        if ((P.phases & ~(2 * bit - 1)) == (1 << last)) pdl_trigger();
    };
    if (P.phases == (1 << last)) pdl_trigger();    // single-phase launch: nothing to wait for
    if (P.phases & DC_PROJ) {
        chain_gemm(&tmATT, &tmWo, P.M, P.H, P.H, CH_SPLITS, EPI_PARTIAL, nullptr, P.PART, P.abox, S, warp, lane, it);
        boundary(DC_PROJ);
    }
    if (P.phases & DC_LN2) { chain_reduce_ln(P, P.proj_bias, P.ln2_w, P.ln2_b, warp, lane); boundary(DC_LN2); }
    if (P.phases & DC_FC) {
        chain_gemm(&tmXn, &tmWfc, P.M, P.FF, P.H, 1, EPI_BIAS_GELU_BF16, P.fc_bias, P.FFb, P.abox, S, warp, lane, it);
        boundary(DC_FC);
    }
    if (P.phases & DC_FC2) {
        chain_gemm(&tmFF, &tmWproj, P.M, P.H, P.FF, CH_SPLITS, EPI_PARTIAL, nullptr, P.PART, P.abox, S, warp, lane, it);
        boundary(DC_FC2);
    }
    if (P.phases & DC_LN1) { chain_reduce_ln(P, P.fc2_bias, P.ln1_w, P.ln1_b, warp, lane); boundary(DC_LN1); }
    if (P.phases & DC_QKV)
        chain_gemm(&tmXn, &tmWqkv, P.M, 3 * P.H, P.H, 1, EPI_BIAS_F32, P.qkv_bias, P.QKV, P.abox, S, warp, lane, it);
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
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<128, 0>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<64, 0>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<32, 0>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<64, deep_stages_for(64)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem_bytes<64, deep_stages_for(64)>());
        cudaFuncSetAttribute(gemm_bf16_tc_kernel<32, deep_stages_for(32)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem_bytes<32, deep_stages_for(32)>());
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

int launch_gemm_bf16_tc(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, const float* resid,
                        void* out, int M, int N, int K, int flags, cudaStream_t st, bool pdl, DepFlag dep) {
    if (M <= 0 || N <= 0) return 0;
    if (K % BK != 0 || N % 32 != 0) throw CudaError("gemm_bf16_tc: need K % 64 == 0 and N % 32 == 0");
    if (g_gemm_wide && !pdl && !dep.wait && !dep.arrive && gemm_wide_supported(M, N, K)) {       // prefill-shaped: persistent wide tiles
        launch_gemm_bf16_wide(A, W, bias, resid, out, M, N, K, flags, st);
        return 0;
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
    if (bn == 128) return launch_bn<128>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl, dep);
    if (bn == 64) return launch_bn<64>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl, dep);
    return launch_bn<32>(tmA, tmB, bias, resid, out, M, N, K, flags, st, 1, abox, pdl, dep);
}


// split-K variant for the skinny decode GEMMs (N = hidden): partials[z][M][N] = A[:, kz] . W[:, kz]^T, fp32, no epilogue
int launch_gemm_bf16_tc_splitk(const __nv_bfloat16* A, const __nv_bfloat16* W, float* partials, int M, int N, int K,
                               int splits, cudaStream_t st, bool pdl, DepFlag dep, int flags) {
    flags &= GEMM_F16;
    if (M <= 0 || N <= 0) return 0;
    if (K % BK != 0 || N % 32 != 0 || splits < 1 || (K / BK) % splits != 0) throw CudaError("gemm_bf16_tc_splitk: bad shape");
    if (!g_encode) { std::string err; if (!gemm_tc_init(&err)) throw CudaError(err); }
    const int bn = pick_bn(M, N, splits);
    CUtensorMap tmA, tmB;
    const int abox = a_box_rows_for(M);
    tma_encode_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint32_t)abox);
    tma_encode_bf16_2d(&tmB, W, (uint64_t)N, (uint64_t)K, (uint32_t)bn);
    if (bn == 128) return launch_bn<128>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl, dep);
    if (bn == 64) return launch_bn<64>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl, dep);
    return launch_bn<32>(tmA, tmB, nullptr, nullptr, partials, M, N, K, flags, st, splits, abox, pdl, dep);
}


bool decode_chain_supported(int M, int H, int FF) {
    return M >= 1 && H % 128 == 0 && H <= 1024 && (H / BK) % CH_SPLITS == 0 && FF % CH_BN == 0 && (FF / BK) % CH_SPLITS == 0;
}

// one launch = the phases of `a.phases` (DC_* bits) for one layer boundary of the decode step
void launch_decode_chain(const DecodeChainArgs& a, cudaStream_t st, bool pdl) {
    if (a.M <= 0 || a.phases == 0) return;
    if (!decode_chain_supported(a.M, a.H, a.FF)) throw CudaError("decode_chain: unsupported geometry");
    if (!g_encode) { std::string err; if (!gemm_tc_init(&err)) throw CudaError(err); }
    static bool attr_set[64] = {};
    constexpr size_t smem = CH_STAGES * (BM * BK * 2 + CH_BN * BK * 2) + 1024;
    const int n_sm = sm_count();
    if (first_on_device(attr_set))
        CUDA_CHECK(cudaFuncSetAttribute(decode_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int abox = a_box_rows_for(a.M);
    const int H = a.H, FF = a.FF;
    CUtensorMap tATT, tWo, tXn, tWfc, tFF, tWproj, tWqkv;
    tma_encode_bf16_2d(&tATT, a.ATT, (uint64_t)a.M, (uint64_t)H, (uint32_t)abox);
    tma_encode_bf16_2d(&tXn, a.Xn, (uint64_t)a.M, (uint64_t)H, (uint32_t)abox);
    tma_encode_bf16_2d(&tFF, a.FFb, (uint64_t)a.M, (uint64_t)FF, (uint32_t)abox);
    tma_encode_bf16_2d(&tWo, a.Wo, (uint64_t)H, (uint64_t)H, CH_BN);
    tma_encode_bf16_2d(&tWfc, a.Wfc, (uint64_t)FF, (uint64_t)H, CH_BN);
    tma_encode_bf16_2d(&tWproj, a.Wproj, (uint64_t)H, (uint64_t)FF, CH_BN);
    tma_encode_bf16_2d(&tWqkv, a.Wqkv ? a.Wqkv : a.Wo, (uint64_t)(a.Wqkv ? 3 * H : H), (uint64_t)H, CH_BN);
    ChainParams P{};
    P.phases = a.phases; P.M = a.M; P.H = H; P.FF = FF; P.abox = abox; P.eps = a.eps;
    P.proj_bias = a.proj_bias; P.ln2_w = a.ln2_w; P.ln2_b = a.ln2_b; P.fc_bias = a.fc_bias; P.fc2_bias = a.fc2_bias;
    P.ln1_w = a.ln1_w; P.ln1_b = a.ln1_b; P.qkv_bias = a.qkv_bias;
    P.X = a.X; P.Xn = a.Xn; P.FFb = a.FFb; P.QKV = a.QKV; P.PART = a.PART; P.sync = a.sync;
    double fl = 0, by = 0;
    const double M = a.M;
    if (a.phases & DC_PROJ) { fl += 2.0 * M * H * H; by += 2.0 * (M * H + (double)H * H) + 4.0 * CH_SPLITS * M * H; }
    if (a.phases & DC_LN2) by += (8.0 + 4.0 * CH_SPLITS + 2.0) * M * H;
    if (a.phases & DC_FC) { fl += 2.0 * M * H * FF; by += 2.0 * (M * H + (double)H * FF) + 2.0 * M * FF; }
    if (a.phases & DC_FC2) { fl += 2.0 * M * H * FF; by += 2.0 * (M * FF + (double)H * FF) + 4.0 * CH_SPLITS * M * H; }
    if (a.phases & DC_LN1) by += (8.0 + 4.0 * CH_SPLITS + 2.0) * M * H;
    if (a.phases & DC_QKV) { fl += 6.0 * M * H * H; by += 2.0 * (M * H + 3.0 * H * H) + 12.0 * M * H; }
    ProfScope ps(KF_DECODE_CHAIN, st, fl, by);
    launch_k(decode_chain_kernel, dim3(n_sm), dim3(kThreads), smem, st, pdl, tATT, tWo, tXn, tWfc, tFF, tWproj, tWqkv, P);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
