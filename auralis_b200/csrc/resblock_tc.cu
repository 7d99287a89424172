// One whole vocoder ResBlock1 as one tensor-core kernel (fast mode, stages with C <= 64 channels):
//
//   for t = 0, 1, 2:   x <- x + c2_t(lrelu(c1_t(lrelu(x), dil_t)), dil 1)        then   MRF sum (=|+=) x
//
// conv1d_tc runs this as six launches with the residual stream (fp32 r1, r2) and every activation (fp16 atoms) passing
// through HBM between them.  Here a persistent CTA takes one time tile of one batch item and keeps the whole chain on chip:
//   * the tile's span (tile_rows + 2 * halo rows, halo = (K-1)/2 * (dil_0 + dil_1 + dil_2 + 3)) of the input atoms and of
//     the fp32 residual x are bulk-copied into shared memory once;
//   * the six convs run back to back on two atom buffers (c1 writes T, c2 writes A: c2's atoms overwrite c1's input) and
//     the fp32 residual buffer R, which c2 updates in place;
//   * only the tile's own rows leave the chip: the MRF sum (store or accumulate) and, optionally, its activated atoms.
// Every conv is the implicit GEMM of conv1d_tc with the same arithmetic per output element: wgmma m64nCk16 (f16 x f16 ->
// f32) over tap j, then k-step, accumulated from zero; epilogue ((acc + bias) + resid) + base, atoms lrelu(y * scale16).
// Each conv only computes the rows the next one needs: its valid span shrinks by its own halo on both sides.  Atom rows
// outside the item's signal [0, L_i) are written as zeros, as the zero pads of the six-launch path hold them.
// Warp roles: warps 0-7 two consumer warpgroups (MMA + epilogue; warp 0 also issues the span loads), warp 8 streams the
// packed weight tiles (one per conv and tap) through a bulk-copy ring.
#include <algorithm>

#include "hopper.cuh"
#include "kernels.h"

namespace xtts {
namespace {

using namespace hop;

constexpr int kConsumersRb = 256, kThreadsRb = kConsumersRb + 32, kConsumerWarpsRb = kConsumersRb / 32;
__device__ __forceinline__ float lrelu_rb(float v, float slope) { return v > 0.f ? v : v * slope; }

struct ResblockTcParams {
    const __half* xa;              // input atoms [batch][C/8][lpad][8]: lrelu(x)
    const float* x;                // residual stream [batch][C][L] fp32
    const __half* w[6];            // packed weights (conv1d_tc_pack) of c1_0, c2_0, c1_1, c2_1, c1_2, c2_2
    const float* bias[6];
    float* zs;                     // MRF sum [batch][C][L]
    __half* pa;                    // lrelu(sum * scale16, slope) atoms [batch][C/8][lpad][8], or nullptr
    int L, lpad, K, mode, dil[3];
    float slope, scale16;
    int halo, tile_rows, batch;
    int item_L[kVocMaxItems];
};

// Shared memory: A and T atom buffers [C/8][S][8] fp16, R [C][S + 4] fp32, weight ring [RING][C/8][C][8] fp16.
// The +4-float row pad keeps R's epilogue access (8 rows x 4 column pairs per warp) conflict-free.  A tap's MMAs take
// well under a microsecond, so the ring is as deep as the budget allows to hide the weight tiles' L2 latency: 3 tiles of
// 8 KB at C = 64, 12 of 2 KB at C = 32.
template <int C, int MB>
struct RbGeom {
    static constexpr int S = 128 * MB, LDR = S + 4, PL = C / 8, RING = C == 32 ? 12 : 3;
    static constexpr uint32_t a_plane = S * 16, a_buf = PL * a_plane, r_bytes = C * LDR * 4, b_stage = C * C * 2;
    static constexpr uint32_t smem = 2 * a_buf + r_bytes + RING * b_stage;
};

template <int C, int MB>
__global__ void __launch_bounds__(kThreadsRb, 1) resblock_tc_kernel(const ResblockTcParams P) {
    using G = RbGeom<C, MB>;
    constexpr int S = G::S, LDR = G::LDR, PL = G::PL, KS = C / 16, RING = G::RING;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t x_full, b_full[RING], b_empty[RING];
    __shared__ float sbias[6][C];
    __shared__ int s_cum[kVocMaxItems + 1], s_len[kVocMaxItems];
    uint8_t* sA = smem;
    uint8_t* sT = smem + G::a_buf;
    float* sR = reinterpret_cast<float*>(smem + 2 * G::a_buf);
    uint8_t* sB = smem + 2 * G::a_buf + G::r_bytes;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int TR = P.tile_rows, H = P.halo, cK = (P.K - 1) / 2;
    if (threadIdx.x == 0) {
        int c = 0;
        for (int i = 0; i < P.batch; ++i) {
            const int Li = P.item_L[i];
            s_cum[i] = c; s_len[i] = Li;
            c += Li > 0 ? ceil_div(Li, TR) : 0;
        }
        s_cum[P.batch] = c;
        mbar_init(&x_full, 1);
        for (int i = 0; i < RING; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], kConsumerWarpsRb); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // the six launches' bias table: bias + cbias with no speaker bias (+ 0.f, kept for the sign of zero)
    for (int i = threadIdx.x; i < 6 * C; i += blockDim.x) sbias[i / C][i % C] = __fadd_rn(__ldg(P.bias[i / C] + i % C), 0.f);
    __syncthreads();
    const int total_tiles = s_cum[P.batch];
    auto decode_tile = [&](int tile, int& zi, int& tx, int& Li) {
        zi = 0;
        while (zi + 1 < P.batch && tile >= s_cum[zi + 1]) ++zi;
        Li = s_len[zi];
        tx = tile - s_cum[zi];
    };

    if (warp == kConsumerWarpsRb) {
        // ------------------------------------------------ producer: the weight tile of every (conv, tap), in MMA order
        if (lane == 0) {
            int it = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x)
                for (int i = 0; i < 6; ++i)
                    for (int j = 0; j < P.K; ++j, ++it) {
                        const int s = it % RING;
                        mbar_wait(&b_empty[s], ((it / RING) & 1) ^ 1);
                        mbar_expect_tx(&b_full[s], G::b_stage);
                        bulk_g2s(sB + (size_t)s * G::b_stage, P.w[i] + (size_t)j * (G::b_stage / 2), G::b_stage, &b_full[s]);
                    }
        }
    } else {
        // ------------------------------------------------ consumers: warpgroup wg takes the 64-row blocks 2m + wg of a conv
        const int wg = warp >> 2, tid = threadIdx.x;
        auto cbar = [] { asm volatile("bar.sync 1, %0;" ::"r"(kConsumersRb) : "memory"); };
        const bool accum = P.mode == CONV_ACCUM;
        const size_t Ls = (size_t)P.L;
        int it = 0, lt = 0;
        float acc[MB][C / 2];
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
            int zi, tx, Li;
            decode_tile(tile, zi, tx, Li);
            const int T0 = tx * TR, g0 = T0 - H;                    // span row p is time step g0 + p
            const int ga = max(0, g0), gb = min(Li, g0 + S);         // signal rows of the span
            const int n4 = ((gb - ga) + 3) & ~3;                     // fp32 rows copied: whole 16-byte units (L % 4 == 0)
            const float* xsrc = P.x + (size_t)zi * C * Ls;
            if (warp == 0) {
                if (lane == 0) mbar_expect_tx(&x_full, (uint32_t)(PL * (gb - ga) * 16 + C * n4 * 4));
                __syncwarp();
                for (int q = lane; q < PL + C; q += 32) {
                    if (q < PL)
                        bulk_g2s(sA + (size_t)q * G::a_plane + (size_t)(ga - g0) * 16,
                                 P.xa + (((size_t)zi * PL + q) * P.lpad + kAtomPadL + ga) * 8, (uint32_t)(gb - ga) * 16u, &x_full);
                    else
                        bulk_g2s(sR + (size_t)(q - PL) * LDR + (ga - g0), xsrc + (size_t)(q - PL) * Ls + ga, (uint32_t)n4 * 4u,
                                 &x_full);
                }
            }
            for (int i = tid; i < PL * S; i += kConsumersRb) {        // span rows outside the signal: zero atoms
                const int p = i % S;
                if (p < ga - g0 || p >= gb - g0) *reinterpret_cast<uint4*>(sA + (size_t)i * 16) = make_uint4(0u, 0u, 0u, 0u);
            }
            mbar_wait(&x_full, lt & 1);
            fence_proxy_async_smem();
            cbar();

            int e = 0;                                               // span rows consumed so far on each side
            for (int ci = 0; ci < 6; ++ci) {
                const int t = ci >> 1;
                const bool is_c2 = ci & 1;
                const int dil = is_c2 ? 1 : P.dil[t], h = cK * dil;
                const int lo = e + h, hi = S - e - h;                    // output rows [lo, hi)
                e += h;
                const uint32_t in_addr = smem_u32(is_c2 ? sT : sA);
#pragma unroll
                for (int m = 0; m < MB; ++m)
#pragma unroll
                    for (int q = 0; q < C / 2; ++q) acc[m][q] = 0.f;
                int prev = -1;
                for (int j = 0; j < P.K; ++j, ++it) {
                    const int s = it % RING;
                    mbar_wait(&b_full[s], (it / RING) & 1);
                    const uint32_t b_addr = smem_u32(sB + (size_t)s * G::b_stage);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < KS; ++k) {
                        const uint64_t bd = desc_nosw(b_addr + (uint32_t)(2 * k) * (C * 16), C * 16);
#pragma unroll
                        for (int m = 0; m < MB; ++m) {
                            // the last block ends at hi; blocks past it repeat it (kept uniform: no divergent wgmma)
                            // and store nothing
                            const int p0 = min(lo + 64 * (2 * m + wg), hi - 64);
                            const uint64_t ad = desc_nosw(in_addr + (uint32_t)(2 * k) * G::a_plane +
                                                              (uint32_t)(p0 + (j - cK) * dil) * 16u, G::a_plane);
                            Wgmma<C>::run(acc[m], ad, bd, 1, true);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                                 // the previous tap's wgmmas have retired
#pragma unroll
                    for (int m = 0; m < MB; ++m) fence_acc(acc[m]);
                    __syncwarp();
                    if (lane == 0 && prev >= 0) mbar_arrive(&b_empty[prev]);
                    prev = s;
                }
                wgmma_wait<0>();
#pragma unroll
                for (int m = 0; m < MB; ++m) fence_acc(acc[m]);
                __syncwarp();
                if (lane == 0) mbar_arrive(&b_empty[prev]);

                // ---- epilogue: a lane holds columns (col, col + 1) of rows r and r + 8 of each of its blocks
                const float* sb = sbias[ci];
                uint8_t* out16 = ci == 5 ? nullptr : (is_c2 ? sA : sT);
#pragma unroll
                for (int m = 0; m < MB; ++m) {
                    const int nom = lo + 64 * (2 * m + wg), p0 = min(nom, hi - 64);
                    if (nom >= hi) continue;
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int p = p0 + 16 * (warp & 3) + (lane >> 2) + 8 * hh;
                        if (p < nom) continue;                       // the shifted last block: rows the block before wrote
                        const int g = g0 + p;
                        const bool sig = g >= 0 && g < Li;
                        if (ci == 5 && !sig) continue;
#pragma unroll
                        for (int ii = 0; ii < C / 8; ++ii) {
                            const int col = 8 * ii + 2 * (lane & 3);
                            float y0 = acc[m][4 * ii + 2 * hh] + sb[col], y1 = acc[m][4 * ii + 2 * hh + 1] + sb[col + 1];
                            if (is_c2) {
                                float* r = sR + (size_t)col * LDR + p;
                                y0 += r[0]; y1 += r[LDR];
                                if (ci == 5) {
                                    float* op = P.zs + ((size_t)zi * C + col) * Ls + g;
                                    if (accum) { y0 += op[0]; y1 += op[Ls]; }
                                    op[0] = y0; op[Ls] = y1;
                                    if (P.pa)
                                        *reinterpret_cast<__half2*>(P.pa + (((size_t)zi * PL + ii) * P.lpad + kAtomPadL + g) * 8 + 2 * (lane & 3)) =
                                            __floats2half2_rn(lrelu_rb(y0 * P.scale16, P.slope), lrelu_rb(y1 * P.scale16, P.slope));
                                    continue;
                                }
                                r[0] = y0; r[LDR] = y1;
                            }
                            const __half2 v = sig ? __floats2half2_rn(lrelu_rb(y0, P.slope), lrelu_rb(y1, P.slope))
                                                  : __floats2half2_rn(0.f, 0.f);
                            *reinterpret_cast<__half2*>(out16 + ((size_t)ii * S + p) * 16 + 4 * (lane & 3)) = v;
                        }
                    }
                }
                fence_proxy_async_smem();                            // the next conv's wgmmas / the next span load
                cbar();
            }
        }
    }
    __syncthreads();
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// 64-row blocks per consumer warpgroup: the span is 128 * MB rows; each fits the shared-memory budget of conv1d_tc
template <int C> constexpr int rb_mb() { return C == 64 ? 3 : 6; }

static int rb_halo(int K, const int* dil) { return (K - 1) / 2 * (dil[0] + dil[1] + dil[2] + 3); }
static int rb_span(int C) { return C == 64 ? 128 * rb_mb<64>() : (C == 32 ? 128 * rb_mb<32>() : 0); }

// The span's fp32 residual rows are bulk-copied in whole 16-byte units, so a tile's first time step (a multiple of
// tile_rows, minus the halo) and the row stride L must be multiples of 4 floats: the halo must be a multiple of 4
// (every k at dilations 1, 3, 5: 12 * (k-1)/2) and so must L (every stage of up-rates 8, 8, 2, 2).
int resblock_tc_tile_rows(int C, int K, const int* dil, int L) {
    const int S = rb_span(C);
    if (S == 0 || K < 1 || K % 2 == 0 || dil[0] < 1 || dil[1] < 1 || dil[2] < 1 || L % 4 != 0) return 0;
    const int H = rb_halo(K, dil), tr = S - 2 * H;
    return (H % 4 == 0 && tr >= 64) ? tr : 0;
}

template <int C>
static void launch_rb(const ResblockTcParams& P, dim3 grid, cudaStream_t st) {
    constexpr int MB = rb_mb<C>();
    static_assert(RbGeom<C, MB>::smem <= (uint32_t)kMaxDynTc, "resblock_tc: shared memory budget");
    static bool attr[64] = {};
    if (first_on_device(attr))
        CUDA_CHECK(cudaFuncSetAttribute(resblock_tc_kernel<C, MB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        RbGeom<C, MB>::smem));
    resblock_tc_kernel<C, MB><<<grid, kThreadsRb, RbGeom<C, MB>::smem, st>>>(P);
}

void launch_resblock_tc(const __half* xa, const float* x, const __half* const* wblob, const float* const* bias, float* zs,
                        __half* pa, int C, int L, int lpad, int K, const int* dil, int mode, float scale16, int batch,
                        const int* item_len, cudaStream_t st) {
    if (L <= 0 || batch <= 0) return;
    const int TR = resblock_tc_tile_rows(C, K, dil, L);
    if (TR == 0) throw CudaError("resblock_tc: unsupported geometry");
    if (batch > kVocMaxItems) throw CudaError("resblock_tc: batch exceeds kVocMaxItems");
    if (mode != CONV_STORE && mode != CONV_ACCUM) throw CudaError("resblock_tc: mode must be STORE or ACCUM");
    if (((uintptr_t)x & 15) != 0 || lpad < kAtomPadL + L) throw CudaError("resblock_tc: buffer layout");
    ResblockTcParams P{};
    P.xa = xa; P.x = x; P.zs = zs; P.pa = pa;
    for (int i = 0; i < 6; ++i) { P.w[i] = wblob[i]; P.bias[i] = bias[i]; }
    P.L = L; P.lpad = lpad; P.K = K; P.mode = mode;
    for (int t = 0; t < 3; ++t) P.dil[t] = dil[t];
    P.slope = 0.1f; P.scale16 = scale16;
    P.halo = rb_halo(K, dil); P.tile_rows = TR; P.batch = batch;
    double Lsum = 0;
    int total_tiles = 0;
    for (int i = 0; i < batch; ++i) {
        const int Li = item_len ? item_len[i] : L;
        if (Li < 0 || Li > L) throw CudaError("resblock_tc: item length out of range");
        P.item_L[i] = Li;
        Lsum += Li;
        total_tiles += Li > 0 ? ceil_div(Li, TR) : 0;
    }
    if (total_tiles == 0) return;
    const int n_sm = sm_count();
    const int cap = (g_voc_sm_cap > 0 && g_voc_sm_cap < n_sm) ? g_voc_sm_cap : n_sm;
    dim3 grid(std::min(total_tiles, cap));
    // algorithmic counts (halo recompute excluded): six convs; atoms + fp32 x in, the MRF sum out (accumulate: read too)
    const double flops = 6.0 * 2.0 * C * C * K * Lsum;
    const double bytes = Lsum * C * (2.0 + 4.0 + (mode == CONV_ACCUM ? 8.0 : 4.0) + (pa ? 2.0 : 0.0)) + 6.0 * 2.0 * C * C * K;
    ProfScope ps(KF_RESBLOCK_TC, st, flops, bytes);
    if (C == 64) launch_rb<64>(P, grid, st);
    else launch_rb<32>(P, grid, st);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
