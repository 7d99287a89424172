// Dilated Conv1d ("same" padding) as an implicit GEMM on the Hopper tensor cores (fast mode of the vocoder).
//
//   y[co][t] = bias[co] + cbias[co] + resid[co][t] + sum_j sum_ci W_j[co][ci] * a[ci][t + (j-c)*d]
//
// where `a` is the ALREADY ACTIVATED fp16 input kept in HBM in the tensor-core operand layout
//   "atoms":  [C/8 plane][PADL + L + PADR time rows][8 channels]   (16-byte atoms, zero pads)
// which is byte-for-byte the wgmma no-swizzle K-major image (8-row core matrices 128 B apart => rows linear in time), so
//   * the A tile of a ci-chunk is `CK/8` contiguous cp.async.bulk copies (one per plane), a tap is a start-address
//     shift of j*d rows inside the staged tile (no im2col, no conversion work in this kernel);
//   * weights are pre-packed per (ci-chunk, tap) into the same layout: one bulk copy per tile.
// wgmma.mma_async m64nNk16 (f16 x f16 -> f32), accumulators in registers: each of the two consumer warpgroups owns MB
// blocks of 64 time rows (MB * N / 2 accumulators per thread), so a tile is 128 * MB time rows x N output channels and
// every staged weight tile feeds all of them.  The consumers' epilogue (straight from the accumulators) can emit
//   * out32: fp32 channel-major [C][L]  (store or accumulate)  — the residual stream / MRF sum
//   * out16: lrelu(y, slope_out) as fp16 atoms                 — the next conv's operand, written once, read once.
// Warp roles: warps 0-7 consumer warpgroups (MMA + epilogue), warp 8 bulk-copy producer.  Persistent CTAs walk the tile list.
//
// Replaces the cuDNN fp16-autocast Conv1d calls of HifiganGenerator.forward / ResBlock1.forward
// (hifigan_decoder.py:76-91,241-259; the reference runs them in fp16 under torch.amp.autocast on GPU, App. B.8).
#include <algorithm>
#include <vector>

#include "hopper.cuh"
#include "kernels.h"

namespace xtts {
namespace {

using namespace hop;

constexpr int kConsumers = 256, kThreadsTc = kConsumers + 32, kConsumerWarps = kConsumers / 32;
constexpr int SA = 2, SB = 3;          // ring depths (activation chunks, weight tiles)
__device__ __forceinline__ float lrelu_s(float v, float slope) { return v > 0.f ? v : v * slope; }

struct ConvTcParams {
    const __half* a16;       // input atoms  [batch][Cin/8][lpad][8]
    const __half* wblob;
    const float* bias; const float* cbias; const float* resid;
    float* out32;            // [batch][Cout][L] or nullptr
    __half* out16;           // output atoms [batch][Cout/8][lpad][8] or nullptr
    int Cin, Cout, L, lpad, K, dil, mode;
    float slope_out, scale16;   // out16 = lrelu(y * scale16, slope_out)
    int center;              // tap j reads a[t + (j - center) * dil]
    int up;                  // 0: Conv1d.  u > 0: ConvTranspose1d(stride u, kernel 2u, pad u/2) as u two-tap phases:
                             //    GEMM channel n' = co * u + phase, GEMM row s -> output step s*u + phase - u/2
    int Cr, Lout, lpad_out;  // real output channels, output length, padded rows of the output atoms
    int CK;         // input channels per chunk (<= 64, multiple of 16)
    int rows;       // time rows staged per chunk = tile_rows + (K-1)*dil
    int cbias_bs;   // elements between the speaker-bias vectors of consecutive batch items
    int tile_rows, tiles_n, batch; // persistent-CTA tile space: per item ceil(rows_i / tile_rows) x tiles_n tiles
    int item_L[kVocMaxItems];      // ragged batch: input time steps of each item (<= L; buffers are strided by L)
};

// N output channels (GEMM columns) per tile, MB 64-row blocks per consumer warpgroup (tile_rows = 128 * MB)
template <int N, int MB>
__global__ void __launch_bounds__(kThreadsTc, 1)
conv1d_tc_kernel(const ConvTcParams P) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t a_full[SA], a_empty[SA], b_full[SB], b_empty[SB];
    __shared__ __align__(16) float sbias[2][N];     // per-tile bias + speaker bias (double buffered across tiles)
    __shared__ int s_cum[kVocMaxItems + 1], s_len[kVocMaxItems];   // ragged batch: first tile / input length of every item

    trace_pt(TR_CONV, 0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int halo = P.center * P.dil;
    const int planes = P.CK / 8, ksteps = P.CK / 16, nch = P.Cin / P.CK;
    const uint32_t a_plane = (uint32_t)P.rows * 16u;               // bytes per ci-plane of a staged chunk
    const uint32_t a_stage = a_plane * planes;
    constexpr uint32_t b_plane = (uint32_t)N * 16u;
    const uint32_t b_stage = b_plane * planes;
    uint8_t* sA = smem;
    uint8_t* sB = smem + ((SA * a_stage + 127) & ~127u);
    const int tiles_n = P.tiles_n;
    const int extra_rows = P.up ? 1 : 0;             // a transposed conv also consumes the zero row x[L]

    if (threadIdx.x == 0) {
        int c = 0;
        for (int i = 0; i < P.batch; ++i) {
            const int Li = P.item_L[i];
            s_cum[i] = c; s_len[i] = Li;
            c += (Li > 0 ? ceil_div(Li + extra_rows, P.tile_rows) : 0) * tiles_n;
        }
        s_cum[P.batch] = c;
        for (int i = 0; i < SA; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], kConsumerWarps); }
        for (int i = 0; i < SB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int total_tiles = s_cum[P.batch];
    // tile -> (batch item, time tile, C_out tile); every role walks the same compact tile list
    auto decode_tile = [&](int tile, int& zi, int& tx, int& ty, int& Li) {
        zi = 0;
        while (zi + 1 < P.batch && tile >= s_cum[zi + 1]) ++zi;
        Li = s_len[zi];
        const int tt = ceil_div(Li + extra_rows, P.tile_rows);
        const int local = tile - s_cum[zi];
        tx = local % tt; ty = local / tt;
    };

    if (warp == kConsumerWarps) {
        // ------------------------------------------------ producer: activation planes + weight tiles, all bulk copies
        if (lane == 0) {
            int ita = 0, itb = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                int zi, tx, ty, Li;
                decode_tile(tile, zi, tx, ty, Li);
                const size_t zo = (size_t)zi;
                const int T0 = tx * P.tile_rows;
                const __half* wsrc = P.wblob + (size_t)ty * nch * P.K * (b_stage / 2);
                const __half* asrc = P.a16 + zo * (size_t)(P.Cin / 8) * P.lpad * 8;
                const int row0 = T0 - halo + kAtomPadL;             // first staged time row inside the padded plane
                int wt = 0;
                for (int c = 0; c < nch; ++c, ++ita) {
                    const int sa = ita % SA;
                    mbar_wait(&a_empty[sa], ((ita / SA) & 1) ^ 1);
                    mbar_expect_tx(&a_full[sa], a_stage);
                    for (int p = 0; p < planes; ++p)
                        bulk_g2s(sA + (size_t)sa * a_stage + (size_t)p * a_plane,
                                 asrc + ((size_t)(c * planes + p) * P.lpad + row0) * 8, a_plane, &a_full[sa]);
                    for (int j = 0; j < P.K; ++j, ++itb, ++wt) {
                        const int s = itb % SB;
                        mbar_wait(&b_empty[s], ((itb / SB) & 1) ^ 1);
                        mbar_expect_tx(&b_full[s], b_stage);
                        bulk_g2s(sB + (size_t)s * b_stage, wsrc + (size_t)wt * (b_stage / 2), b_stage, &b_full[s]);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------ consumer warpgroup wg: time rows [T0 + 64*MB*wg, +64*MB) of a tile.
        // Weight slots are handed back one tap late (after the next tap's wgmmas are issued), so the tensor cores never
        // drain between taps; an activation slot is handed back with the last weight slot of its chunk.
        const int wg = warp >> 2, etid = threadIdx.x;
        const bool has_res = P.resid != nullptr, accum = (P.mode == CONV_ACCUM);
        const size_t Ls = (size_t)P.Lout;
        int ita = 0, itb = 0, lt = 0;
        float acc[MB][N / 2];
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
            int zi, tx, ty, Li;
            decode_tile(tile, zi, tx, ty, Li);
            const size_t zo = (size_t)zi;
            const int row_limit = Li + extra_rows, Lout_i = P.up ? Li * P.up : Li;
            const int T0 = tx * P.tile_rows, n0 = ty * N;
            const float* cbias = P.cbias ? P.cbias + zo * P.cbias_bs : nullptr;
            float* sb = sbias[lt & 1];
            for (int j = etid; j < N; j += kConsumers) {
                const int co = P.up ? (n0 + j) / P.up : n0 + j;      // GEMM column -> output channel (transposed conv: co * u + phase)
                sb[j] = (P.bias ? __ldg(P.bias + co) : 0.f) + (cbias ? __ldg(cbias + co) : 0.f);
            }
#pragma unroll
            for (int m = 0; m < MB; ++m)
#pragma unroll
                for (int i = 0; i < N / 2; ++i) acc[m][i] = 0.f;
            const uint32_t row_off = (uint32_t)(64 * MB * wg) * 16u;
            int prev_b = -1, prev_a = -1;
            auto release = [&] {
                __syncwarp();
                if (lane == 0) {
                    if (prev_b >= 0) mbar_arrive(&b_empty[prev_b]);
                    if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                }
                prev_b = prev_a = -1;
            };
            for (int c = 0; c < nch; ++c, ++ita) {
                const int sa = ita % SA;
                mbar_wait(&a_full[sa], (ita / SA) & 1);
                const uint32_t a_addr = smem_u32(sA + (size_t)sa * a_stage) + row_off;
                for (int j = 0; j < P.K; ++j, ++itb) {
                    const int sbi = itb % SB;
                    mbar_wait(&b_full[sbi], (itb / SB) & 1);
                    const uint32_t b_addr = smem_u32(sB + (size_t)sbi * b_stage);
                    wgmma_fence();
                    for (int k = 0; k < ksteps; ++k) {
                        const uint64_t bd = desc_nosw(b_addr + (uint32_t)(2 * k) * b_plane, b_plane);
#pragma unroll
                        for (int m = 0; m < MB; ++m) {
                            const uint64_t ad = desc_nosw(a_addr + (uint32_t)(2 * k) * a_plane + (uint32_t)(m * 64 + j * P.dil) * 16u, a_plane);
                            Wgmma<N>::run(acc[m], ad, bd, 1, true);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                             // the previous tap's wgmmas have retired
#pragma unroll
                    for (int m = 0; m < MB; ++m) fence_acc(acc[m]);
                    release();
                    prev_b = sbi;
                    if (j == P.K - 1) prev_a = sa;
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int m = 0; m < MB; ++m) fence_acc(acc[m]);
            release();
            asm volatile("bar.sync 1, %0;" ::"r"(kConsumers) : "memory");      // bias table visible to every consumer warp

            // ---- epilogue: a lane holds GEMM columns (col, col+1) of time rows s and s + 8 of each 64-row block
            float* out32 = P.out32 ? P.out32 + zo * P.Cr * P.Lout : nullptr;
            const float* resid = has_res ? P.resid + zo * P.Cr * P.Lout : nullptr;
            __half* out16 = P.out16 ? P.out16 + zo * (size_t)(P.Cr / 8) * P.lpad_out * 8 : nullptr;
            const int s_base = T0 + 64 * MB * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
            for (int m = 0; m < MB; ++m)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int srow = s_base + 64 * m + 8 * h;
                    if (srow >= row_limit) continue;
#pragma unroll
                    for (int i = 0; i < N / 8; ++i) {
                        const int col = 8 * i + 2 * (lane & 3);
                        const float v0 = acc[m][4 * i + 2 * h] + sb[col], v1 = acc[m][4 * i + 2 * h + 1] + sb[col + 1];
                        if (P.up) {
                            // ---- ConvTranspose1d: column n' = co * u + phase (u even: the pair is one channel, phases p, p + 1)
                            const int u = P.up, np = n0 + col, co = np / u, p = np - co * u;
                            const int tt = srow * u - u / 2 + p;
                            const float w2[2] = {v0, v1};
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int t = tt + e;
                                if (t < 0 || t >= Lout_i) continue;
                                if (out32) out32[(size_t)co * Ls + t] = w2[e];
                                if (out16) out16[((size_t)(co / 8) * P.lpad_out + (t + kAtomPadL)) * 8 + (co % 8)] =
                                               __float2half_rn(lrelu_s(w2[e] * P.scale16, P.slope_out));
                            }
                            continue;
                        }
                        const int t = srow, co = n0 + col;
                        if (t >= Lout_i) continue;
                        float y0 = v0, y1 = v1;
                        if (has_res) { y0 += resid[(size_t)co * Ls + t]; y1 += resid[(size_t)(co + 1) * Ls + t]; }
                        if (out32) {
                            float* op = out32 + (size_t)co * Ls + t;
                            if (accum) { y0 += op[0]; y1 += op[Ls]; }
                            op[0] = y0; op[Ls] = y1;
                        }
                        if (out16) {                                 // (after an accumulate: the activated SUM)
                            const __half2 hv = __floats2half2_rn(lrelu_s(y0 * P.scale16, P.slope_out), lrelu_s(y1 * P.scale16, P.slope_out));
                            *reinterpret_cast<__half2*>(out16 + ((size_t)(co / 8) * P.lpad_out + (t + kAtomPadL)) * 8 + (co % 8)) = hv;
                        }
                    }
                }
        }
    }
    __syncthreads();
    trace_pt(TR_CONV, 2);
}

// zero the head pad and the rows behind the signal, for every plane of every batch item.  Ragged batches: item i's signal
// ends at its own L_i; the rows a valid output can reach behind it (halo <= kAtomPadL) plus one tile of slack are cleared,
// rows further out are only ever read by output rows that are never stored.
struct ZeroPadLens { int planes_per_item; int len[kVocMaxItems]; };
__global__ void atoms_zero_pads_kernel(uint4* __restrict__ buf, int planes_total, int lpad, const ZeroPadLens Z) {
    const int pl = blockIdx.y;
    if (pl >= planes_total) return;
    uint4* p = buf + (size_t)pl * lpad;
    const int L = Z.len[pl / Z.planes_per_item];
    const int tail0 = kAtomPadL + L;
    const int n = kAtomPadL + min(lpad - tail0, 640);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int row = (i < kAtomPadL) ? i : tail0 + (i - kAtomPadL);
        p[row] = make_uint4(0u, 0u, 0u, 0u);
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
XTTS_TRACE_SETTER(trace_set_conv)

ConvTcPlan conv1d_tc_plan(int Cin, int Cout, int K) {
    ConvTcPlan pl{};
    pl.N = Cout > 256 ? 256 : Cout;
    pl.CK = Cin >= 64 ? 64 : Cin;
    pl.n_tiles = ceil_div(Cout, pl.N);
    // 128-row blocks per tile: MB = nacc 64-row blocks per consumer warpgroup, MB * N / 2 <= 128 accumulator registers
    // per thread (N = 256: 1, N = 128: 2); narrower tiles stop at 4 (512 rows: the time tiling of atoms_lpad)
    pl.nacc = pl.N >= 256 ? 1 : (pl.N >= 128 ? 2 : 4);
    pl.ok = (Cin % pl.CK == 0) && (pl.CK % 16 == 0) && (pl.N == 32 || pl.N == 64 || pl.N == 128 || pl.N == 256) &&
            (Cout % pl.N == 0) && K >= 1;
    pl.tile_halves = (size_t)(pl.CK / 8) * pl.N * 8;
    pl.blob_halves = (size_t)pl.n_tiles * (Cin / pl.CK) * K * pl.tile_halves;
    return pl;
}

// w: folded Conv1d weight [Cout][Cin][K] fp32 -> blob [n_tile][ci-chunk][tap][plane][co][8] fp16
void conv1d_tc_pack(const float* w, int Cin, int Cout, int K, const ConvTcPlan& pl, __half* blob) {
    const int nch = Cin / pl.CK, planes = pl.CK / 8;
    for (int nt = 0; nt < pl.n_tiles; ++nt)
        for (int c = 0; c < nch; ++c)
            for (int j = 0; j < K; ++j) {
                __half* tile = blob + (((size_t)nt * nch + c) * K + j) * pl.tile_halves;
                for (int p = 0; p < planes; ++p)
                    for (int n = 0; n < pl.N; ++n)
                        for (int e = 0; e < 8; ++e) {
                            const int co = nt * pl.N + n, ci = c * pl.CK + p * 8 + e;
                            tile[((size_t)p * pl.N + n) * 8 + e] = __float2half_rn(w[((size_t)co * Cin + ci) * K + j]);
                        }
            }
}

int atoms_lpad(int L) { return kAtomPadL + ceil_div(L + 1, 512) * 512 + kAtomPadR; }

constexpr int kMaxDynTc = 227 * 1024 - 4096;      // opt-in limit minus the kernel's static shared memory
template <int N, int MB>
static void launch_inst(const ConvTcParams& P, dim3 grid, size_t smem, cudaStream_t st) {
    static bool attr[64] = {};
    if (first_on_device(attr)) CUDA_CHECK(cudaFuncSetAttribute(conv1d_tc_kernel<N, MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynTc));
    conv1d_tc_kernel<N, MB><<<grid, kThreadsTc, smem, st>>>(P);
}

static void launch_tc_common(ConvTcParams& P, const ConvTcPlan& pl, int rows_to_cover, int batch, const int* item_len,
                             double flops, double bytes, cudaStream_t st) {
    const int tile = 128 * pl.nacc;
    P.CK = pl.CK;
    P.rows = tile + (P.K - 1) * P.dil;
    if (P.lpad < kAtomPadL + ceil_div(rows_to_cover, tile) * tile + (P.K - 1 - P.center) * P.dil || P.center * P.dil > kAtomPadL)
        throw CudaError("conv1d_tc: atom buffer pad too small");
    const size_t a_stage = (size_t)P.rows * 16 * (pl.CK / 8), b_stage = (size_t)pl.N * 16 * (pl.CK / 8);
    const size_t smem = ((SA * a_stage + 127) & ~(size_t)127) + SB * b_stage + 128;
    if (smem > (size_t)kMaxDynTc) throw CudaError("conv1d_tc: shared memory budget exceeded");
    if (batch > kVocMaxItems) throw CudaError("conv1d_tc: batch exceeds kVocMaxItems");
    P.tile_rows = tile; P.tiles_n = pl.n_tiles; P.batch = batch;
    const int extra = P.up ? 1 : 0;
    int total_tiles = 0;
    for (int i = 0; i < batch; ++i) {
        const int Li = item_len ? item_len[i] : P.L;
        if (Li < 0 || Li > P.L) throw CudaError("conv1d_tc: item length out of range");
        P.item_L[i] = Li;
        total_tiles += (Li > 0 ? ceil_div(Li + extra, tile) : 0) * P.tiles_n;
    }
    if (total_tiles == 0) return;
    const int n_sm = sm_count();
    const int cap = (g_voc_sm_cap > 0 && g_voc_sm_cap < n_sm) ? g_voc_sm_cap : n_sm;
    dim3 grid(std::min(total_tiles, cap));           // one persistent CTA per SM (of the SMs this launch may take)
    ProfScope ps(KF_CONV1D_TC, st, flops, bytes);
    switch (pl.N) {
        case 256: launch_inst<256, 1>(P, grid, smem, st); break;
        case 128: launch_inst<128, 2>(P, grid, smem, st); break;
        case 64: launch_inst<64, 4>(P, grid, smem, st); break;
        case 32: launch_inst<32, 4>(P, grid, smem, st); break;
        default: throw CudaError("conv1d_tc: tile width must be 32, 64, 128 or 256");
    }
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_conv1d_tc(const __half* a16, const __half* wblob, const ConvTcPlan& pl, const float* bias, const float* cbias,
                      const float* resid, float* out32, __half* out16, int Cin, int Cout, int L, int lpad, int K, int dil,
                      float slope_out, float scale16, int mode, int batch, int cbias_batch_stride, cudaStream_t st,
                      const int* item_len) {
    if (L <= 0 || batch <= 0) return;
    if (!pl.ok || K % 2 != 1) throw CudaError("conv1d_tc: unsupported geometry");
    double Lsum = 0;                                  // time steps actually computed (ragged batch: sum of the item lengths)
    for (int i = 0; i < batch; ++i) Lsum += item_len ? item_len[i] : L;
    ConvTcParams P{};
    P.a16 = a16; P.wblob = wblob; P.bias = bias; P.cbias = cbias; P.resid = resid; P.out32 = out32; P.out16 = out16;
    P.Cin = Cin; P.Cout = Cout; P.L = L; P.lpad = lpad; P.K = K; P.dil = dil; P.mode = mode; P.slope_out = slope_out;
    P.scale16 = scale16; P.center = (K - 1) / 2; P.up = 0; P.Cr = Cout; P.Lout = L; P.lpad_out = lpad;
    P.cbias_bs = cbias_batch_stride;
    // algorithmic traffic: fp16 atoms in, fp32 residual in, fp32 and/or fp16 out, weights once
    const double by = Lsum * (2.0 * Cin + (resid ? 4.0 * Cout : 0) + (out32 ? (mode == CONV_ACCUM ? 8.0 : 4.0) * Cout : 0) +
                              (out16 ? 2.0 * Cout : 0)) + 2.0 * Cin * Cout * K;
    launch_tc_common(P, pl, L, batch, item_len, 2.0 * Cin * Cout * K * Lsum, by, st);
}

// ConvTranspose1d(Cin -> Cr, kernel 2u, stride u, padding u/2) on the same kernel: u phases x 2 taps.
// `pl`/`wblob` come from conv1d_tc_plan(Cin, u*Cr, 2) / convT_tc_pack.
void launch_convT_tc(const __half* a16, const __half* wblob, const ConvTcPlan& pl, const float* bias, const float* cbias,
                     float* out32, __half* out16, int Cin, int Cr, int Lin, int lpad_in, int lpad_out, int u, float slope_out,
                     int batch, int cbias_batch_stride, cudaStream_t st, const int* item_len) {
    if (Lin <= 0 || batch <= 0) return;
    double Lsum = 0;
    for (int i = 0; i < batch; ++i) Lsum += item_len ? item_len[i] : Lin;
    if (!pl.ok || (u != 2 && u != 4 && u != 8) || Cr % 32 != 0) throw CudaError("convT_tc: unsupported geometry");
    ConvTcParams P{};
    P.a16 = a16; P.wblob = wblob; P.bias = bias; P.cbias = cbias; P.resid = nullptr; P.out32 = out32; P.out16 = out16;
    P.Cin = Cin; P.Cout = u * Cr; P.L = Lin; P.lpad = lpad_in; P.K = 2; P.dil = 1; P.mode = CONV_STORE; P.slope_out = slope_out;
    P.scale16 = 1.0f; P.center = 1; P.up = u; P.Cr = Cr; P.Lout = Lin * u; P.lpad_out = lpad_out;
    P.cbias_bs = cbias_batch_stride;
    const double by = Lsum * 2.0 * Cin + Lsum * u * Cr * ((out32 ? 4.0 : 0) + (out16 ? 2.0 : 0)) + 4.0 * Cin * Cr * u;
    launch_tc_common(P, pl, Lin + 1, batch, item_len, 4.0 * Cin * Cr * Lsum * u, by, st);
}

// ConvTranspose1d weight [Cin][Cr][2u] fp32 -> two-tap phase blob, GEMM column n' = co*u + p (co-major: the u phases of a
// channel are adjacent columns, so an epilogue lane holds u consecutive output steps of it):
//   W'[co*u+p][ci][0] = w[ci][co][p+u] (x[s-1]),   W'[co*u+p][ci][1] = w[ci][co][p] (x[s])
void convT_tc_pack(const float* w, int Cin, int Cr, int u, const ConvTcPlan& pl, __half* blob) {
    std::vector<float> tmp((size_t)u * Cr * Cin * 2);
    for (int p = 0; p < u; ++p)
        for (int co = 0; co < Cr; ++co)
            for (int ci = 0; ci < Cin; ++ci) {
                const size_t o = (((size_t)co * u + p) * Cin + ci) * 2;
                tmp[o + 0] = w[((size_t)ci * Cr + co) * (2 * u) + p + u];
                tmp[o + 1] = w[((size_t)ci * Cr + co) * (2 * u) + p];
            }
    conv1d_tc_pack(tmp.data(), Cin, u * Cr, 2, pl, blob);
}

void launch_atoms_zero_pads(__half* buf, int planes_total, int lpad, int L, cudaStream_t st, int batch, const int* item_len) {
    if (planes_total <= 0) return;
    if (batch < 1 || batch > kVocMaxItems || planes_total % batch != 0) throw CudaError("atoms_zero_pads: bad batch");
    ZeroPadLens Z{};
    Z.planes_per_item = planes_total / batch;
    for (int i = 0; i < batch; ++i) Z.len[i] = item_len ? item_len[i] : L;
    ProfScope ps(KF_MISC, st, 0, 16.0 * planes_total * (lpad - L));
    atoms_zero_pads_kernel<<<dim3(2, planes_total), 256, 0, st>>>(reinterpret_cast<uint4*>(buf), planes_total, lpad, Z);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
