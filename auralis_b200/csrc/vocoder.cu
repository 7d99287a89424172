// HiFi-GAN vocoder kernels, fp32 CUDA-core version (channel-major activations [C][L]).
//
// Reference call sites (SURVEY.md §2.4 K13-K17):
//   hifigan_decoder.py:787-800  two F.interpolate(linear, align_corners=False)        -> interp_kernel
//   hifigan_decoder.py:243-245  conv_pre (k7) + cond_layer(g)                          -> conv1d_kernel<7>
//   hifigan_decoder.py:246-251  leaky_relu(0.1) -> ConvTranspose1d -> + conds[i](g)    -> conv_transpose1d_kernel
//   hifigan_decoder.py:76-91    ResBlock1: lrelu -> conv(k,d) -> lrelu -> conv(k,1) -> +x  -> conv1d_kernel<3|7|11>
//   hifigan_decoder.py:253-256  MRF sum / num_kernels                                  -> CONV_ACCUM + in_scale=1/3
//   hifigan_decoder.py:257-259  leaky_relu(0.01) -> conv_post (k7, no bias) -> tanh    -> conv_post_kernel
//
// Dense conv C->C with kernel k is a GEMM with K-dim = C*k; here it is register-tiled on the FP32 pipe:
// a CTA computes 64 (or 32) output channels x 128 time steps, staging 8 input channels (+halo) and
// the matching [8][k][64] weight slab in shared memory per iteration.
#include <algorithm>

#include "kernels.h"

namespace xtts {
namespace {

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

// ------------------------------------------------------------------------------------------------
// fused double (triple, with a speaking rate) linear interpolation + transpose:  latents [T][C]  ->  z [C][Tz]
// ------------------------------------------------------------------------------------------------
// The roundings of this stage are spelled out with intrinsics (no contraction left to the compiler): every level rounds
// l0 * x0 + l1 * x1 as ATen's CPU kernel does, so z equals the chained F.interpolate calls bit for bit, with or without a
// speaking rate (tests/test_gpu_vocoder_f32.py), whatever code surrounds it.
__device__ __forceinline__ void lin_src(int dst, float rscale, int in_len, int& i0, int& i1, float& l0, float& l1) {
    float src = __fmaf_rn(rscale, (float)dst + 0.5f, -0.5f);
    if (src < 0.f) src = 0.f;
    i0 = (int)src;
    if (i0 > in_len - 1) i0 = in_len - 1;
    i1 = i0 + ((i0 < in_len - 1) ? 1 : 0);
    l1 = src - (float)i0;
    l0 = 1.0f - l1;
}

// l0 * x0 + l1 * x1 rounded as ATen's CPU kernel does, fma(l0, x0, l1 * x1)
__device__ __forceinline__ float lerp_aten(float l0, float x0, float l1, float x1) { return __fmaf_rn(l0, x0, __fmul_rn(l1, x1)); }
// speed stage, channel c: frame b of the time-scaled latents, then frame a of the first chunk-level interpolation on them
__device__ __forceinline__ float speed_frame(const float* __restrict__ lat, int b, float r0, int T, int C, int c) {
    int i0, i1; float l0, l1;
    lin_src(b, r0, T, i0, i1, l0, l1);
    return lerp_aten(l0, lat[(size_t)i0 * C + c], l1, lat[(size_t)i1 * C + c]);
}
__device__ __forceinline__ float speed_level1(const float* __restrict__ lat, int a, float r1, int T0, float r0, int T, int C, int c) {
    int b0, b1; float n0, n1;
    lin_src(a, r1, T0, b0, b1, n0, n1);
    return lerp_aten(n0, speed_frame(lat, b0, r0, T, C, c), n1, speed_frame(lat, b1, r0, T, C, c));
}

struct PostLens { int len[kVocMaxItems]; };
struct InterpBatch { InterpItem it[kVocMaxItems]; };

// Block (x: 32 z-frames, y: 32 channels, z: batch item).  Output column j of item i is the chunk's z-frame it.z0 + j:
// a window of a chunk gets the very values the whole chunk would (the source positions depend on the global index only).
__global__ void __launch_bounds__(256)
interp_kernel(const InterpBatch B, float* __restrict__ z_, uint4* __restrict__ z16_, int lpad, int C, int Lz, float r1, float r2) {
    __shared__ float tile[32][33];
    const InterpItem it = B.it[blockIdx.z];
    const float* __restrict__ lat = it.lat;
    const int T = it.T, T1 = it.T1, nz = it.nz;
    const int c0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
    if (j0 >= nz) return;
    const int tx = threadIdx.x, ty = threadIdx.y;       // (32, 8)
    for (int k = 0; k < 4; ++k) {
        const int j = j0 + ty + 8 * k, c = c0 + tx;
        float v = 0.f;
        if (j < nz && c < C) {
            int a0, a1; float m0, m1;
            lin_src(it.z0 + j, r2, T1, a0, a1, m0, m1);
            if (it.r0 > 0.f) {                          // three levels: up to 8 latent rows per value (L1 / L2 hits)
                const float za = speed_level1(lat, a0, r1, it.T0, it.r0, T, C, c);
                const float zb = speed_level1(lat, a1, r1, it.T0, it.r0, T, C, c);
                v = lerp_aten(m0, za, m1, zb);
            } else {                                    // two levels, the latents read directly
                int b0, b1; float n0, n1;
                lin_src(a0, r1, T, b0, b1, n0, n1);
                const float za = lerp_aten(n0, lat[(size_t)b0 * C + c], n1, lat[(size_t)b1 * C + c]);
                lin_src(a1, r1, T, b0, b1, n0, n1);
                const float zb = lerp_aten(n0, lat[(size_t)b0 * C + c], n1, lat[(size_t)b1 * C + c]);
                v = lerp_aten(m0, za, m1, zb);
            }
        }
        tile[ty + 8 * k][tx] = v;                       // tile[j][c]
    }
    __syncthreads();
    if (z_) {
        float* z = z_ + (size_t)blockIdx.z * C * Lz;
        for (int k = 0; k < 4; ++k) {
            const int c = c0 + ty + 8 * k, j = j0 + tx;
            if (c < C && j < nz) z[(size_t)c * Lz + j] = tile[tx][ty + 8 * k];
        }
    }
    if (z16_ && ty < 4) {                               // 32 time steps x 4 atoms of 8 channels
        const int j = j0 + tx, cg = c0 / 8 + ty;
        if (j < nz && c0 + ty * 8 < C) {
            const float* r = &tile[tx][ty * 8];
            __half2 h0 = __floats2half2_rn(r[0], r[1]), h1 = __floats2half2_rn(r[2], r[3]);
            __half2 h2 = __floats2half2_rn(r[4], r[5]), h3 = __floats2half2_rn(r[6], r[7]);
            uint4 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
            pk.z = *reinterpret_cast<uint32_t*>(&h2); pk.w = *reinterpret_cast<uint32_t*>(&h3);
            z16_[((size_t)blockIdx.z * (C / 8) + cg) * lpad + kAtomPadL + j] = pk;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// dilated Conv1d, "same" padding, fused input scale + leaky-relu, bias, speaker bias, residual, store/accumulate
// ------------------------------------------------------------------------------------------------
constexpr int CT_T = 128;      // time steps per CTA (4 per thread, stride 32)
constexpr int CT_CI = 8;       // input channels staged per iteration
constexpr int CT_TC = 8;       // output channels per thread

template <int K, int NTY>
__global__ void __launch_bounds__(32 * NTY)
conv1d_kernel(const float* __restrict__ x_, const float* __restrict__ w_t, const float* __restrict__ bias,
              const float* __restrict__ cbias_, const float* resid_, float* out_, int Cin, int Cout, int L, int dil,
              float in_scale, float slope, int mode, int cbias_bs) {
    constexpr int CO_T = CT_TC * NTY;
    const float* x = x_ + (size_t)blockIdx.z * Cin * L;
    float* out = out_ + (size_t)blockIdx.z * Cout * L;
    const float* resid = resid_ ? resid_ + (size_t)blockIdx.z * Cout * L : nullptr;
    const float* cbias = cbias_ ? cbias_ + (size_t)blockIdx.z * cbias_bs : nullptr;
    extern __shared__ __align__(16) float smem[];
    const int halo = (K - 1) / 2 * dil;
    const int XW = CT_T + 2 * halo;
    float* xs = smem;                              // [CT_CI][XW]
    float* ws = smem + CT_CI * XW + ((4 - (CT_CI * XW) % 4) % 4);   // [CT_CI][K][CO_T], 16-byte aligned
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int tid = ty * 32 + tx;
    const int nthr = 32 * NTY;
    const int t0 = blockIdx.x * CT_T, co0 = blockIdx.y * CO_T;

    float acc[CT_TC][4];
#pragma unroll
    for (int c = 0; c < CT_TC; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[c][i] = 0.f;

    for (int ci0 = 0; ci0 < Cin; ci0 += CT_CI) {
        __syncthreads();
        for (int e = tid; e < CT_CI * XW; e += nthr) {
            const int ci = e / XW, p = e - ci * XW;
            const int gt = t0 - halo + p;
            float v = 0.f;
            if (gt >= 0 && gt < L && ci0 + ci < Cin) v = lrelu(in_scale * x[(size_t)(ci0 + ci) * L + gt], slope);
            xs[e] = v;
        }
        for (int e = tid; e < CT_CI * K * CO_T; e += nthr) {
            const int ci = e / (K * CO_T);
            const int r = e - ci * (K * CO_T);
            const int j = r / CO_T, co = r - j * CO_T;
            float v = 0.f;
            if (ci0 + ci < Cin && co0 + co < Cout) v = w_t[((size_t)(ci0 + ci) * K + j) * Cout + co0 + co];
            ws[e] = v;
        }
        __syncthreads();
#pragma unroll 2
        for (int ci = 0; ci < CT_CI; ++ci) {
            const float* xr = xs + ci * XW + tx;
            const float* wr = ws + (ci * K) * CO_T + ty * CT_TC;
#pragma unroll
            for (int j = 0; j < K; ++j) {
                float xv[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) xv[i] = xr[32 * i + j * dil];
                const float4 wa = *reinterpret_cast<const float4*>(wr + j * CO_T);
                const float4 wb = *reinterpret_cast<const float4*>(wr + j * CO_T + 4);
                const float wv[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
                for (int c = 0; c < CT_TC; ++c)
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[c][i] = fmaf(wv[c], xv[i], acc[c][i]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CT_TC; ++c) {
        const int co = co0 + ty * CT_TC + c;
        if (co >= Cout) continue;
        const float b = (bias ? bias[co] : 0.f) + (cbias ? cbias[co] : 0.f);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int t = t0 + tx + 32 * i;
            if (t >= L) continue;
            const size_t o = (size_t)co * L + t;
            float v = acc[c][i] + b;
            if (resid) v += resid[o];
            if (mode == CONV_ACCUM) v += out[o];
            out[o] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// ConvTranspose1d with K == 2*stride, padding = stride/2: every output sample has exactly two taps.
//   out[co][t] = b + sum_ci act(x[ci][s0]) w[ci][j0][co] + act(x[ci][s0-1]) w[ci][j0+u][co],
//   q = t + u/2, j0 = q % u, s0 = q / u
// ------------------------------------------------------------------------------------------------
constexpr int UP_T = 128, UP_CI = 8, UP_CO = 16;

__global__ void __launch_bounds__(UP_T)
conv_transpose1d_kernel(const float* __restrict__ x_, const float* __restrict__ w_t, const float* __restrict__ bias,
                        const float* __restrict__ cbias_, float* __restrict__ out_, int Cin, int Cout, int Lin, int K, int u,
                        float in_scale, float slope, int cbias_bs) {
    extern __shared__ __align__(16) float smem[];
    const float* x = x_ + (size_t)blockIdx.z * Cin * Lin;
    float* out = out_ + (size_t)blockIdx.z * Cout * Lin * u;
    const float* cbias = cbias_ ? cbias_ + (size_t)blockIdx.z * cbias_bs : nullptr;
    const int pad = (K - u) / 2;
    const int XS = UP_T / u + 3;                   // source frames touched by the tile (+ slack)
    constexpr int WROW = UP_CO + 4;
    float* xs = smem;                              // [UP_CI][XS]
    float* ws = smem + ((UP_CI * XS + 3) / 4) * 4; // [UP_CI][K][WROW]
    const int tid = threadIdx.x;
    const int t0 = blockIdx.x * UP_T, co0 = blockIdx.y * UP_CO;
    const int Lout = Lin * u;
    const int s_base = (t0 + pad) / u - 1;         // first source frame the tile may touch
    const int t = t0 + tid;
    const int q = t + pad;
    const int j0 = q % u, s0 = q / u;
    float acc[UP_CO];
#pragma unroll
    for (int c = 0; c < UP_CO; ++c) acc[c] = 0.f;
    for (int ci0 = 0; ci0 < Cin; ci0 += UP_CI) {
        __syncthreads();
        for (int e = tid; e < UP_CI * XS; e += UP_T) {
            const int ci = e / XS, p = e - ci * XS;
            const int s = s_base + p;
            float v = 0.f;
            if (s >= 0 && s < Lin && ci0 + ci < Cin) v = lrelu(in_scale * x[(size_t)(ci0 + ci) * Lin + s], slope);
            xs[e] = v;
        }
        for (int e = tid; e < UP_CI * K * UP_CO; e += UP_T) {
            const int ci = e / (K * UP_CO);
            const int r = e - ci * (K * UP_CO);
            const int j = r / UP_CO, co = r - j * UP_CO;
            float v = 0.f;
            if (ci0 + ci < Cin && co0 + co < Cout) v = w_t[((size_t)(ci0 + ci) * K + j) * Cout + co0 + co];
            ws[(ci * K + j) * WROW + co] = v;
        }
        __syncthreads();
#pragma unroll
        for (int ci = 0; ci < UP_CI; ++ci) {
            const float xa = xs[ci * XS + (s0 - s_base)];
            const float xb = xs[ci * XS + (s0 - 1 - s_base)];
            const float* wa = ws + (ci * K + j0) * WROW;
            const float* wb = ws + (ci * K + j0 + u) * WROW;
#pragma unroll
            for (int c4 = 0; c4 < UP_CO / 4; ++c4) {
                const float4 a = *reinterpret_cast<const float4*>(wa + 4 * c4);
                const float4 b = *reinterpret_cast<const float4*>(wb + 4 * c4);
                acc[4 * c4 + 0] = fmaf(xa, a.x, fmaf(xb, b.x, acc[4 * c4 + 0]));
                acc[4 * c4 + 1] = fmaf(xa, a.y, fmaf(xb, b.y, acc[4 * c4 + 1]));
                acc[4 * c4 + 2] = fmaf(xa, a.z, fmaf(xb, b.z, acc[4 * c4 + 2]));
                acc[4 * c4 + 3] = fmaf(xa, a.w, fmaf(xb, b.w, acc[4 * c4 + 3]));
            }
        }
    }
    if (t < Lout) {
#pragma unroll
        for (int c = 0; c < UP_CO; ++c) {
            const int co = co0 + c;
            if (co < Cout) {
                acc[c] += (bias ? bias[co] : 0.f) + (cbias ? cbias[co] : 0.f);
                out[(size_t)co * Lout + t] = acc[c];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// conv_post (C->1, k7, no bias) + tanh; HBM-bound (reads C*L floats, writes L)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv_post_kernel(const float* __restrict__ x_, const float* __restrict__ w, float* __restrict__ wav_, int Cin, int Ls,
                 int wav_stride, int K, float in_scale, float slope, const PostLens PL) {
    extern __shared__ float wsm[];                 // [Cin*K]
    const int L = PL.len[blockIdx.y];              // this item's signal length; rows are strided by Ls
    if ((int)(blockIdx.x * blockDim.x) >= L) return;
    const float* x = x_ + (size_t)blockIdx.y * Cin * Ls;
    float* wav = wav_ + (size_t)blockIdx.y * wav_stride;
    for (int e = threadIdx.x; e < Cin * K; e += blockDim.x) wsm[e] = w[e];
    __syncthreads();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= L) return;
    const int half = (K - 1) / 2;
    float acc = 0.f;
    for (int ci = 0; ci < Cin; ++ci) {
        const float* xr = x + (size_t)ci * Ls;
        for (int j = 0; j < K; ++j) {
            const int s = t + j - half;
            if (s >= 0 && s < L) acc = fmaf(wsm[ci * K + j], lrelu(in_scale * xr[s], slope), acc);
        }
    }
    wav[t] = tanhf(acc);
}

template <int K>
void conv1d_dispatch(const float* x, const float* w_t, const float* bias, const float* cbias, const float* resid,
                     float* out, int Cin, int Cout, int L, int dil, float in_scale, float slope, int mode, int batch,
                     int cbias_bs, cudaStream_t st) {
    const int halo = (K - 1) / 2 * dil;
    const int XW = CT_T + 2 * halo;
    const int xs_f = CT_CI * XW + ((4 - (CT_CI * XW) % 4) % 4);
    // algorithmic traffic: read x once, write out once (+ residual / accumulate reads), weights once
    ProfScope ps(KF_CONV1D, st, 2.0 * Cin * Cout * K * (double)L * batch,
                 4.0 * (batch * (double)L * (Cin + Cout * (1 + (resid ? 1 : 0) + (mode == CONV_ACCUM ? 1 : 0))) + (double)Cin * Cout * K));
    if (Cout > 32) {
        constexpr int NTY = 8;
        const size_t smem = (size_t)(xs_f + CT_CI * K * CT_TC * NTY) * sizeof(float);
        dim3 grid(ceil_div(L, CT_T), ceil_div(Cout, CT_TC * NTY), batch);
        conv1d_kernel<K, NTY><<<grid, dim3(32, NTY), smem, st>>>(x, w_t, bias, cbias, resid, out, Cin, Cout, L, dil,
                                                                 in_scale, slope, mode, cbias_bs);
    } else {
        constexpr int NTY = 4;
        const size_t smem = (size_t)(xs_f + CT_CI * K * CT_TC * NTY) * sizeof(float);
        dim3 grid(ceil_div(L, CT_T), ceil_div(Cout, CT_TC * NTY), batch);
        conv1d_kernel<K, NTY><<<grid, dim3(32, NTY), smem, st>>>(x, w_t, bias, cbias, resid, out, Cin, Cout, L, dil,
                                                                 in_scale, slope, mode, cbias_bs);
    }
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace

void conv_weight_ckc(const float* w, int Cin, int Cout, int K, bool transposed, float* w_t) {
    for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
            for (int j = 0; j < K; ++j)
                w_t[((size_t)ci * K + j) * Cout + co] = transposed ? w[((size_t)ci * Cout + co) * K + j] : w[((size_t)co * Cin + ci) * K + j];
}

void launch_interp(const InterpItem* items, int batch, float* z32, __half* z16, int lpad, int C, int Lz, double scale1,
                   double scale2, cudaStream_t st) {
    if (batch < 1 || batch > kVocMaxItems) throw CudaError("interp: batch out of range");
    const float r1 = (float)(1.0 / scale1), r2 = (float)(1.0 / scale2);
    InterpBatch B{};
    int nz_max = 0; double nz_sum = 0;
    for (int i = 0; i < batch; ++i) {
        B.it[i] = items[i];
        if (items[i].nz > Lz) throw CudaError("interp: window longer than the row stride");
        nz_max = std::max(nz_max, items[i].nz); nz_sum += items[i].nz;
    }
    if (nz_max <= 0) return;
    ProfScope ps(KF_INTERP, st, 0, C * nz_sum * (4.0 / (scale1 * scale2) + (z32 ? 4.0 : 0.0) + (z16 ? 2.0 : 0.0)));
    interp_kernel<<<dim3(ceil_div(nz_max, 32), ceil_div(C, 32), batch), dim3(32, 8), 0, st>>>(
        B, z32, reinterpret_cast<uint4*>(z16), lpad, C, Lz, r1, r2);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_conv1d(const float* x, const float* w_t, const float* bias, const float* cbias, const float* resid,
                   float* out, int Cin, int Cout, int L, int K, int dil, float in_scale, float slope, int mode,
                   int batch, int cbias_bs, cudaStream_t st) {
    if (L <= 0 || batch <= 0) return;
    switch (K) {
        case 3: conv1d_dispatch<3>(x, w_t, bias, cbias, resid, out, Cin, Cout, L, dil, in_scale, slope, mode, batch, cbias_bs, st); break;
        case 7: conv1d_dispatch<7>(x, w_t, bias, cbias, resid, out, Cin, Cout, L, dil, in_scale, slope, mode, batch, cbias_bs, st); break;
        case 11: conv1d_dispatch<11>(x, w_t, bias, cbias, resid, out, Cin, Cout, L, dil, in_scale, slope, mode, batch, cbias_bs, st); break;
        default: throw CudaError("conv1d: unsupported kernel size (3, 7, 11 only)");
    }
}

void launch_conv_transpose1d(const float* x, const float* w_t, const float* bias, const float* cbias, float* out, int Cin,
                             int Cout, int Lin, int K, int u, float in_scale, float slope, int batch, int cbias_bs,
                             cudaStream_t st) {
    if (K != 2 * u || (u & 1)) throw CudaError("conv_transpose1d: only kernel == 2*stride with even stride is supported");
    if (UP_T % u != 0) throw CudaError("conv_transpose1d: stride must divide 128");
    const int XS = UP_T / u + 3;
    const size_t smem = (size_t)(((UP_CI * XS + 3) / 4) * 4 + UP_CI * K * (UP_CO + 4)) * sizeof(float);
    dim3 grid(ceil_div(Lin * u, UP_T), ceil_div(Cout, UP_CO), batch);
    ProfScope ps(KF_CONVT, st, 4.0 * Cin * Cout * (double)Lin * u * batch, 4.0 * (batch * ((double)Lin * Cin + (double)Lin * u * Cout) + (double)Cin * Cout * K));
    conv_transpose1d_kernel<<<grid, UP_T, smem, st>>>(x, w_t, bias, cbias, out, Cin, Cout, Lin, K, u, in_scale, slope, cbias_bs);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_conv_post(const float* x, const float* w, float* wav, int Cin, int L, int K, float in_scale, float slope,
                      int batch, cudaStream_t st, const int* item_len, int wav_stride) {
    if (batch < 1 || batch > kVocMaxItems) throw CudaError("conv_post: batch out of range");
    if (wav_stride <= 0) wav_stride = L;
    PostLens PL{};
    double Lsum = 0;
    for (int i = 0; i < batch; ++i) { PL.len[i] = item_len ? item_len[i] : L; Lsum += PL.len[i]; }
    ProfScope ps(KF_CONV_POST, st, 2.0 * Cin * K * Lsum, 4.0 * Lsum * (Cin + 1));
    conv_post_kernel<<<dim3(ceil_div(L, 256), batch), 256, Cin * K * sizeof(float), st>>>(x, w, wav, Cin, L, wav_stride, K, in_scale, slope, PL);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
