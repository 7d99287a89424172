// Speaker-conditioning kernels and driver (see cond.h).  Activations are time-major rows [T, C] so every
// 1x1 convolution / nn.Linear is one call of the shared NT GEMM; the STFTs are DFT-by-GEMM against
// precomputed (cos | -sin) bases restricted to the window support (n_fft 2048 -> 1024 live taps).
// Per-speaker, cached by the engine: clarity over peak speed, fp32 throughout.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>

#include "cond.h"

namespace xtts {
namespace {

// mode 0: log(clamp(x,1e-5)) / stats[c]   (utilities.py:66-70);  mode 1: log(x + 1e-6)   (hifigan_decoder.py:616)
__global__ void mel_log_kernel(float* __restrict__ M, const float* __restrict__ stats, size_t n, int C, int mode) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = M[i];
    M[i] = mode == 0 ? logf(fmaxf(v, 1e-5f)) / stats[i % C] : logf(v + 1e-6f);
}
__global__ void preemphasis_kernel(const float* __restrict__ x, float* __restrict__ y, int n, float coef) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float prev = (i == 0) ? x[min(1, n - 1)] : x[i - 1];      // reflect pad (1,0)
    y[i] = x[i] - coef * prev;
}
// InstanceNorm1d over time per mel channel; in [T][C] -> out [C][T]
__global__ void instnorm_transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int C, float eps) {
    __shared__ float red[32];
    const int c = blockIdx.x;
    float s = 0.f;
    for (int t = threadIdx.x; t < T; t += blockDim.x) s += in[(size_t)t * C + c];
    const float mean = block_sum(s, red) / (float)T;
    float v = 0.f;
    for (int t = threadIdx.x; t < T; t += blockDim.x) { const float d = in[(size_t)t * C + c] - mean; v = fmaf(d, d, v); }
    const float rstd = 1.0f / sqrtf(block_sum(v, red) / (float)T + eps);
    for (int t = threadIdx.x; t < T; t += blockDim.x) out[(size_t)c * T + t] = (in[(size_t)t * C + c] - mean) * rstd;
}

// ---------------------------------------------------------------------------------------- encoder pieces
// GroupNorm over rows [T][C]; one CTA per group (latent_encoder.py:10-24,53-72)
__global__ void groupnorm_rows_kernel(const float* __restrict__ X, const float* __restrict__ w, const float* __restrict__ b,
                                      float* __restrict__ Y, int T, int C, int groups, float eps) {
    __shared__ float red[32];
    const int g = blockIdx.x, cpg = C / groups, c0 = g * cpg;
    const int n = T * cpg;
    float s = 0.f;
    for (int e = threadIdx.x; e < n; e += blockDim.x) s += X[(size_t)(e / cpg) * C + c0 + e % cpg];
    const float mean = block_sum(s, red) / (float)n;
    float v = 0.f;
    for (int e = threadIdx.x; e < n; e += blockDim.x) { const float d = X[(size_t)(e / cpg) * C + c0 + e % cpg] - mean; v = fmaf(d, d, v); }
    const float rstd = 1.0f / sqrtf(block_sum(v, red) / (float)n + eps);
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int c = c0 + e % cpg;
        const size_t i = (size_t)(e / cpg) * C + c;
        Y[i] = (X[i] - mean) * rstd * w[c] + b[c];
    }
}
// GEGLU (perceiver_encoder.py:322-336): out[r][j] = gelu_erf(h[r][F+j]) * h[r][j]
__global__ void geglu_kernel(const float* __restrict__ Hc, float* __restrict__ out, int rows, int F) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * F) return;
    const int r = (int)(i / F), j = (int)(i % F);
    const float x = Hc[(size_t)r * 2 * F + j], gate = Hc[(size_t)r * 2 * F + F + j];
    out[i] = 0.5f * gate * (1.0f + erff(gate * 0.70710678118654752f)) * x;
}
// RMSNorm (perceiver_encoder.py:262-276): normalize(x) * sqrt(C) * gamma ; then acc += y * scale
__global__ void rmsnorm_accum_kernel(const float* __restrict__ X, const float* __restrict__ gamma, float* __restrict__ acc,
                                     int C, float scale) {
    __shared__ float red[32];
    const float* x = X + (size_t)blockIdx.x * C;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s = fmaf(x[c], x[c], s);
    const float nrm = fmaxf(sqrtf(block_sum(s, red)), 1e-12f);
    const float k = sqrtf((float)C) / nrm;
    for (int c = threadIdx.x; c < C; c += blockDim.x) acc[(size_t)blockIdx.x * C + c] += x[c] * k * gamma[c] * scale;
}

// ---------------------------------------------------------------------------------------- speaker ResNet
// direct conv2d (k x k, stride s, pad k/2), NCHW with N=1; optional bias, relu-then-BN or BN epilogue
// (SEBasicBlock order: conv1 -> relu -> bn1 -> conv2 -> bn2, hifigan_decoder.py:414-424)
constexpr int C2_CO = 4;     // 4 x 256 x 9 floats of weights = 36 KB of shared memory at the widest layer
__global__ void __launch_bounds__(128)
conv2d_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
              const float* __restrict__ bn_scale, const float* __restrict__ bn_shift, float* __restrict__ out, int Cin,
              int Cout, int Hin, int Win, int Hout, int Wout, int k, int stride, int relu_before_bn) {
    extern __shared__ float wsm[];                     // [C2_CO][Cin][k*k]
    const int co0 = blockIdx.z * C2_CO, y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    const int kk = k * k, pad = k / 2;
    for (int e = threadIdx.x; e < C2_CO * Cin * kk; e += blockDim.x) {
        const int c = e / (Cin * kk);
        wsm[e] = (co0 + c < Cout) ? w[(size_t)(co0 + c) * Cin * kk + e % (Cin * kk)] : 0.f;
    }
    __syncthreads();
    if (x >= Wout) return;
    float acc[C2_CO];
#pragma unroll
    for (int c = 0; c < C2_CO; ++c) acc[c] = 0.f;
    for (int ci = 0; ci < Cin; ++ci) {
        for (int ky = 0; ky < k; ++ky) {
            const int iy = y * stride + ky - pad;
            if (iy < 0 || iy >= Hin) continue;
            for (int kx = 0; kx < k; ++kx) {
                const int ix = x * stride + kx - pad;
                if (ix < 0 || ix >= Win) continue;
                const float v = in[((size_t)ci * Hin + iy) * Win + ix];
#pragma unroll
                for (int c = 0; c < C2_CO; ++c) acc[c] = fmaf(v, wsm[(c * Cin + ci) * kk + ky * k + kx], acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < C2_CO; ++c) {
        const int co = co0 + c;
        if (co >= Cout) continue;
        float v = acc[c] + (bias ? bias[co] : 0.f);
        if (relu_before_bn) v = fmaxf(v, 0.f);
        if (bn_scale) v = v * bn_scale[co] + bn_shift[co];
        out[((size_t)co * Hout + y) * Wout + x] = v;
    }
}
__global__ void channel_mean_kernel(const float* __restrict__ x, float* __restrict__ m, int HW) {
    __shared__ float red[32];
    const float* p = x + (size_t)blockIdx.x * HW;
    float s = 0.f;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) s += p[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) m[blockIdx.x] = s / (float)HW;
}
// SE gate (hifigan_decoder.py:353-376): s = sigmoid(W2 relu(W1 m + b1) + b2); single CTA
__global__ void se_gate_kernel(const float* __restrict__ m, const float* __restrict__ w1, const float* __restrict__ b1,
                               const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ gate, int C, int R) {
    extern __shared__ float hid[];
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        float s = b1[r];
        for (int c = 0; c < C; ++c) s = fmaf(w1[(size_t)r * C + c], m[c], s);
        hid[r] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = b2[c];
        for (int r = 0; r < R; ++r) s = fmaf(w2[(size_t)c * R + r], hid[r], s);
        gate[c] = 1.0f / (1.0f + expf(-s));
    }
}
// out = relu(x * gate[c] + resid)
__global__ void se_apply_kernel(const float* __restrict__ x, const float* __restrict__ gate, const float* __restrict__ resid,
                                float* __restrict__ out, int HW, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = fmaxf(fmaf(x[i], gate[i / HW], resid[i]), 0.f);
}
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cc) {   // [R][Cc] -> [Cc][R]
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)R * Cc) return;
    const int r = (int)(i / Cc), c = (int)(i % Cc);
    out[(size_t)c * R + r] = in[i];
}
// rows [T][C]: y = bn(relu(x))  (attention.1-2, hifigan_decoder.py:573-577)
__global__ void relu_bn_rows_kernel(float* __restrict__ X, const float* __restrict__ sc, const float* __restrict__ sh, size_t n, int C) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = (int)(i % C);
    X[i] = fmaxf(X[i], 0.f) * sc[c] + sh[c];
}
// attentive statistics pooling over time for channel c (hifigan_decoder.py:632-640): logits A [T][C], feats X [C][T]
__global__ void asp_kernel(const float* __restrict__ A, const float* __restrict__ X, float* __restrict__ out, int T, int C) {
    __shared__ float red[32];
    const int c = blockIdx.x;
    float mx = -INFINITY;
    for (int t = threadIdx.x; t < T; t += blockDim.x) mx = fmaxf(mx, A[(size_t)t * C + c]);
    mx = block_max(mx, red);
    float se = 0.f, s1 = 0.f, s2 = 0.f;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float e = expf(A[(size_t)t * C + c] - mx), x = X[(size_t)c * T + t];
        se += e; s1 = fmaf(e, x, s1); s2 = fmaf(e, x * x, s2);
    }
    se = block_sum(se, red); s1 = block_sum(s1, red); s2 = block_sum(s2, red);
    if (threadIdx.x == 0) {
        const float mu = s1 / se;
        out[c] = mu;
        out[C + c] = sqrtf(fmaxf(s2 / se - mu * mu, 1e-5f));
    }
}
__global__ void l2norm_kernel(float* __restrict__ x, int n) {
    __shared__ float red[32];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s = fmaf(x[i], x[i], s);
    const float nrm = fmaxf(sqrtf(block_sum(s, red)), 1e-12f);
    for (int i = threadIdx.x; i < n; i += blockDim.x) x[i] /= nrm;
}

}  // namespace

// ---------------------------------------------------------------------------------------- STFT front-end (cond.h)
// F[t][i] = win[i] * xp[t*hop + off + i].  PAD_REFLECT: xp = reflect-pad(x, pad) (torch.stft center=True);
// PAD_ZERO: xp = zero-pad(nan_to_num(x), pad) (librosa.stft center=True after np.nan_to_num)
__global__ void frame_window_kernel(const float* __restrict__ x, int n, const float* __restrict__ win, int wlen, int hop,
                                    int off, int pad, int pad_mode, float* __restrict__ F, int frames) {
    const int t = blockIdx.x;
    for (int i = threadIdx.x; i < wlen; i += blockDim.x) {
        int p = t * hop + off + i - pad;
        float v;
        if (pad_mode == PAD_ZERO) {
            v = (p < 0 || p >= n) ? 0.f : x[p];
            if (!isfinite(v)) v = 0.f;
        } else {
            if (p < 0) p = -p;
            if (p >= n) p = 2 * (n - 1) - p;
            p = max(0, min(n - 1, p));
            v = x[p];
        }
        F[(size_t)t * wlen + i] = win[i] * v;
    }
}
// P[t][k] = re^2 + im^2 from D [frames, 2*nb]
__global__ void power_kernel(const float* __restrict__ D, float* __restrict__ P, int frames, int nb) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)frames * nb) return;
    const int t = (int)(i / nb), k = (int)(i % nb);
    const float re = D[(size_t)t * 2 * nb + k], im = D[(size_t)t * 2 * nb + nb + k];
    P[i] = re * re + im * im;
}

// ---------------------------------------------------------------------------------------- launches
// One helper per kernel, called by Conditioner::run and by cond_debug (xtts_debug_cond), so a kernel under test runs with
// the production grid, block size and shared memory.
namespace {

int conv_out(int n, int k, int stride) { return (n + 2 * (k / 2) - k) / stride + 1; }
size_t conv2d_smem(int Cin, int k) { return (size_t)C2_CO * Cin * k * k * sizeof(float); }
constexpr size_t kSmemLimit = 48 * 1024;           // dynamic shared memory without an opt-in attribute

// block size: 256 threads for the 22.05 kHz front-end (wlen 1024), 128 for the 16 kHz one (wlen 400)
void launch_frame_window(const float* x, int n, const float* win, int wlen, int hop, int off, int pad, int pad_mode, float* F,
                         int frames, int threads, cudaStream_t st) {
    frame_window_kernel<<<frames, threads, 0, st>>>(x, n, win, wlen, hop, off, pad, pad_mode, F, frames);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_power(const float* D, float* P, int frames, int nb, cudaStream_t st) {
    power_kernel<<<nblk((size_t)frames * nb), 256, 0, st>>>(D, P, frames, nb); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_mel_log(float* M, const float* stats, size_t n, int C, int mode, cudaStream_t st) {
    mel_log_kernel<<<nblk(n), 256, 0, st>>>(M, stats, n, C, mode); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_preemphasis(const float* x, float* y, int n, float coef, cudaStream_t st) {
    preemphasis_kernel<<<nblk(n), 256, 0, st>>>(x, y, n, coef); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_instnorm_t(const float* in, float* out, int T, int C, float eps, cudaStream_t st) {
    instnorm_transpose_kernel<<<C, 256, 0, st>>>(in, out, T, C, eps); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_groupnorm(const float* X, const float* w, const float* b, float* Y, int T, int C, int groups, float eps, cudaStream_t st) {
    groupnorm_rows_kernel<<<groups, 256, 0, st>>>(X, w, b, Y, T, C, groups, eps); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_geglu(const float* Hc, float* out, int rows, int F, cudaStream_t st) {
    geglu_kernel<<<nblk((size_t)rows * F), 256, 0, st>>>(Hc, out, rows, F); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_rmsnorm_accum(const float* X, const float* gamma, float* acc, int rows, int C, float scale, cudaStream_t st) {
    rmsnorm_accum_kernel<<<rows, 256, 0, st>>>(X, gamma, acc, C, scale); COUNT_LAUNCH(); KERNEL_CHECK();
}
// out [Cout][Hout][Wout] must fit in `cap` floats; throws before the launch otherwise, or when the weight slice of C2_CO
// output channels exceeds 48 KB of shared memory
void launch_conv2d(const float* in, const float* w, const float* bias, const float* bn_scale, const float* bn_shift, float* out,
                   size_t cap, int Cin, int Cout, int Hin, int Win, int k, int stride, int relu_before_bn, int& Hout, int& Wout,
                   cudaStream_t st) {
    Hout = conv_out(Hin, k, stride); Wout = conv_out(Win, k, stride);
    if ((size_t)Cout * Hout * Wout > cap)
        throw std::runtime_error("conv2d: output [" + std::to_string(Cout) + "][" + std::to_string(Hout) + "][" + std::to_string(Wout) +
                                 "] exceeds its buffer of " + std::to_string(cap) + " floats");
    if (conv2d_smem(Cin, k) > kSmemLimit) throw std::runtime_error("conv2d: weight slice exceeds 48 KB of shared memory");
    dim3 grid(ceil_div(Wout, 128), Hout, ceil_div(Cout, C2_CO));
    conv2d_kernel<<<grid, 128, conv2d_smem(Cin, k), st>>>(in, w, bias, bn_scale, bn_shift, out, Cin, Cout, Hin, Win, Hout, Wout, k,
                                                           stride, relu_before_bn);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_channel_mean(const float* x, float* m, int C, int HW, cudaStream_t st) {
    channel_mean_kernel<<<C, 256, 0, st>>>(x, m, HW); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_se_gate(const float* m, const float* w1, const float* b1, const float* w2, const float* b2, float* gate, int C, int R,
                    cudaStream_t st) {
    se_gate_kernel<<<1, 256, (size_t)R * sizeof(float), st>>>(m, w1, b1, w2, b2, gate, C, R); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_se_apply(const float* x, const float* gate, const float* resid, float* out, int HW, size_t n, cudaStream_t st) {
    se_apply_kernel<<<nblk(n), 256, 0, st>>>(x, gate, resid, out, HW, n); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_transpose(const float* in, float* out, int R, int Cc, cudaStream_t st) {
    transpose_kernel<<<nblk((size_t)R * Cc), 256, 0, st>>>(in, out, R, Cc); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_relu_bn_rows(float* X, const float* sc, const float* sh, size_t n, int C, cudaStream_t st) {
    relu_bn_rows_kernel<<<nblk(n), 256, 0, st>>>(X, sc, sh, n, C); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_asp(const float* A, const float* X, float* out, int T, int C, cudaStream_t st) {
    asp_kernel<<<C, 128, 0, st>>>(A, X, out, T, C); COUNT_LAUNCH(); KERNEL_CHECK();
}
void launch_l2norm(float* x, int n, cudaStream_t st) {
    l2norm_kernel<<<1, 256, 0, st>>>(x, n); COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace

std::vector<float> dft_basis(int n_fft, int wlen, int off) {          // [(2*nb)][wlen]: cos rows then -sin rows
    const int nb = n_fft / 2 + 1;
    std::vector<float> B((size_t)2 * nb * wlen);
    for (int k = 0; k < nb; ++k)
        for (int i = 0; i < wlen; ++i) {
            const double a = 2.0 * kPi * (double)k * (double)((off + i) % n_fft) / (double)n_fft;
            B[(size_t)k * wlen + i] = (float)std::cos(a);
            B[(size_t)(nb + k) * wlen + i] = (float)(-std::sin(a));
        }
    return B;
}
// torchaudio.functional.melscale_fbanks (htk), transposed to [n_mels][n_freqs] for the NT GEMM
std::vector<float> mel_fb_t(int n_freqs, double f_min, double f_max, int n_mels, int sr, bool slaney) {
    std::vector<double> freqs(n_freqs), fpts(n_mels + 2);
    for (int i = 0; i < n_freqs; ++i) freqs[i] = (double)(sr / 2) * i / (n_freqs - 1);
    const double mmin = 2595.0 * std::log10(1.0 + f_min / 700.0), mmax = 2595.0 * std::log10(1.0 + f_max / 700.0);
    for (int i = 0; i < n_mels + 2; ++i) fpts[i] = 700.0 * (std::pow(10.0, (mmin + (mmax - mmin) * i / (n_mels + 1)) / 2595.0) - 1.0);
    std::vector<float> fb((size_t)n_mels * n_freqs);
    for (int m = 0; m < n_mels; ++m) {
        const double lo = fpts[m], ce = fpts[m + 1], hi = fpts[m + 2];
        const double en = slaney ? 2.0 / (hi - lo) : 1.0;
        for (int f = 0; f < n_freqs; ++f) {
            const double down = (freqs[f] - lo) / (ce - lo), up = (hi - freqs[f]) / (hi - ce);
            fb[(size_t)m * n_freqs + f] = (float)(std::max(0.0, std::min(down, up)) * en);
        }
    }
    return fb;
}

namespace {

struct Lin { Dev<float> w, b; int N = 0, K = 0; bool has_b = false; };
struct Bn { Dev<float> scale, shift; };
struct Block { Dev<float> c1, c2, ds; Bn bn1, bn2, bnd; Lin se1, se2; int cin = 0, cout = 0, stride = 1; bool has_ds = false; };

}  // namespace

struct Conditioner::Impl {
    xtts_config c;
    cudaStream_t st;
    int H, NH;
    // front-ends
    Dev<float> hann, basis22, fb22, mel_stats, hamm, basis16, fb16;
    // cond encoder
    Lin init; struct AB { Dev<float> nw, nb; Lin qkv, proj; }; std::vector<std::unique_ptr<AB>> blocks;
    // perceiver
    Dev<float> latents, gamma; struct PL { Lin q, kv, o, f1, f2; }; std::vector<std::unique_ptr<PL>> pl;
    int inner = 0, ffi = 0;
    // speaker encoder
    Dev<float> conv1_w, conv1_b; Bn bn1; std::vector<std::unique_ptr<Block>> res; Lin att0, att3, fc; Bn att_bn;
    // workspaces
    Dev<float> wav22, wav16, pre16, F, D, P, mel, h0, h1, xn, qkv, att, kvin, q, kv, o, lat, ff, gg, img, a0, a1, a2, ds,
        chm, gate, xT, at1, at2, pooled;
    Dev<AttnSeq> seq;

    void lin(Lin& l, const HostTensorView& w, const HostTensorView* b) {
        l.N = (int)w.shape[0]; l.K = (int)(w.numel() / w.shape[0]);
        l.w.up(std::vector<float>(w.data, w.data + w.numel()), st);
        std::vector<float> bias(l.N, 0.f);
        if (b) std::copy(b->data, b->data + l.N, bias.begin());
        l.b.up(bias, st); l.has_b = b != nullptr;
    }
    void bn(Bn& o, const std::function<HostTensorView(const std::string&)>& get, const std::string& p) {
        auto w = get(p + ".weight"), b = get(p + ".bias"), m = get(p + ".running_mean"), v = get(p + ".running_var");
        const size_t n = w.numel();
        std::vector<float> sc(n), sh(n);
        for (size_t i = 0; i < n; ++i) { sc[i] = w.data[i] / std::sqrt(v.data[i] + 1e-5f); sh[i] = b.data[i] - m.data[i] * sc[i]; }
        o.scale.up(sc, st); o.shift.up(sh, st);
    }
    void gemm(const float* A, const Lin& l, const float* resid, float* out, int M, int flags = 0) {
        launch_gemm_f32(A, l.w.p, l.b.p, resid, out, M, l.N, l.K, flags | (resid ? GEMM_RESID : 0), st);
    }
    // `cap`: floats `out` holds (launch_conv2d throws before launching when the output does not fit)
    void conv2d(const float* in, const float* w, const float* bias, const Bn* bnp, float* out, size_t cap, int Cin, int Cout,
                int Hin, int Win, int k, int stride, int relu_before_bn, int& Hout, int& Wout) {
        launch_conv2d(in, w, bias, bnp ? bnp->scale.p : nullptr, bnp ? bnp->shift.p : nullptr, out, cap, Cin, Cout, Hin, Win, k,
                      stride, relu_before_bn, Hout, Wout, st);
    }
    // 22.05 kHz front-end: x [len] (device) -> mel [1 + len/256][n_mels] (utilities.py:53-70 with XTTSv2.py:374-386)
    void mel22(const float* x, int len, float* mel_out, size_t cap) {
        const int T = 1 + len / 256, nb = 1025;
        if ((size_t)T * c.n_mels > cap) throw std::runtime_error("mel22: output exceeds its buffer");
        F.ensure((size_t)T * 1024); D.ensure((size_t)T * 2 * nb); P.ensure((size_t)T * nb);
        launch_frame_window(x, len, hann.p, 1024, 256, 512, 1024, PAD_REFLECT, F.p, T, 256, st);
        launch_gemm_f32(F.p, basis22.p, nullptr, nullptr, D.p, T, 2 * nb, 1024, 0, st);
        launch_power(D.p, P.p, T, nb, st);
        launch_gemm_f32(P.p, fb22.p, nullptr, nullptr, mel_out, T, c.n_mels, nb, 0, st);
        launch_mel_log(mel_out, mel_stats.p, (size_t)T * c.n_mels, c.n_mels, 0, st);
    }
    // 16 kHz front-end: x [N] (device) -> InstanceNorm'd log-mel image [spk_mels][1 + N/160] (hifigan_decoder.py:602-613)
    void mel16(const float* x, int N, float* img_out, size_t cap) {
        const int T = 1 + N / 160, nb = 257, NM = c.spk_mels;
        if ((size_t)NM * T > cap) throw std::runtime_error("mel16: output exceeds its buffer");
        pre16.ensure(N); F.ensure((size_t)T * 400); D.ensure((size_t)T * 2 * nb); P.ensure((size_t)T * nb); mel.ensure((size_t)T * NM);
        launch_preemphasis(x, pre16.p, N, 0.97f, st);
        launch_frame_window(pre16.p, N, hamm.p, 400, 160, 56, 256, PAD_REFLECT, F.p, T, 128, st);
        launch_gemm_f32(F.p, basis16.p, nullptr, nullptr, D.p, T, 2 * nb, 400, 0, st);
        launch_power(D.p, P.p, T, nb, st);
        launch_gemm_f32(P.p, fb16.p, nullptr, nullptr, mel.p, T, NM, nb, 0, st);
        launch_mel_log(mel.p, nullptr, (size_t)T * NM, NM, 1, st);
        launch_instnorm_t(mel.p, img_out, T, NM, 1e-5f, st);
    }
};

Conditioner::Conditioner(const xtts_config& cfg, const std::function<HostTensorView(const std::string&)>& get, cudaStream_t st)
    : impl(new Impl()) {
    Impl& m = *impl;
    m.c = cfg; m.st = st; m.H = cfg.hidden; m.NH = cfg.heads;
    auto vec = [&](const std::string& n) { auto t = get(n); return std::vector<float>(t.data, t.data + t.numel()); };
    // ---- 22.05 kHz mel front-end (utilities.py:53-70 with XTTSv2.py:374-386 arguments)
    {
        std::vector<float> w(1024);
        for (int i = 0; i < 1024; ++i) w[i] = (float)(0.5 - 0.5 * std::cos(2.0 * kPi * i / 1024.0));    // periodic hann
        m.hann.up(w, st);
        m.basis22.up(dft_basis(2048, 1024, 512), st);
        m.fb22.up(mel_fb_t(1025, 0.0, 8000.0, cfg.n_mels, 22050, true), st);
        m.mel_stats.up(vec("mel_stats"), st);
    }
    // ---- ConditioningEncoder
    { auto w = get("conditioning_encoder.init.weight"), b = get("conditioning_encoder.init.bias"); m.lin(m.init, w, &b); }
    for (int i = 0; i < cfg.cond_blocks; ++i) {
        const std::string p = "conditioning_encoder.attn." + std::to_string(i) + ".";
        std::unique_ptr<Impl::AB> ab(new Impl::AB());
        ab->nw.up(vec(p + "norm.weight"), st); ab->nb.up(vec(p + "norm.bias"), st);
        { auto w = get(p + "qkv.weight"), b = get(p + "qkv.bias"); m.lin(ab->qkv, w, &b); }
        { auto w = get(p + "proj_out.weight"), b = get(p + "proj_out.bias"); m.lin(ab->proj, w, &b); }
        m.blocks.push_back(std::move(ab));
    }
    // ---- Perceiver
    m.latents.up(vec("conditioning_perceiver.latents"), st);
    m.gamma.up(vec("conditioning_perceiver.norm.gamma"), st);
    for (int l = 0; l < cfg.perceiver_depth; ++l) {
        const std::string p = "conditioning_perceiver.layers." + std::to_string(l) + ".";
        std::unique_ptr<Impl::PL> pl(new Impl::PL());
        { auto w = get(p + "0.to_q.weight"); m.lin(pl->q, w, nullptr); }
        { auto w = get(p + "0.to_kv.weight"); m.lin(pl->kv, w, nullptr); }
        { auto w = get(p + "0.to_out.weight"); m.lin(pl->o, w, nullptr); }
        { auto w = get(p + "1.0.weight"), b = get(p + "1.0.bias"); m.lin(pl->f1, w, &b); }
        { auto w = get(p + "1.2.weight"), b = get(p + "1.2.bias"); m.lin(pl->f2, w, &b); }
        m.inner = pl->q.N; m.ffi = pl->f2.K;
        m.pl.push_back(std::move(pl));
    }
    if (m.inner != cfg.perceiver_heads * kHeadDim) throw std::runtime_error("perceiver: heads*64 != to_q rows");
    // ---- speaker encoder
    const std::string s = "hifigan_decoder.speaker_encoder.";
    m.hamm.up(vec(s + "torch_spec.1.spectrogram.window"), st);
    m.basis16.up(dft_basis(512, 400, 56), st);
    {   // stored fb is [n_freqs, n_mels]; transpose for the NT GEMM
        auto fb = get(s + "torch_spec.1.mel_scale.fb");
        const int nf = (int)fb.shape[0], nm = (int)fb.shape[1];
        std::vector<float> t((size_t)nf * nm);
        for (int f = 0; f < nf; ++f) for (int k = 0; k < nm; ++k) t[(size_t)k * nf + f] = fb.data[(size_t)f * nm + k];
        m.fb16.up(t, st);
    }
    m.conv1_w.up(vec(s + "conv1.weight"), st); m.conv1_b.up(vec(s + "conv1.bias"), st);
    m.bn(m.bn1, get, s + "bn1");
    int inpl = cfg.spk_filters[0];
    for (int li = 0; li < 4; ++li) {
        const int planes = cfg.spk_filters[li];
        for (int b = 0; b < cfg.spk_layers[li]; ++b) {
            const std::string p = s + "layer" + std::to_string(li + 1) + "." + std::to_string(b) + ".";
            std::unique_ptr<Block> blk(new Block());
            blk->cin = (b == 0) ? inpl : planes; blk->cout = planes; blk->stride = (li > 0 && b == 0) ? 2 : 1;
            blk->c1.up(vec(p + "conv1.weight"), st); blk->c2.up(vec(p + "conv2.weight"), st);
            m.bn(blk->bn1, get, p + "bn1"); m.bn(blk->bn2, get, p + "bn2");
            { auto w = get(p + "se.fc.0.weight"), bb = get(p + "se.fc.0.bias"); m.lin(blk->se1, w, &bb); }
            { auto w = get(p + "se.fc.2.weight"), bb = get(p + "se.fc.2.bias"); m.lin(blk->se2, w, &bb); }
            blk->has_ds = (b == 0) && (blk->stride != 1 || inpl != planes);
            if (blk->has_ds) { blk->ds.up(vec(p + "downsample.0.weight"), st); m.bn(blk->bnd, get, p + "downsample.1"); }
            m.res.push_back(std::move(blk));
        }
        inpl = planes;
    }
    { auto w = get(s + "attention.0.weight"), b = get(s + "attention.0.bias"); m.lin(m.att0, w, &b); }
    m.bn(m.att_bn, get, s + "attention.2");
    { auto w = get(s + "attention.3.weight"), b = get(s + "attention.3.bias"); m.lin(m.att3, w, &b); }
    { auto w = get(s + "fc.weight"), b = get(s + "fc.bias"); m.lin(m.fc, w, &b); }
    m.seq.alloc(1);
}

Conditioner::~Conditioner() = default;

void Conditioner::run(const float* wav22k_host, int64_t n22, const float* wav16k_host, int64_t n16, int cond_len_s,
                      int chunk_len_s, float* cond_dev, float* g_dev) {
    Impl& m = *impl;
    const auto& c = m.c;
    cudaStream_t st = m.st;
    const int H = m.H, NC = c.n_cond_latents;
    // ================= GPT conditioning latents (XTTSv2.py:349-407)
    int64_t n = n22;
    if (cond_len_s > 0) n = std::min<int64_t>(n, (int64_t)22050 * cond_len_s);
    if (n < 2) throw std::runtime_error("condition: reference audio too short");
    m.wav22.ensure((size_t)n);
    CUDA_CHECK(cudaMemcpyAsync(m.wav22.p, wav22k_host, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
    const int64_t piece = (int64_t)22050 * std::max(1, chunk_len_s);
    std::vector<std::pair<int64_t, int64_t>> pieces;
    for (int64_t i = 0; i < n; i += piece) {
        const int64_t len = std::min(piece, n - i);
        if ((double)len < 22050 * 0.33) continue;                       // too short: ignored (XTTSv2.py:367-369)
        pieces.emplace_back(i, len);
    }
    if (pieces.empty()) throw std::runtime_error("condition: no usable reference piece (>= 0.33 s)");
    CUDA_CHECK(cudaMemsetAsync(cond_dev, 0, (size_t)NC * H * sizeof(float), st));
    for (auto& pc : pieces) {
        const int len = (int)pc.second;
        const int T = 1 + len / 256;
        m.mel.ensure((size_t)T * c.n_mels);
        m.mel22(m.wav22.p + pc.first, len, m.mel.p, m.mel.n);
        // ---- ConditioningEncoder (latent_encoder.py:242-253)
        m.h0.ensure((size_t)T * H); m.h1.ensure((size_t)T * H); m.xn.ensure((size_t)T * H); m.qkv.ensure((size_t)T * 3 * H); m.att.ensure((size_t)T * H);
        m.gemm(m.mel.p, m.init, nullptr, m.h0.p, T);
        float* h = m.h0.p; float* hn = m.h1.p;
        int groups = 32;
        if (H <= 16) groups = 8; else if (H <= 64) groups = 16;
        while (H % groups != 0) groups /= 2;
        for (auto& ab : m.blocks) {
            launch_groupnorm(h, ab->nw.p, ab->nb.p, m.xn.p, T, H, groups, 1e-5f, st);
            m.gemm(m.xn.p, ab->qkv, nullptr, m.qkv.p, T);
            AttnSeq sq{0, T, 0, T};
            CUDA_CHECK(cudaMemcpyAsync(m.seq.p, &sq, sizeof(sq), cudaMemcpyHostToDevice, st));
            AttnLayout A;
            A.q = m.qkv.p; A.k = m.qkv.p + kHeadDim; A.v = m.qkv.p + 2 * kHeadDim;
            A.q_row_stride = 3 * H; A.kv_row_stride = 3 * H; A.q_head_stride = 3 * kHeadDim; A.kv_head_stride = 3 * kHeadDim;
            A.heads = m.NH; A.scale = 0.125f; A.causal = 0;      // (q*64^-1/4).(k*64^-1/4), latent_encoder.py:120-121
            launch_attn_generic<float>(A, m.seq.p, 1, T, m.att.p, H, st);
            m.gemm(m.att.p, ab->proj, m.xn.p, hn, T);            // residual adds the NORMALISED x (App. B.6)
            std::swap(h, hn);
        }
        // ---- Perceiver (perceiver_encoder.py:422-442)
        const int NK = NC + T, inner = m.inner, ffi = m.ffi;
        m.lat.ensure((size_t)NC * H); m.kvin.ensure((size_t)NK * H); m.q.ensure((size_t)NC * inner); m.kv.ensure((size_t)NK * 2 * inner);
        m.o.ensure((size_t)NC * inner); m.ff.ensure((size_t)NC * 2 * ffi); m.gg.ensure((size_t)NC * ffi);
        CUDA_CHECK(cudaMemcpyAsync(m.lat.p, m.latents.p, (size_t)NC * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
        for (auto& pl : m.pl) {
            CUDA_CHECK(cudaMemcpyAsync(m.kvin.p, m.lat.p, (size_t)NC * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(m.kvin.p + (size_t)NC * H, h, (size_t)T * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
            m.gemm(m.lat.p, pl->q, nullptr, m.q.p, NC);
            m.gemm(m.kvin.p, pl->kv, nullptr, m.kv.p, NK);
            AttnSeq sq{0, NC, 0, NK};
            CUDA_CHECK(cudaMemcpyAsync(m.seq.p, &sq, sizeof(sq), cudaMemcpyHostToDevice, st));
            AttnLayout A;
            A.q = m.q.p; A.k = m.kv.p; A.v = m.kv.p + inner;
            A.q_row_stride = inner; A.kv_row_stride = 2 * inner; A.q_head_stride = kHeadDim; A.kv_head_stride = kHeadDim;
            A.heads = c.perceiver_heads; A.scale = 0.125f; A.causal = 0;
            launch_attn_generic<float>(A, m.seq.p, 1, NC, m.o.p, inner, st);
            m.gemm(m.o.p, pl->o, m.lat.p, m.lat.p, NC);
            m.gemm(m.lat.p, pl->f1, nullptr, m.ff.p, NC);
            launch_geglu(m.ff.p, m.gg.p, NC, ffi, st);
            m.gemm(m.gg.p, pl->f2, m.lat.p, m.lat.p, NC);
        }
        launch_rmsnorm_accum(m.lat.p, m.gamma.p, cond_dev, NC, H, 1.0f / (float)pieces.size(), st);
    }
    // ================= d-vector (hifigan_decoder.py:602-646)
    {
        const int N = (int)n16;
        if (N < 400) throw std::runtime_error("condition: 16 kHz reference too short");
        const int T = 1 + N / 160, NM = c.spk_mels;
        m.wav16.ensure(N); m.img.ensure((size_t)NM * T);
        CUDA_CHECK(cudaMemcpyAsync(m.wav16.p, wav16k_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
        m.mel16(m.wav16.p, N, m.img.p, m.img.n);
        const size_t big = (size_t)c.spk_filters[0] * NM * T;
        m.a0.ensure(big); m.a1.ensure(big); m.a2.ensure(big);
        const size_t acap = std::min(m.a0.n, std::min(m.a1.n, m.a2.n));
        int Hc = NM, Wc = T, Ho, Wo;
        m.conv2d(m.img.p, m.conv1_w.p, m.conv1_b.p, &m.bn1, m.a0.p, acap, 1, c.spk_filters[0], Hc, Wc, 3, 1, 1, Ho, Wo);
        float* x = m.a0.p; float* t1 = m.a1.p; float* t2 = m.a2.p;
        m.chm.ensure(4096); m.gate.ensure(4096);
        for (auto& blk : m.res) {
            int H1, W1, H2, W2;
            m.conv2d(x, blk->c1.p, nullptr, &blk->bn1, t1, acap, blk->cin, blk->cout, Hc, Wc, 3, blk->stride, 1, H1, W1);
            m.conv2d(t1, blk->c2.p, nullptr, &blk->bn2, t2, acap, blk->cout, blk->cout, H1, W1, 3, 1, 0, H2, W2);
            const int HW = H2 * W2;
            launch_channel_mean(t2, m.chm.p, blk->cout, HW, st);
            launch_se_gate(m.chm.p, blk->se1.w.p, blk->se1.b.p, blk->se2.w.p, blk->se2.b.p, m.gate.p, blk->cout, blk->se1.N, st);
            const float* resid = x;
            if (blk->has_ds) {      // 1x1 conv at the block's stride: [cout][(Hc-1)/stride+1][(Wc-1)/stride+1]
                int Hd, Wd;
                m.ds.ensure((size_t)blk->cout * conv_out(Hc, 1, blk->stride) * conv_out(Wc, 1, blk->stride));
                m.conv2d(x, blk->ds.p, nullptr, &blk->bnd, m.ds.p, m.ds.n, blk->cin, blk->cout, Hc, Wc, 1, blk->stride, 0, Hd, Wd);
                resid = m.ds.p;
            }
            launch_se_apply(t2, m.gate.p, resid, t1, HW, (size_t)blk->cout * HW, st);
            std::swap(x, t1);
            Hc = H2; Wc = W2;
        }
        // x: [C4][Hc][Wc] -> feats [C4*Hc][Wc]
        const int CF = c.spk_filters[3] * Hc, Tt = Wc;
        m.xT.ensure((size_t)Tt * CF); m.at1.ensure((size_t)Tt * m.att0.N); m.at2.ensure((size_t)Tt * CF); m.pooled.ensure(2 * CF);
        launch_transpose(x, m.xT.p, CF, Tt, st);
        m.gemm(m.xT.p, m.att0, nullptr, m.at1.p, Tt);
        launch_relu_bn_rows(m.at1.p, m.att_bn.scale.p, m.att_bn.shift.p, (size_t)Tt * m.att0.N, m.att0.N, st);
        m.gemm(m.at1.p, m.att3, nullptr, m.at2.p, Tt);
        launch_asp(m.at2.p, x, m.pooled.p, Tt, CF, st);
        launch_gemv(m.fc.w.p, m.fc.b.p, m.pooled.p, g_dev, m.fc.N, m.fc.K, st);
        launch_l2norm(g_dev, m.fc.N, st);
    }
}

void Conditioner::frontend(int op, const float* x_dev, int n, float* out_dev, size_t cap) {
    if (op == XTTS_COND_MEL22) impl->mel22(x_dev, n, out_dev, cap);
    else impl->mel16(x_dev, n, out_dev, cap);
}
int Conditioner::n_mels() const { return impl->c.n_mels; }
int Conditioner::spk_mels() const { return impl->c.spk_mels; }

// ---------------------------------------------------------------------------------------- xtts_debug_cond
namespace {
constexpr int kGuardWords = 256;
constexpr uint32_t kGuardBits = 0x7fc5a5a5u;       // a quiet-NaN payload no kernel here produces
}  // namespace

void cond_debug(Conditioner* cnd, int op, const int32_t* dims, int n_dims, const float* scal, int n_scal, const float* const* in,
                const int64_t* in_len, int n_in, float* out, int64_t out_len, cudaStream_t st) {
    static const int kDims[XTTS_COND_N_OPS] = {8, 2, 3, 1, 2, 3, 2, 2, 9, 2, 2, 2, 2, 2, 2, 1, 3, 1, 1};
    static const int kScal[XTTS_COND_N_OPS] = {0, 0, 0, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    auto bad = [](const std::string& s) { return std::runtime_error("debug_cond: " + s); };
    if (op < 0 || op >= XTTS_COND_N_OPS) throw bad("unknown op " + std::to_string(op));
    if (n_dims != kDims[op] || n_scal != kScal[op])
        throw bad("op " + std::to_string(op) + " takes " + std::to_string(kDims[op]) + " dims and " + std::to_string(kScal[op]) + " scalars");
    if ((n_dims && !dims) || (n_scal && !scal) || (n_in > 0 && (!in || !in_len)) || !out) throw bad("NULL argument");
    for (int i = 0; i < n_dims; ++i)
        if (dims[i] < 0) throw bad("negative dim");
    auto d = [&](int i) { return (int64_t)dims[i]; };
    auto pos = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (dims[i] < 1) throw bad("dim " + std::to_string(i) + " must be >= 1");
    };
    std::vector<int64_t> need;       // in_len each input must have
    int64_t need_out = 0;
    switch (op) {
    case XTTS_COND_FRAME_WINDOW:     // n, wlen, hop, off, pad, pad_mode, frames, threads
        pos({0, 1, 2, 6});
        if (d(5) != PAD_REFLECT && d(5) != PAD_ZERO) throw bad("pad_mode must be 0 (reflect) or 1 (zero)");
        if (d(7) != 128 && d(7) != 256) throw bad("frame_window runs 128 or 256 threads");
        need = {d(0), d(1)}; need_out = d(6) * d(1); break;
    case XTTS_COND_POWER:            // frames, nb
        pos({0, 1}); need = {d(0) * 2 * d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_MEL_LOG:          // n, C, mode
        pos({0, 1});
        if (d(2) > 1) throw bad("mel_log mode must be 0 or 1");
        need = d(2) == 0 ? std::vector<int64_t>{d(1)} : std::vector<int64_t>{}; need_out = d(0); break;
    case XTTS_COND_PREEMPHASIS:      // n
        if (d(0) < 2) throw bad("preemphasis needs n >= 2");
        need = {d(0)}; need_out = d(0); break;
    case XTTS_COND_INSTNORM_T:       // T, C
        pos({0, 1}); need = {d(0) * d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_GROUPNORM:        // T, C, groups
        pos({0, 1, 2});
        if (d(1) % d(2) != 0) throw bad("groupnorm needs C % groups == 0");
        need = {d(0) * d(1), d(1), d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_GEGLU:            // rows, F
        pos({0, 1}); need = {d(0) * 2 * d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_RMSNORM_ACCUM:    // rows, C
        pos({0, 1}); need = {d(0) * d(1), d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_CONV2D: {         // Cin, Cout, Hin, Win, k, stride, relu_before_bn, has_bias, has_bn
        pos({0, 1, 2, 3, 4, 5});
        if (d(4) % 2 == 0) throw bad("conv2d needs an odd k");
        if (d(6) > 1 || d(7) > 1 || d(8) > 1) throw bad("conv2d flags must be 0 or 1");
        if (conv2d_smem(dims[0], dims[4]) > kSmemLimit) throw bad("conv2d weight slice exceeds 48 KB of shared memory");
        const int64_t Ho = conv_out(dims[2], dims[4], dims[5]), Wo = conv_out(dims[3], dims[4], dims[5]);
        if (Ho < 1 || Wo < 1) throw bad("conv2d output is empty");
        need = {d(0) * d(2) * d(3), d(1) * d(0) * d(4) * d(4)};
        if (d(7)) need.push_back(d(1));
        if (d(8)) { need.push_back(d(1)); need.push_back(d(1)); }
        need_out = d(1) * Ho * Wo; break;
    }
    case XTTS_COND_CHANNEL_MEAN:     // C, HW
        pos({0, 1}); need = {d(0) * d(1)}; need_out = d(0); break;
    case XTTS_COND_SE_GATE:          // C, R
        pos({0, 1});
        if ((size_t)d(1) * sizeof(float) > kSmemLimit) throw bad("se_gate hidden layer exceeds 48 KB of shared memory");
        need = {d(0), d(1) * d(0), d(1), d(0) * d(1), d(0)}; need_out = d(0); break;
    case XTTS_COND_SE_APPLY:         // C, HW
        pos({0, 1}); need = {d(0) * d(1), d(0), d(0) * d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_TRANSPOSE:        // R, Cc
        pos({0, 1}); need = {d(0) * d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_RELU_BN_ROWS:     // rows, C
        pos({0, 1}); need = {d(1), d(1)}; need_out = d(0) * d(1); break;
    case XTTS_COND_ASP:              // T, C
        pos({0, 1}); need = {d(0) * d(1), d(1) * d(0)}; need_out = 2 * d(1); break;
    case XTTS_COND_L2NORM:           // n
        pos({0}); need = {}; need_out = d(0); break;
    case XTTS_COND_GEMV:             // rows, cols, has_bias
        pos({0, 1});
        if (d(2) > 1) throw bad("gemv has_bias must be 0 or 1");
        need = {d(0) * d(1), d(1)};
        if (d(2)) need.push_back(d(0));
        need_out = d(0); break;
    case XTTS_COND_MEL22:            // n
    case XTTS_COND_MEL16:
        if (!cnd) throw bad("the checkpoint has no conditioning weights");
        if (op == XTTS_COND_MEL22 && d(0) < 2) throw bad("mel22 needs n >= 2");
        if (op == XTTS_COND_MEL16 && d(0) < 400) throw bad("mel16 needs n >= 400");
        need = {d(0)};
        need_out = op == XTTS_COND_MEL22 ? (1 + d(0) / 256) * cnd->n_mels() : (int64_t)cnd->spk_mels() * (1 + d(0) / 160);
        break;
    }
    if (n_in != (int)need.size()) throw bad("op " + std::to_string(op) + " takes " + std::to_string(need.size()) + " inputs");
    for (int i = 0; i < n_in; ++i) {
        if (in_len[i] != need[i])
            throw bad("input " + std::to_string(i) + " has " + std::to_string(in_len[i]) + " floats, expected " + std::to_string(need[i]));
        if (!in[i]) throw bad("input " + std::to_string(i) + " is NULL");
    }
    if (out_len < 1 || out_len != need_out) throw bad("out has " + std::to_string(out_len) + " floats, expected " + std::to_string(need_out));

    std::vector<std::unique_ptr<Dev<float>>> din;
    std::vector<const float*> ip(n_in);
    for (int i = 0; i < n_in; ++i) {
        din.emplace_back(new Dev<float>());
        din.back()->up(std::vector<float>(in[i], in[i] + in_len[i]), st);
        ip[i] = din.back()->p;
    }
    // out with kGuardWords sentinel words on each side; its incoming contents are uploaded (in-place kernels read them)
    std::vector<uint32_t> h((size_t)out_len + 2 * kGuardWords, kGuardBits);
    std::memcpy(h.data() + kGuardWords, out, (size_t)out_len * sizeof(float));
    Dev<float> dout;
    dout.alloc(h.size());
    CUDA_CHECK(cudaMemcpyAsync(dout.p, h.data(), h.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    float* o = dout.p + kGuardWords;
    const float* const* I = ip.data();
    const int* D = dims;
    int Ho = 0, Wo = 0;
    switch (op) {
    case XTTS_COND_FRAME_WINDOW:
        launch_frame_window(I[0], D[0], I[1], D[1], D[2], D[3], D[4], D[5], o, D[6], D[7], st); break;
    case XTTS_COND_POWER: launch_power(I[0], o, D[0], D[1], st); break;
    case XTTS_COND_MEL_LOG: launch_mel_log(o, D[2] == 0 ? I[0] : nullptr, (size_t)D[0], D[1], D[2], st); break;
    case XTTS_COND_PREEMPHASIS: launch_preemphasis(I[0], o, D[0], scal[0], st); break;
    case XTTS_COND_INSTNORM_T: launch_instnorm_t(I[0], o, D[0], D[1], scal[0], st); break;
    case XTTS_COND_GROUPNORM: launch_groupnorm(I[0], I[1], I[2], o, D[0], D[1], D[2], scal[0], st); break;
    case XTTS_COND_GEGLU: launch_geglu(I[0], o, D[0], D[1], st); break;
    case XTTS_COND_RMSNORM_ACCUM: launch_rmsnorm_accum(I[0], I[1], o, D[0], D[1], scal[0], st); break;
    case XTTS_COND_CONV2D: {
        const float* bias = D[7] ? I[2] : nullptr;
        const float* sc = D[8] ? I[2 + D[7]] : nullptr;
        const float* sh = D[8] ? I[3 + D[7]] : nullptr;
        launch_conv2d(I[0], I[1], bias, sc, sh, o, (size_t)out_len, D[0], D[1], D[2], D[3], D[4], D[5], D[6], Ho, Wo, st);
        break;
    }
    case XTTS_COND_CHANNEL_MEAN: launch_channel_mean(I[0], o, D[0], D[1], st); break;
    case XTTS_COND_SE_GATE: launch_se_gate(I[0], I[1], I[2], I[3], I[4], o, D[0], D[1], st); break;
    case XTTS_COND_SE_APPLY: launch_se_apply(I[0], I[1], I[2], o, D[1], (size_t)D[0] * D[1], st); break;
    case XTTS_COND_TRANSPOSE: launch_transpose(I[0], o, D[0], D[1], st); break;
    case XTTS_COND_RELU_BN_ROWS: launch_relu_bn_rows(o, I[0], I[1], (size_t)D[0] * D[1], D[1], st); break;
    case XTTS_COND_ASP: launch_asp(I[0], I[1], o, D[0], D[1], st); break;
    case XTTS_COND_L2NORM: launch_l2norm(o, D[0], st); break;
    case XTTS_COND_GEMV: launch_gemv(I[0], D[2] ? I[2] : nullptr, I[1], o, D[0], D[1], st); break;
    case XTTS_COND_MEL22:
    case XTTS_COND_MEL16: cnd->frontend(op, I[0], D[0], o, (size_t)out_len); break;
    }
    CUDA_CHECK(cudaMemcpyAsync(h.data(), dout.p, h.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    for (int i = 0; i < kGuardWords; ++i)
        if (h[i] != kGuardBits || h[kGuardWords + out_len + i] != kGuardBits)
            throw bad("op " + std::to_string(op) + " wrote outside its output");
    std::memcpy(out, h.data() + kGuardWords, (size_t)out_len * sizeof(float));
}

}  // namespace xtts
