// Speaker-conditioning kernels and driver (see cond.h).  Activations are time-major rows [T, C] so every
// 1x1 convolution / nn.Linear is one call of the shared NT GEMM; the STFTs are DFT-by-GEMM against
// precomputed (cos | -sin) bases restricted to the window support (n_fft 2048 -> 1024 live taps).
// Per-speaker, cached by the engine: clarity over peak speed, fp32 throughout.
#include <cmath>
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
    Dev<float> wav22, wav16, pre16, F, D, P, mel, h0, h1, xn, qkv, att, kvin, q, kv, o, lat, ff, gg, img, a0, a1, a2,
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
    void conv2d(const float* in, const float* w, const float* bias, const Bn* bnp, float* out, int Cin, int Cout, int Hin,
                int Win, int k, int stride, int relu_before_bn, int& Hout, int& Wout) {
        const int pad = k / 2;
        Hout = (Hin + 2 * pad - k) / stride + 1; Wout = (Win + 2 * pad - k) / stride + 1;
        dim3 grid(ceil_div(Wout, 128), Hout, ceil_div(Cout, C2_CO));
        conv2d_kernel<<<grid, 128, (size_t)C2_CO * Cin * k * k * sizeof(float), st>>>(
            in, w, bias, bnp ? bnp->scale.p : nullptr, bnp ? bnp->shift.p : nullptr, out, Cin, Cout, Hin, Win, Hout, Wout, k,
            stride, relu_before_bn);
        COUNT_LAUNCH(); KERNEL_CHECK();
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
    const int nb22 = 1025;
    bool first = true;
    for (auto& pc : pieces) {
        const int len = (int)pc.second;
        const int T = 1 + len / 256;
        m.F.ensure((size_t)T * 1024); m.D.ensure((size_t)T * 2 * nb22); m.P.ensure((size_t)T * nb22); m.mel.ensure((size_t)T * c.n_mels);
        frame_window_kernel<<<T, 256, 0, st>>>(m.wav22.p + pc.first, len, m.hann.p, 1024, 256, 512, 1024, PAD_REFLECT, m.F.p, T);
        COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(m.F.p, m.basis22.p, nullptr, nullptr, m.D.p, T, 2 * nb22, 1024, 0, st);
        power_kernel<<<nblk((size_t)T * nb22), 256, 0, st>>>(m.D.p, m.P.p, T, nb22); COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(m.P.p, m.fb22.p, nullptr, nullptr, m.mel.p, T, c.n_mels, nb22, 0, st);
        mel_log_kernel<<<nblk((size_t)T * c.n_mels), 256, 0, st>>>(m.mel.p, m.mel_stats.p, (size_t)T * c.n_mels, c.n_mels, 0);
        COUNT_LAUNCH(); KERNEL_CHECK();
        if (first) {
            last_mel.resize((size_t)T * c.n_mels); last_mel_frames = T;
            CUDA_CHECK(cudaMemcpyAsync(last_mel.data(), m.mel.p, last_mel.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
            first = false;
        }
        // ---- ConditioningEncoder (latent_encoder.py:242-253)
        m.h0.ensure((size_t)T * H); m.h1.ensure((size_t)T * H); m.xn.ensure((size_t)T * H); m.qkv.ensure((size_t)T * 3 * H); m.att.ensure((size_t)T * H);
        m.gemm(m.mel.p, m.init, nullptr, m.h0.p, T);
        float* h = m.h0.p; float* hn = m.h1.p;
        int groups = 32;
        if (H <= 16) groups = 8; else if (H <= 64) groups = 16;
        while (H % groups != 0) groups /= 2;
        for (auto& ab : m.blocks) {
            groupnorm_rows_kernel<<<groups, 256, 0, st>>>(h, ab->nw.p, ab->nb.p, m.xn.p, T, H, groups, 1e-5f);
            COUNT_LAUNCH(); KERNEL_CHECK();
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
            geglu_kernel<<<nblk((size_t)NC * ffi), 256, 0, st>>>(m.ff.p, m.gg.p, NC, ffi); COUNT_LAUNCH(); KERNEL_CHECK();
            m.gemm(m.gg.p, pl->f2, m.lat.p, m.lat.p, NC);
        }
        rmsnorm_accum_kernel<<<NC, 256, 0, st>>>(m.lat.p, m.gamma.p, cond_dev, H, 1.0f / (float)pieces.size());
        COUNT_LAUNCH(); KERNEL_CHECK();
    }
    // ================= d-vector (hifigan_decoder.py:602-646)
    {
        const int N = (int)n16;
        if (N < 400) throw std::runtime_error("condition: 16 kHz reference too short");
        m.wav16.ensure(N); m.pre16.ensure(N);
        CUDA_CHECK(cudaMemcpyAsync(m.wav16.p, wav16k_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
        preemphasis_kernel<<<nblk(N), 256, 0, st>>>(m.wav16.p, m.pre16.p, N, 0.97f); COUNT_LAUNCH(); KERNEL_CHECK();
        const int T = 1 + N / 160, nb = 257, NM = c.spk_mels;
        m.F.ensure((size_t)T * 400); m.D.ensure((size_t)T * 2 * nb); m.P.ensure((size_t)T * nb); m.mel.ensure((size_t)T * NM);
        frame_window_kernel<<<T, 128, 0, st>>>(m.pre16.p, N, m.hamm.p, 400, 160, 56, 256, PAD_REFLECT, m.F.p, T); COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(m.F.p, m.basis16.p, nullptr, nullptr, m.D.p, T, 2 * nb, 400, 0, st);
        power_kernel<<<nblk((size_t)T * nb), 256, 0, st>>>(m.D.p, m.P.p, T, nb); COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(m.P.p, m.fb16.p, nullptr, nullptr, m.mel.p, T, NM, nb, 0, st);
        mel_log_kernel<<<nblk((size_t)T * NM), 256, 0, st>>>(m.mel.p, nullptr, (size_t)T * NM, NM, 1); COUNT_LAUNCH(); KERNEL_CHECK();
        m.img.ensure((size_t)NM * T);
        instnorm_transpose_kernel<<<NM, 256, 0, st>>>(m.mel.p, m.img.p, T, NM, 1e-5f); COUNT_LAUNCH(); KERNEL_CHECK();
        const size_t big = (size_t)c.spk_filters[0] * NM * T;
        m.a0.ensure(big); m.a1.ensure(big); m.a2.ensure(big);
        int Hc = NM, Wc = T, Ho, Wo;
        m.conv2d(m.img.p, m.conv1_w.p, m.conv1_b.p, &m.bn1, m.a0.p, 1, c.spk_filters[0], Hc, Wc, 3, 1, 1, Ho, Wo);
        float* x = m.a0.p; float* t1 = m.a1.p; float* t2 = m.a2.p;
        m.chm.ensure(4096); m.gate.ensure(4096);
        Dev<float> dsbuf; dsbuf.alloc(big / 2 + 16);
        for (auto& blk : m.res) {
            int H1, W1, H2, W2;
            m.conv2d(x, blk->c1.p, nullptr, &blk->bn1, t1, blk->cin, blk->cout, Hc, Wc, 3, blk->stride, 1, H1, W1);
            m.conv2d(t1, blk->c2.p, nullptr, &blk->bn2, t2, blk->cout, blk->cout, H1, W1, 3, 1, 0, H2, W2);
            const int HW = H2 * W2;
            channel_mean_kernel<<<blk->cout, 256, 0, st>>>(t2, m.chm.p, HW); COUNT_LAUNCH(); KERNEL_CHECK();
            se_gate_kernel<<<1, 256, blk->se1.N * sizeof(float), st>>>(m.chm.p, blk->se1.w.p, blk->se1.b.p, blk->se2.w.p,
                                                                        blk->se2.b.p, m.gate.p, blk->cout, blk->se1.N);
            COUNT_LAUNCH(); KERNEL_CHECK();
            const float* resid = x;
            if (blk->has_ds) {
                int Hd, Wd;
                m.conv2d(x, blk->ds.p, nullptr, &blk->bnd, dsbuf.p, blk->cin, blk->cout, Hc, Wc, 1, blk->stride, 0, Hd, Wd);
                resid = dsbuf.p;
            }
            const size_t ne = (size_t)blk->cout * HW;
            se_apply_kernel<<<nblk(ne), 256, 0, st>>>(t2, m.gate.p, resid, t1, HW, ne); COUNT_LAUNCH(); KERNEL_CHECK();
            std::swap(x, t1);
            Hc = H2; Wc = W2;
        }
        // x: [C4][Hc][Wc] -> feats [C4*Hc][Wc]
        const int CF = c.spk_filters[3] * Hc, Tt = Wc;
        m.xT.ensure((size_t)Tt * CF); m.at1.ensure((size_t)Tt * m.att0.N); m.at2.ensure((size_t)Tt * CF); m.pooled.ensure(2 * CF);
        transpose_kernel<<<nblk((size_t)CF * Tt), 256, 0, st>>>(x, m.xT.p, CF, Tt); COUNT_LAUNCH(); KERNEL_CHECK();
        m.gemm(m.xT.p, m.att0, nullptr, m.at1.p, Tt);
        relu_bn_rows_kernel<<<nblk((size_t)Tt * m.att0.N), 256, 0, st>>>(m.at1.p, m.att_bn.scale.p, m.att_bn.shift.p, (size_t)Tt * m.att0.N, m.att0.N);
        COUNT_LAUNCH(); KERNEL_CHECK();
        m.gemm(m.at1.p, m.att3, nullptr, m.at2.p, Tt);
        asp_kernel<<<CF, 128, 0, st>>>(m.at2.p, x, m.pooled.p, Tt, CF); COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemv(m.fc.w.p, m.fc.b.p, m.pooled.p, g_dev, m.fc.N, m.fc.K, st);
        l2norm_kernel<<<1, 256, 0, st>>>(g_dev, m.fc.N); COUNT_LAUNCH(); KERNEL_CHECK();
        CUDA_CHECK(cudaStreamSynchronize(st));      // dsbuf goes out of scope
    }
}

}  // namespace xtts
