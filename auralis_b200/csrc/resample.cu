// Resampler (see cond.h): torchaudio.functional.resample(x, orig, new) for float32 x with its defaults
// (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), the reference's resampler (common/utilities.py:94,
// models/base.py:220, XTTSv2.py:322,362), on the GPU.
//
// With g = gcd(orig, new), L = orig / g, M = new / g, base = min(L, M) * 0.99 (double), width = ceil(6 L / base):
//   tap k in [0, 2 width + L) of phase p in [0, M) has the scaled argument
//     t = f32(f32(f32(-p) / M) + f32(k - width) / L) * f32(base)
//   and torchaudio's float32 coefficient (its kernel is built in the waveform's dtype, in this operation order)
//     c = (t' == 0 ? 1 : sin(t') / t') * (cos(t * pi / 6 / 2)^2 * f32(base / L)),   t' = t * pi,   t clamped to +-6
//   output j = q M + p is sum_k c[p][k] * x[q L + k - width], x = 0 outside [0, n); n_out = ceil(M n / L).
// torchaudio evaluates all 2 width + L taps.  t is non-decreasing in k, so the taps with -6 < t < 6 are one run per
// phase, of at most 2 width + 2 taps; outside it t is clamped to +-6 and |c| < 5e-24.  Those taps are skipped: each
// output is a T-tap fp32 FMA chain, T = min(2 width + 2, 2 width + L), over a band that starts at kstart[p] and holds
// the run (zero coefficients pad it).  IEEE division and the accurate sinf / cosf, no fast-math.  The chain's order is
// fixed per output, so the result does not depend on the launch shape or on the pass size.
//
// Workspace: the band table (T x M floats + M ints, at most ~17 M floats for rates up to 2^20 - 1), cached for the last
// (L, M); per pass at most B outputs (engine option "resample_block_samples") and the B + 2 width + L input samples they
// read: (2 B + 2 width + L) floats.
#include <cmath>
#include <cstring>
#include <numeric>
#include <stdexcept>

#include "cond.h"

namespace xtts {
namespace {

constexpr int kWidth = 6;
constexpr int kThreads = 256, kPerThread = 4, kOutPerCta = kThreads * kPerThread;
constexpr int kSmemFloats = 24 * 1024;                 // 96 KB: the largest input span a CTA stages
constexpr int64_t kMaxIn = (int64_t)1 << 40;           // keeps M * n inside int64
constexpr float kPiF = (float)kPi;

struct Geo {
    int L, M, width, K, T;    // K = 2 width + L dense taps, T band taps
    float base, scale;        // f32(base), f32(base / L)
};

__device__ __forceinline__ float scaled_arg(int p, int k, const Geo& g) {
    const float idx = __fdiv_rn((float)(k - g.width), (float)g.L);
    return __fmul_rn(__fadd_rn(__fdiv_rn((float)(-p), (float)g.M), idx), g.base);
}

// kstart[p]: the first tap of phase p with t > -6, moved left so that the T-tap band ends inside [0, K).  bad |= 2 when
// the run of taps with -6 < t < 6 would not fit in T (cannot happen for width = ceil(6 L / base); checked all the same).
__global__ void rs_band_kernel(Geo g, int* __restrict__ kstart, int* __restrict__ bad) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.M) return;
    int lo = 0, hi = g.K;                                // smallest k with t(k) > -6, K if none
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (scaled_arg(p, mid, g) > -(float)kWidth) hi = mid; else lo = mid + 1;
    }
    const int ks = min(lo, g.K - g.T);
    if (ks + g.T < g.K && scaled_arg(p, ks + g.T, g) < (float)kWidth) atomicOr(bad, 2);
    kstart[p] = ks;
}

// tab[i][p] = c(p, kstart[p] + i) for the taps inside the window, 0 for the others (tap-major: the 32 consecutive
// outputs of a warp have consecutive phases, so each tap's coefficients are one coalesced read)
__global__ void rs_coef_kernel(Geo g, const int* __restrict__ kstart, float* __restrict__ tab) {
    const int64_t total = (int64_t)g.M * g.T;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)(e / g.T), i = (int)(e % g.T);
        const float t = scaled_arg(p, kstart[p] + i, g);
        float c = 0.f;
        if (t > -(float)kWidth && t < (float)kWidth) {
            const float cw = cosf(__fdiv_rn(__fdiv_rn(__fmul_rn(t, kPiF), (float)kWidth), 2.f));
            const float win = __fmul_rn(cw, cw);
            const float tp = __fmul_rn(t, kPiF);
            const float s = tp == 0.f ? 1.f : __fdiv_rn(sinf(tp), tp);
            c = __fmul_rn(s, __fmul_rn(win, g.scale));
        }
        tab[(size_t)i * g.M + p] = c;
    }
}

// bad |= 1 when any of the n samples is not finite
__global__ void rs_finite_kernel(const float* __restrict__ x, int64_t n, int* __restrict__ bad) {
    int nf = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        nf |= !isfinite(x[i]);
    if (__reduce_or_sync(0xffffffffu, (unsigned)nf) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
}

// Outputs j0 .. j0 + n - 1 -> y[0 .. n).  xb holds x[b0 .. b1) (the pass's input; every sample an output reads that lies
// in [0, n_in) is there), anything else reads as 0.  Each CTA covers kOutPerCta consecutive outputs; thread t computes
// outputs t, t + 256, t + 512, t + 768 of them.  kStage: the CTA first copies the dense span its outputs read,
// [qa L - width, qb L + L + width), into shared memory; otherwise (a span above kSmemFloats) the taps are read from
// global memory.  Both run the same chain.
template <bool kStage>
__global__ void __launch_bounds__(kThreads) rs_resample_kernel(const float* __restrict__ xb, int64_t b0, int64_t b1,
                                                               const float* __restrict__ tab,
                                                               const int* __restrict__ kstart, Geo g, int64_t j0,
                                                               int64_t n, float* __restrict__ y) {
    extern __shared__ float sx[];
    const int64_t ja = j0 + (int64_t)blockIdx.x * kOutPerCta;
    const int64_t jb = min(j0 + n, ja + kOutPerCta);
    const int64_t s = (ja / g.M) * g.L - g.width;                       // first input sample of the CTA's span
    if (kStage) {
        const int64_t e = ((jb - 1) / g.M) * g.L + g.L + g.width;
        for (int64_t i = threadIdx.x; i < e - s; i += kThreads) {
            const int64_t gi = s + i;
            sx[i] = gi >= b0 && gi < b1 ? xb[gi - b0] : 0.f;
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < kPerThread; ++r) {
        const int64_t j = ja + threadIdx.x + r * kThreads;
        if (j >= jb) break;
        const int64_t q = j / g.M;
        const int p = (int)(j - q * g.M);
        const int64_t first = q * g.L - g.width + kstart[p];             // input index of band tap 0
        const float* c = tab + p;
        float acc = 0.f;
        if (kStage) {
            const float* xs = sx + (first - s);
#pragma unroll 4
            for (int i = 0; i < g.T; ++i) acc = __fmaf_rn(__ldg(c + (size_t)i * g.M), xs[i], acc);
        } else {
#pragma unroll 4
            for (int i = 0; i < g.T; ++i) {
                const int64_t gi = first + i;
                const float v = gi >= b0 && gi < b1 ? __ldg(xb + (gi - b0)) : 0.f;
                acc = __fmaf_rn(__ldg(c + (size_t)i * g.M), v, acc);
            }
        }
        y[j - j0] = acc;
    }
}

void invalid(const std::string& s) { throw std::invalid_argument("resample: " + s); }

bool rate_ok(int r) { return r >= 1 && r <= (1 << 20) - 1; }

Geo geometry(int orig, int new_sr) {
    const int gd = std::gcd(orig, new_sr);
    Geo g{};
    g.L = orig / gd; g.M = new_sr / gd;
    const double base = (double)std::min(g.L, g.M) * 0.99;             // Python: min(L, M) * rolloff
    g.width = (int)std::ceil((double)kWidth * (double)g.L / base);     // math.ceil(6 * L / base)
    g.K = 2 * g.width + g.L;
    g.T = std::min(2 * g.width + 2, g.K);
    g.base = (float)base;
    g.scale = (float)(base / g.L);
    return g;
}

}  // namespace

struct Resampler::Impl {
    cudaStream_t st;
    int L = 0, M = 0;                        // the geometry `tab` / `kstart` hold
    Dev<float> tab, x, y;
    Dev<int> kstart, bad;
};

Resampler::Resampler(cudaStream_t st) : impl(new Impl()) {
    impl->st = st;
    CUDA_CHECK(cudaFuncSetAttribute(rs_resample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    kSmemFloats * (int)sizeof(float)));
}
Resampler::~Resampler() = default;

int64_t Resampler::out_len(int64_t n, int orig, int new_sr) {
    if (!rate_ok(orig) || !rate_ok(new_sr) || n < 0 || n > kMaxIn) return 0;
    if (orig == new_sr) return n;
    const Geo g = geometry(orig, new_sr);
    return ((int64_t)g.M * n + g.L - 1) / g.L;
}

int64_t Resampler::run(const float* wav, int64_t n, int orig, int new_sr, float* out, int64_t cap, int block_samples) {
    Impl& m = *impl;
    cudaStream_t st = m.st;
    if (!rate_ok(orig) || !rate_ok(new_sr)) invalid("sample rates must lie in 1 .. 1048575");
    if (n < 0 || (n > 0 && !wav)) invalid("no input");
    if (n > kMaxIn) invalid("input longer than 2^40 samples");
    if (block_samples < 1) invalid("block_samples < 1");
    const int64_t n_out = out_len(n, orig, new_sr);
    if (cap < n_out || (n_out > 0 && !out)) invalid("output buffer too small");
    if (n_out == 0) return 0;
    if (orig == new_sr) {                                // torchaudio returns the waveform itself
        std::memcpy(out, wav, (size_t)n * sizeof(float));
        return n;
    }

    const Geo g = geometry(orig, new_sr);
    m.bad.ensure(1);
    CUDA_CHECK(cudaMemsetAsync(m.bad.p, 0, sizeof(int), st));
    if (g.L != m.L || g.M != m.M) {                      // band table of this rate pair
        m.L = m.M = 0;
        m.kstart.ensure((size_t)g.M);
        m.tab.ensure((size_t)g.M * g.T);
        rs_band_kernel<<<nblk((size_t)g.M), 256, 0, st>>>(g, m.kstart.p, m.bad.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        rs_coef_kernel<<<std::min(nblk((size_t)g.M * g.T), 64 * sm_count()), 256, 0, st>>>(g, m.kstart.p, m.tab.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        int bad = 0;
        CUDA_CHECK(cudaMemcpyAsync(&bad, m.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (bad) throw std::runtime_error("resample: a filter band exceeds its table");
        m.L = g.L; m.M = g.M;
    }

    // the largest input span a CTA of kOutPerCta consecutive outputs reads
    const int64_t span = ((kOutPerCta - 1) / g.M + 1) * (int64_t)g.L + g.K;
    const bool stage = span <= kSmemFloats;
    const int64_t B = block_samples;
    m.x.ensure((size_t)std::min<int64_t>(n, B + g.K));
    m.y.ensure((size_t)std::min<int64_t>(n_out, B));
    for (int64_t j0 = 0; j0 < n_out;) {
        // outputs j0 .. j1-1: at most B, and their q = j / M within B / L of q0, so the input they read,
        // [q0 L - width, qb L + L + width), is at most B + 2 width + L samples
        const int64_t q0 = j0 / g.M;
        const int64_t j1 = std::min({n_out, j0 + B, (q0 + B / g.L + 1) * g.M});
        const int64_t qb = (j1 - 1) / g.M;
        const int64_t b0 = std::max<int64_t>(0, q0 * g.L - g.width), b1 = std::min<int64_t>(n, qb * g.L + g.L + g.width);
        CUDA_CHECK(cudaMemcpyAsync(m.x.p, wav + b0, (size_t)(b1 - b0) * sizeof(float), cudaMemcpyHostToDevice, st));
        rs_finite_kernel<<<std::min(nblk((size_t)(b1 - b0)), 4 * sm_count()), 256, 0, st>>>(m.x.p, b1 - b0, m.bad.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        const int grid = (int)((j1 - j0 + kOutPerCta - 1) / kOutPerCta);
        if (stage)
            rs_resample_kernel<true><<<grid, kThreads, (size_t)span * sizeof(float), st>>>(m.x.p, b0, b1, m.tab.p, m.kstart.p,
                                                                                      g, j0, j1 - j0, m.y.p);
        else
            rs_resample_kernel<false><<<grid, kThreads, 0, st>>>(m.x.p, b0, b1, m.tab.p, m.kstart.p, g, j0, j1 - j0, m.y.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        CUDA_CHECK(cudaMemcpyAsync(out + j0, m.y.p, (size_t)(j1 - j0) * sizeof(float), cudaMemcpyDeviceToHost, st));
        j0 = j1;
    }
    int bad = 0;
    CUDA_CHECK(cudaMemcpyAsync(&bad, m.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (bad) invalid("input is not finite");
    return n_out;
}

}  // namespace xtts
