// Reference-audio enhancer (see cond.h): the reference's EnhancedAudioProcessor.process (enhancer.py:34-153) on the
// GPU, stage by stage, then the 16-bit PCM round trip of the file it writes.
//   VAD        frame energies + a torchaudio mel log-sum, max-normalised, brought to one length with np.interp,
//              thresholded, the 0/1 decisions np.interp'ed to every sample and multiplied in
//   gating     librosa.stft (n_fft 2048, hop 512, periodic Hann, zero padding) -> per-bin noise floor = mean of the
//              k smallest magnitudes -> mask = clip(mag - floor*margin, 0) / (. + floor) -> librosa.istft
//   clarity    nan_to_num -> stft -> gain per bin -> istft
//   loudness   K-weighting (two RBJ biquads, fp64) -> 400 ms / 75 % blocks -> absolute and relative gates -> gain,
//              tanh, rint(x * 32767) / 32768
// The STFTs reuse cond.cu's framing, DFT basis and the fp32 NT GEMM.  fp32 IEEE arithmetic throughout the spectral
// stages (no fast-math): a bin whose noise floor is exactly 0 gates a silent frame to 0/0 = NaN as numpy does, and the
// inverse-DFT GEMM spreads it over the frame's samples; the clarity stage's nan_to_num then zeroes them.
#include <cfloat>
#include <cmath>
#include <map>
#include <stdexcept>

#include "cond.h"

namespace xtts {
namespace {

constexpr int kFft = 2048, kHop = 512, kBins = kFft / 2 + 1, kMels = 80;
constexpr int kMaxChunks = 1024;       // loudness scan: chunks per signal (one CTA scans the carries)
constexpr int kScanLevels = 10;        // log2(kMaxChunks)

// np.linspace(0, 1, n)[i]: i * (1 / (n - 1)), the last point exactly 1
__device__ __forceinline__ double lin01(int64_t i, int64_t n) {
    if (n <= 1) return 0.0;
    return i == n - 1 ? 1.0 : (double)i * (1.0 / (double)(n - 1));
}
// np.interp's bracket of x in np.linspace(0, 1, n): j with xp[j] <= x < xp[j+1] (j = n-1 at x == 1)
__device__ __forceinline__ int64_t bracket(double x, int64_t n) {
    if (n <= 1 || x >= 1.0) return n - 1;
    int64_t j = (int64_t)(x * (double)(n - 1));
    j = j < 0 ? 0 : (j > n - 2 ? n - 2 : j);
    while (j > 0 && lin01(j, n) > x) --j;
    while (j < n - 2 && lin01(j + 1, n) <= x) ++j;
    return j;
}
// np.interp(x, linspace(0, 1, n), f) for f given by a functor of the index
template <typename F>
__device__ __forceinline__ double interp01(double x, int64_t n, F f) {
    const int64_t j = bracket(x, n);
    if (j >= n - 1) return f(n - 1);
    const double x0 = lin01(j, n), x1 = lin01(j + 1, n), f0 = f(j), f1 = f(j + 1);
    return (f1 - f0) / (x1 - x0) * (x - x0) + f0;
}
// order-preserving float <-> uint map for atomicMax over signed floats
__device__ __forceinline__ unsigned f2ord(float v) { const unsigned u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : u | 0x80000000u; }
__device__ __forceinline__ float ord2f(unsigned u) { return __uint_as_float((u & 0x80000000u) ? u & 0x7fffffffu : ~u); }

__device__ __forceinline__ double block_sum_d(double v, double* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    double r = (lane < nw) ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    return r;
}

// ---------------------------------------------------------------------------------------------------- VAD
// energy[f] = sum of squares of frame f (librosa.util.frame, no padding); ord_max[0] = max over frames
__global__ void vad_energy_kernel(const float* __restrict__ x, int flen, int hop, float* __restrict__ energy,
                                  unsigned* __restrict__ ord_max) {
    __shared__ float red[32];
    const float* p = x + (size_t)blockIdx.x * hop;
    float s = 0.f;
    for (int i = threadIdx.x; i < flen; i += blockDim.x) s = fmaf(p[i], p[i], s);
    s = block_sum(s, red);
    if (threadIdx.x == 0) { energy[blockIdx.x] = s; atomicMax(ord_max, f2ord(s)); }
}
// lsum[t] = sum over mels of log(clamp(mel, 1e-5)), one warp per frame; ord_max[1] = max over frames
__global__ void mel_logsum_kernel(const float* __restrict__ mel, int T, float* __restrict__ lsum, unsigned* __restrict__ ord_max) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= T) return;
    float s = 0.f;
    for (int m = lane; m < kMels; m += 32) s += logf(fmaxf(mel[(size_t)t * kMels + m], 1e-5f));
    s = warp_sum(s);
    if (lane == 0) { lsum[t] = s; atomicMax(ord_max + 1, f2ord(s)); }
}
// Frame decisions |(e + s) / 2| > thr at the longer curve's length L, upsampled to every sample with np.interp and
// multiplied in: y[n] = x[n] * interp(n / (N-1), linspace(0, 1, L), decisions), in fp64 like numpy.
__global__ void vad_apply_kernel(const float* __restrict__ x, int64_t N, const float* __restrict__ energy, int Te,
                                 const float* __restrict__ lsum, int Tm, const unsigned* __restrict__ ord_max, double thr,
                                 float* __restrict__ y) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float emax = ord2f(ord_max[0]), smax = ord2f(ord_max[1]);
    const int64_t L = Te > Tm ? Te : Tm;
    auto e_at = [&](int64_t i) { return (double)(energy[i] / emax); };        // float32 division, as numpy
    auto s_at = [&](int64_t i) { return (double)(lsum[i] / smax); };
    auto keep = [&](int64_t j) {
        const double xj = lin01(j, L);
        const double e = Te == L ? e_at(j) : interp01(xj, Te, e_at);
        const double s = Tm == L ? s_at(j) : interp01(xj, Tm, s_at);
        return fabs((e + s) / 2) > thr ? 1.0 : 0.0;
    };
    const double m = interp01(lin01(n, N), L, keep);
    y[n] = (float)((double)x[n] * m);
}

// ---------------------------------------------------------------------------------------------------- gating / clarity
// magT[k][t] = |D[t][k]| (np.abs of the complex bin), transposed through a 32 x 32 tile so each bin's row is contiguous
__global__ void mag_t_kernel(const float* __restrict__ D, int T, float* __restrict__ magT) {
    __shared__ float tile[32][33];
    const int t0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int t = t0 + r, k = k0 + threadIdx.x;
        if (t < T && k < kBins) tile[r][threadIdx.x] = hypotf(D[(size_t)t * 2 * kBins + k], D[(size_t)t * 2 * kBins + kBins + k]);
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int k = k0 + r, t = t0 + threadIdx.x;
        if (t < T && k < kBins) magT[(size_t)k * T + t] = tile[threadIdx.x][r];
    }
}
// noise[k] = mean of the `kmin` smallest magnitudes of bin k over frames (all of them when there are fewer): an exact
// radix select on the float bits (non-negative floats order like their bit patterns), 8 bits per pass, then one sum.
__global__ void __launch_bounds__(256) noise_floor_kernel(const float* __restrict__ magT, int T, int kmin,
                                                          float* __restrict__ noise) {
    __shared__ unsigned hist[256];
    __shared__ unsigned s_prefix, s_rank;
    __shared__ double red[32];
    const float* m = magT + (size_t)blockIdx.x * T;
    const unsigned kk = (unsigned)min(kmin, T);
    unsigned prefix = 0, mask = 0, rank = kk;          // the rank-th smallest among values matching prefix under mask
    if (kk < (unsigned)T) {
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            for (int t = threadIdx.x; t < T; t += blockDim.x) {
                const unsigned u = __float_as_uint(m[t]);
                if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned c = 0, d = 0;
                while (c + hist[d] < rank) c += hist[d++];
                s_prefix = prefix | (d << shift); s_rank = rank - c;
            }
            __syncthreads();
            prefix = s_prefix; rank = s_rank; mask |= 255u << shift;
        }
    }
    // kk smallest = every value below the k-th one + `rank` copies of it
    double s = 0.0;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float v = m[t];
        if (kk == (unsigned)T || __float_as_uint(v) < prefix) s += (double)v;
    }
    s = block_sum_d(s, red);
    if (threadIdx.x == 0) {
        if (kk < (unsigned)T) s += (double)rank * (double)__uint_as_float(prefix);
        noise[blockIdx.x] = (float)(s / (double)kk);
    }
}
// In place on D [T][re 1025 | im 1025]: the gating mask (noise != null) and / or the clarity gain (gain != null).
// mask = max(mag - noise*margin, 0) / (that + noise): IEEE 0/0 = NaN is intended (see the file comment).
__global__ void spec_scale_kernel(float* __restrict__ D, int T, const float* __restrict__ noise, float margin,
                                  const float* __restrict__ gain) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)T * kBins) return;
    const int t = (int)(i / kBins), k = (int)(i % kBins);
    float* re = D + (size_t)t * 2 * kBins + k;
    float* im = re + kBins;
    float g = 1.f;
    if (noise) {
        const float nf = noise[k], a = fmaxf(hypotf(*re, *im) - nf * margin, 0.f);
        g = __fdiv_rn(a, a + nf);
    }
    if (gain) g *= gain[k];
    *re *= g; *im *= g;
}
// librosa.istft's overlap-add, gathered per output sample (no atomics): frames Y [T][2048] are already windowed
// (the inverse basis carries the window); divide by the squared-window sum where it exceeds float32 tiny; drop
// n_fft/2 samples at each end.  Frames are summed in ascending order, as librosa accumulates them.
__global__ void ola_kernel(const float* __restrict__ Y, int T, const float* __restrict__ win2, float* __restrict__ y,
                           int64_t nout) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nout) return;
    const int64_t m = s + kFft / 2;
    const int t_hi = (int)(m / kHop < T - 1 ? m / kHop : T - 1);
    const int t_lo = m >= kFft ? (int)((m - kFft) / kHop + 1) : 0;      // frames t with t*hop <= m < t*hop + n_fft
    float acc = 0.f, wss = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) {
        const int i = (int)(m - (int64_t)t * kHop);
        acc += Y[(size_t)t * kFft + i];
        wss += win2[i];
    }
    y[s] = wss > FLT_MIN ? acc / wss : acc;
}

// ---------------------------------------------------------------------------------------------------- loudness
// K-weighting = two transposed-direct-form-II biquads (scipy.signal.lfilter), fp64.  State (z0, z1, w0, w1).
struct KCoef { double b[3], a[3], c[3], d[3]; };
__device__ __forceinline__ double kw_step(const KCoef& k, double x, double* s) {
    const double y1 = k.b[0] * x + s[0];
    s[0] = k.b[1] * x - k.a[1] * y1 + s[1];
    s[1] = k.b[2] * x - k.a[2] * y1;
    const double y2 = k.c[0] * y1 + s[2];
    s[2] = k.c[1] * y1 - k.d[1] * y2 + s[3];
    s[3] = k.c[2] * y1 - k.d[2] * y2;
    return y2;
}
// Phase 1: every chunk of L samples from a zero state -> its end state
__global__ void kw_chunk_kernel(const float* __restrict__ x, int64_t N, int64_t L, int C, KCoef k, double* __restrict__ endst) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s[4] = {0, 0, 0, 0};
    const int64_t e = min(N, (int64_t)(c + 1) * L);
    for (int64_t n = (int64_t)c * L; n < e; ++n) kw_step(k, (double)x[n], s);
    for (int j = 0; j < 4; ++j) endst[(size_t)c * 4 + j] = s[j];
}
// Phase 2 (one CTA): true initial state of every chunk.  Inclusive Hillis-Steele scan of v_c = A^L v_{c-1} + e_c with
// the precomputed powers P_d = A^(L * 2^d); init[c] = v_{c-1}.
__global__ void __launch_bounds__(kMaxChunks) kw_carry_kernel(const double* __restrict__ endst, int C,
                                                              const double* __restrict__ P, double* __restrict__ init) {
    __shared__ double v[kMaxChunks][4];
    const int c = threadIdx.x;
    if (c < C) for (int j = 0; j < 4; ++j) v[c][j] = endst[(size_t)c * 4 + j];
    __syncthreads();
    for (int d = 0, off = 1; off < C; ++d, off <<= 1) {
        double r[4] = {0, 0, 0, 0};
        const bool act = c < C && c >= off;
        if (act) {
            const double* M = P + d * 16;
            for (int i = 0; i < 4; ++i) {
                double a = v[c][i];
                for (int j = 0; j < 4; ++j) a = fma(M[i * 4 + j], v[c - off][j], a);
                r[i] = a;
            }
        }
        __syncthreads();
        if (act) for (int i = 0; i < 4; ++i) v[c][i] = r[i];
        __syncthreads();
    }
    if (c < C) for (int j = 0; j < 4; ++j) init[(size_t)c * 4 + j] = c == 0 ? 0.0 : v[c - 1][j];
}
// Phase 3: every chunk again from its true initial state; csum[n] = sum of y^2 over the chunk up to and including n,
// ctot[c] = the chunk's total
__global__ void kw_apply_kernel(const float* __restrict__ x, int64_t N, int64_t L, int C, KCoef k,
                                const double* __restrict__ init, double* __restrict__ csum, double* __restrict__ ctot) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s[4];
    for (int j = 0; j < 4; ++j) s[j] = init[(size_t)c * 4 + j];
    double acc = 0.0;
    const int64_t e = min(N, (int64_t)(c + 1) * L);
    for (int64_t n = (int64_t)c * L; n < e; ++n) {
        const double y = kw_step(k, (double)x[n], s);
        acc = fma(y, y, acc);
        csum[n] = acc;
    }
    ctot[c] = acc;
}
// One CTA: chunk offsets, block energies z_j = (S(hi) - S(lo)) / (0.4 sr) from the prefix sums, the -70 LUFS absolute
// and -10 LU relative gates, the integrated loudness and the gain.  out[0] = LUFS, out[1] = linear gain.
__global__ void __launch_bounds__(kMaxChunks) loudness_gate_kernel(
        const double* __restrict__ csum, const double* __restrict__ ctot, int64_t L, int C, const int64_t* __restrict__ lo,
        const int64_t* __restrict__ hi, int nblocks, double scale, double target, double* __restrict__ z, double* __restrict__ out) {
    __shared__ double off[kMaxChunks];
    __shared__ double red[32];
    const int c = threadIdx.x;
    double v = c < C ? ctot[c] : 0.0;
    if (c < kMaxChunks) off[c] = v;
    __syncthreads();
    for (int o = 1; o < C; o <<= 1) {                 // inclusive scan of the chunk totals
        const double a = (c < C && c >= o) ? off[c - o] : 0.0;
        __syncthreads();
        if (c < C) off[c] += a;
        __syncthreads();
    }
    auto S = [&](int64_t m) -> double {               // sum of y^2 over samples [0, m)
        if (m <= 0) return 0.0;
        const int64_t ch = (m - 1) / L;
        return (ch > 0 ? off[ch - 1] : 0.0) + csum[m - 1];
    };
    double s1 = 0.0, n1 = 0.0;
    for (int j = c; j < nblocks; j += blockDim.x) {
        const double zj = scale * (S(hi[j]) - S(lo[j]));
        z[j] = zj;
        if (-0.691 + 10.0 * log10(zj) >= -70.0) { s1 += zj; n1 += 1.0; }
    }
    s1 = block_sum_d(s1, red); n1 = block_sum_d(n1, red);
    const double rel = -0.691 + 10.0 * log10(s1 / n1) - 10.0;     // NaN when nothing passes: then nothing passes below
    __syncthreads();
    double s2 = 0.0, n2 = 0.0;
    for (int j = c; j < nblocks; j += blockDim.x) {
        const double lj = -0.691 + 10.0 * log10(z[j]);
        if (lj > rel && lj >= -70.0) { s2 += z[j]; n2 += 1.0; }
    }
    s2 = block_sum_d(s2, red); n2 = block_sum_d(n2, red);
    if (c == 0) {
        const double lufs = -0.691 + 10.0 * log10(n2 > 0 ? s2 / n2 : 0.0);
        out[0] = lufs;
        out[1] = pow(10.0, (target - lufs) / 20.0);
    }
}
// Last pass: optional loudness gain + tanh, then the 16-bit PCM write / read; flags a non-finite result
__global__ void finish_kernel(const float* __restrict__ x, int64_t N, const double* __restrict__ lg, float* __restrict__ y,
                              int* __restrict__ bad) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    double v = x[n];
    if (lg) v = tanh(v * lg[1]);
    if (!isfinite(v)) { atomicOr(bad, 1); v = 0.0; }
    const double q = fmin(fmax(rint(v * 32767.0), -32768.0), 32767.0);
    y[n] = (float)(q / 32768.0);
}

// pyloudnorm's RBJ biquads for K-weighting at `rate`, normalised by a0
void rbj(double rate, bool shelf, double* b, double* a) {
    const double G = shelf ? 4.0 : 0.0, Q = shelf ? 1.0 / std::sqrt(2.0) : 0.5, fc = shelf ? 1500.0 : 38.0;
    const double A = std::pow(10.0, G / 40.0), w0 = 2.0 * kPi * (fc / rate), alpha = std::sin(w0) / (2.0 * Q);
    const double cw = std::cos(w0), sA = std::sqrt(A);
    double B[3], Aa[3];
    if (shelf) {
        B[0] = A * ((A + 1) + (A - 1) * cw + 2 * sA * alpha);
        B[1] = -2 * A * ((A - 1) + (A + 1) * cw);
        B[2] = A * ((A + 1) + (A - 1) * cw - 2 * sA * alpha);
        Aa[0] = (A + 1) - (A - 1) * cw + 2 * sA * alpha;
        Aa[1] = 2 * ((A - 1) - (A + 1) * cw);
        Aa[2] = (A + 1) - (A - 1) * cw - 2 * sA * alpha;
    } else {
        B[0] = (1 + cw) / 2; B[1] = -(1 + cw); B[2] = (1 + cw) / 2;
        Aa[0] = 1 + alpha; Aa[1] = -2 * cw; Aa[2] = 1 - alpha;
    }
    for (int i = 0; i < 3; ++i) { b[i] = B[i] / Aa[0]; a[i] = Aa[i] / Aa[0]; }
}
void matmul4(const double* X, const double* Y, double* Z) {
    double r[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += X[i * 4 + k] * Y[k * 4 + j]; r[i * 4 + j] = s; }
    std::copy(r, r + 16, Z);
}
void invalid(const std::string& s) { throw std::invalid_argument("enhance: " + s); }

}  // namespace

struct Enhancer::Impl {
    cudaStream_t st;
    Dev<float> hann, win2, basis, ibasis, gain, x, y, F, D, P, mel, magT, noise, energy, lsum;
    std::map<int, Dev<float>> fb;                    // mel filterbank per sample rate
    Dev<unsigned> ordmax;
    Dev<double> kp, endst, init, csum, ctot, z, lres;
    Dev<int64_t> blo, bhi;
    Dev<int> bad;

    void lazy_init() {
        if (basis.p) return;
        std::vector<float> w(kFft), w2(kFft);
        std::vector<double> wd(kFft);
        for (int i = 0; i < kFft; ++i) {
            wd[i] = 0.5 - 0.5 * std::cos(2.0 * kPi * i / kFft);         // periodic Hann
            w[i] = (float)wd[i]; w2[i] = (float)(wd[i] * wd[i]);
        }
        hann.up(w, st); win2.up(w2, st);
        basis.up(dft_basis(kFft, kFft, 0), st);
        // irfft x window as an NT GEMM operand [2048][re 1025 | im 1025]: (1/N) c_k (Re cos - Im sin), c_k = 1 at DC
        // and Nyquist (whose imaginary parts irfft ignores), 2 elsewhere
        std::vector<float> ib((size_t)kFft * 2 * kBins);
        for (int i = 0; i < kFft; ++i)
            for (int k = 0; k < kBins; ++k) {
                const double a = 2.0 * kPi * (double)k * (double)i / kFft, ck = (k == 0 || k == kFft / 2) ? 1.0 : 2.0;
                ib[(size_t)i * 2 * kBins + k] = (float)(wd[i] * ck * std::cos(a) / kFft);
                ib[(size_t)i * 2 * kBins + kBins + k] = (k == 0 || k == kFft / 2) ? 0.f : (float)(-wd[i] * ck * std::sin(a) / kFft);
            }
        ibasis.up(ib, st);
        ordmax.alloc(2); bad.alloc(1); lres.alloc(2); noise.alloc(kBins); gain.alloc(kBins); kp.alloc(16 * kScanLevels);
    }
    // D [T][2050] = DFT of the zero-padded (nan_to_num'ed) x, T = 1 + N / 512
    int stft(const float* xs, int64_t N) {
        const int T = (int)(1 + N / kHop);
        F.ensure((size_t)T * kFft); D.ensure((size_t)T * 2 * kBins);
        frame_window_kernel<<<T, 256, 0, st>>>(xs, (int)N, hann.p, kFft, kHop, 0, kFft / 2, PAD_ZERO, F.p, T);
        COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(F.p, basis.p, nullptr, nullptr, D.p, T, 2 * kBins, kFft, 0, st);
        return T;
    }
    // inverse of D [T] -> ys, 512 * (T - 1) samples
    void istft(int T, float* ys) {
        launch_gemm_f32(D.p, ibasis.p, nullptr, nullptr, F.p, T, kFft, 2 * kBins, 0, st);
        const int64_t nout = (int64_t)kHop * (T - 1);
        if (nout > 0) { ola_kernel<<<nblk((size_t)nout), 256, 0, st>>>(F.p, T, win2.p, ys, nout); COUNT_LAUNCH(); KERNEL_CHECK(); }
    }
    void vad(const float* xs, int64_t N, const xtts_enhance_config& c, float* ys) {
        const int fl = c.vad_frame_length, fh = fl / 2;
        const int Te = (int)(1 + (N - fl) / fh), Tm = (int)(1 + N / kHop);
        energy.ensure(Te); lsum.ensure(Tm);
        CUDA_CHECK(cudaMemsetAsync(ordmax.p, 0, 2 * sizeof(unsigned), st));
        vad_energy_kernel<<<Te, 256, 0, st>>>(xs, fl, fh, energy.p, ordmax.p); COUNT_LAUNCH(); KERNEL_CHECK();
        // torchaudio MelSpectrogram(sr, n_fft 2048, hop 512, n_mels 80): reflect padding, power 2, htk, no norm
        auto it = fb.find(c.sample_rate);
        if (it == fb.end()) {
            it = fb.emplace(std::piecewise_construct, std::forward_as_tuple(c.sample_rate), std::forward_as_tuple()).first;
            it->second.up(mel_fb_t(kBins, 0.0, (double)(c.sample_rate / 2), kMels, c.sample_rate, false), st);
        }
        F.ensure((size_t)Tm * kFft); D.ensure((size_t)Tm * 2 * kBins); P.ensure((size_t)Tm * kBins); mel.ensure((size_t)Tm * kMels);
        frame_window_kernel<<<Tm, 256, 0, st>>>(xs, (int)N, hann.p, kFft, kHop, 0, kFft / 2, PAD_REFLECT, F.p, Tm);
        COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(F.p, basis.p, nullptr, nullptr, D.p, Tm, 2 * kBins, kFft, 0, st);
        power_kernel<<<nblk((size_t)Tm * kBins), 256, 0, st>>>(D.p, P.p, Tm, kBins); COUNT_LAUNCH(); KERNEL_CHECK();
        launch_gemm_f32(P.p, it->second.p, nullptr, nullptr, mel.p, Tm, kMels, kBins, 0, st);
        mel_logsum_kernel<<<nblk((size_t)Tm * 32), 256, 0, st>>>(mel.p, Tm, lsum.p, ordmax.p); COUNT_LAUNCH(); KERNEL_CHECK();
        vad_apply_kernel<<<nblk((size_t)N), 256, 0, st>>>(xs, N, energy.p, Te, lsum.p, Tm, ordmax.p, (double)c.vad_threshold, ys);
        COUNT_LAUNCH(); KERNEL_CHECK();
    }
    // spectral gating (noise floor) and / or clarity (gain) over one STFT; returns the new length
    int64_t spectral(const float* xs, int64_t N, const xtts_enhance_config& c, bool gate, float* ys) {
        const int T = stft(xs, N);
        if (gate) {
            magT.ensure((size_t)T * kBins);
            mag_t_kernel<<<dim3(ceil_div(T, 32), ceil_div(kBins, 32)), dim3(32, 8), 0, st>>>(D.p, T, magT.p);
            COUNT_LAUNCH(); KERNEL_CHECK();
            noise_floor_kernel<<<kBins, 256, 0, st>>>(magT.p, T, c.noise_reduce_frames, noise.p); COUNT_LAUNCH(); KERNEL_CHECK();
        }
        spec_scale_kernel<<<nblk((size_t)T * kBins), 256, 0, st>>>(D.p, T, gate ? noise.p : nullptr, c.noise_reduce_margin,
                                                                    gate ? nullptr : gain.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        istft(T, ys);
        return (int64_t)kHop * (T - 1);
    }
    // integrated loudness -> lres = {LUFS, gain}
    void loudness(const float* xs, int64_t N, const xtts_enhance_config& c) {
        const double sr = c.sample_rate;
        KCoef k;
        rbj(sr, true, k.b, k.a); rbj(sr, false, k.c, k.d);
        const int64_t L = std::max<int64_t>(256, (N + kMaxChunks - 1) / kMaxChunks);
        const int C = (int)((N + L - 1) / L);
        // one zero-input step of the cascade as a 4 x 4 matrix A (columns = images of the unit states), then A^L,
        // squared once per scan level
        double A[16], M[16], Pw[16 * kScanLevels];
        for (int j = 0; j < 4; ++j) {
            double s[4] = {0, 0, 0, 0}; s[j] = 1;
            const double y1 = s[0];
            double r[4];
            r[0] = -k.a[1] * y1 + s[1]; r[1] = -k.a[2] * y1;
            const double y2 = k.c[0] * y1 + s[2];
            r[2] = k.c[1] * y1 - k.d[1] * y2 + s[3]; r[3] = k.c[2] * y1 - k.d[2] * y2;
            for (int i = 0; i < 4; ++i) A[i * 4 + j] = r[i];
        }
        for (int i = 0; i < 16; ++i) M[i] = (i % 5 == 0) ? 1.0 : 0.0;
        for (int64_t e = L; ; ) {                         // M = A^L by binary powering (A is consumed)
            if (e & 1) matmul4(M, A, M);
            e >>= 1;
            if (!e) break;
            matmul4(A, A, A);
        }
        std::copy(M, M + 16, Pw);
        for (int d = 1; d < kScanLevels; ++d) matmul4(Pw + (d - 1) * 16, Pw + (d - 1) * 16, Pw + d * 16);
        // pyloudnorm's blocks: count from np.round, bounds by int() truncation, clipped to the signal
        const double Tg = 0.4, step = 1.0 - 0.75;
        const int nb = (int)std::nearbyint((((double)N / sr - Tg) / (Tg * step))) + 1;
        std::vector<int64_t> lo(nb), hi(nb);
        for (int j = 0; j < nb; ++j) {
            lo[j] = std::min<int64_t>(N, (int64_t)(Tg * (j * step) * sr));
            hi[j] = std::min<int64_t>(N, (int64_t)(Tg * (j * step + 1) * sr));
        }
        CUDA_CHECK(cudaMemcpyAsync(kp.p, Pw, sizeof(Pw), cudaMemcpyHostToDevice, st));
        blo.up(lo, st); bhi.up(hi, st);
        endst.ensure((size_t)C * 4); init.ensure((size_t)C * 4); csum.ensure((size_t)N); ctot.ensure(C); z.ensure(nb);
        kw_chunk_kernel<<<nblk(C, 128), 128, 0, st>>>(xs, N, L, C, k, endst.p); COUNT_LAUNCH(); KERNEL_CHECK();
        kw_carry_kernel<<<1, kMaxChunks, 0, st>>>(endst.p, C, kp.p, init.p); COUNT_LAUNCH(); KERNEL_CHECK();
        kw_apply_kernel<<<nblk(C, 128), 128, 0, st>>>(xs, N, L, C, k, init.p, csum.p, ctot.p); COUNT_LAUNCH(); KERNEL_CHECK();
        loudness_gate_kernel<<<1, kMaxChunks, 0, st>>>(csum.p, ctot.p, L, C, blo.p, bhi.p, nb, 1.0 / (Tg * sr),
                                                      (double)c.target_lufs, z.p, lres.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
    }
};

Enhancer::Enhancer(cudaStream_t st) : impl(new Impl()) { impl->st = st; }
Enhancer::~Enhancer() = default;

int64_t Enhancer::out_len(int64_t n, const xtts_enhance_config& c) {
    return (c.remove_noise || c.enhance_speech) ? (int64_t)kHop * (n / kHop) : n;
}

int64_t Enhancer::run(const float* wav, int64_t n, const xtts_enhance_config& c, float* out, int64_t cap) {
    Impl& m = *impl;
    cudaStream_t st = m.st;
    // ---- configuration and the reference's own failure conditions (librosa.util.frame, pyloudnorm's block check)
    if (c.sample_rate < 1000 || c.sample_rate > 768000) invalid("sample_rate out of range [1000, 768000]");
    if (c.vad_frame_length < 2) invalid("vad_frame_length < 2");
    if (c.noise_reduce_frames < 1) invalid("noise_reduce_frames < 1");
    if (!std::isfinite(c.vad_threshold) || !std::isfinite(c.noise_reduce_margin) || !std::isfinite(c.enhance_amount) ||
        !std::isfinite(c.target_lufs))
        invalid("non-finite parameter");
    if (!wav || n < 1) invalid("empty input");
    if (n > ((int64_t)1 << 28)) invalid("input longer than 2^28 samples");
    for (int64_t i = 0; i < n; ++i)
        if (!std::isfinite(wav[i])) invalid("input is not finite");
    if (c.trim_silence && n < c.vad_frame_length) invalid("input shorter than vad_frame_length");
    if (c.trim_silence && n <= kFft / 2) invalid("input too short for the VAD mel spectrogram");
    const int64_t n_out = out_len(n, c);
    if (c.normalize && (double)n_out < 0.4 * (double)c.sample_rate) invalid("audio shorter than one 400 ms loudness block");
    if (cap < n_out || (!out && n_out > 0)) invalid("output buffer too small");

    m.lazy_init();
    m.x.ensure((size_t)n); m.y.ensure((size_t)n);
    CUDA_CHECK(cudaMemcpyAsync(m.x.p, wav, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
    float* a = m.x.p; float* b = m.y.p;
    int64_t N = n;
    if (c.trim_silence) { m.vad(a, N, c, b); std::swap(a, b); }
    if (c.remove_noise) { N = m.spectral(a, N, c, true, b); std::swap(a, b); }
    if (c.enhance_speech) {
        // 1 + amount * exp(-|f - 2000| / 1000) with f = np.fft.fftfreq(1025, 1 / sr): the reference's bin "frequencies"
        // are spaced sr / 1025 and negative above bin 512 (not the rfft bins' k * sr / 2048).  Kept bit-for-bit.
        std::vector<float> g(kBins);
        const double val = 1.0 / (kBins * (1.0 / c.sample_rate));
        for (int k = 0; k < kBins; ++k) {
            const double f = (k <= kBins / 2 ? k : k - kBins) * val;
            g[k] = (float)(1.0 + std::exp(-std::fabs(f - 2000.0) / 1000.0) * (double)c.enhance_amount);
        }
        CUDA_CHECK(cudaMemcpyAsync(m.gain.p, g.data(), kBins * sizeof(float), cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));       // g is a host temporary
        N = m.spectral(a, N, c, false, b); std::swap(a, b);
    }
    if (c.normalize) m.loudness(a, N, c);
    CUDA_CHECK(cudaMemsetAsync(m.bad.p, 0, sizeof(int), st));
    if (N > 0) {
        finish_kernel<<<nblk((size_t)N), 256, 0, st>>>(a, N, c.normalize ? m.lres.p : nullptr, b, m.bad.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        CUDA_CHECK(cudaMemcpyAsync(out, b, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    int bad = 0;
    double lres[2] = {0, 0};
    CUDA_CHECK(cudaMemcpyAsync(&bad, m.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (c.normalize) CUDA_CHECK(cudaMemcpyAsync(lres, m.lres.p, sizeof(lres), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (bad || !std::isfinite(lres[0]) || !std::isfinite(lres[1])) invalid("the enhanced audio is not finite");
    return N;
}

}  // namespace xtts
