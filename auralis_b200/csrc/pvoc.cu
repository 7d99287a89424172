// Phase vocoder (see cond.h): the body of the reference's TTSOutput.change_speed (output.py:40-92) on the GPU,
//   librosa.stft(n_fft 2048, hop 512) -> librosa.phase_vocoder(rate) -> librosa.istft -> librosa.util.normalize(norm=inf)
// with librosa 0.10's arithmetic under NumPy's NEP 50 promotion:
//   time_steps  t * rate (float64), T_out = ceil(T / rate) output frames, T = 1 + n / 512 input frames
//   per step    mag = (1 - alpha)|c0| + alpha|c1| (float64), out[t] = (cos, sin)(phase_acc) in float32 times mag, stored
//               as complex64; dphase = f64(angle(c1) - angle(c0)) - phi_advance, wrapped by - 2 pi round(dphase / 2 pi);
//               phase_acc (float32) = f32(f64(phase_acc) + (phi_advance + dphase))
// The spectrum is padded with two zero columns, so input frames >= T read as 0.  Every fp64 step is written with _rn
// intrinsics, which the compiler never contracts into an FMA; fp32 IEEE arithmetic elsewhere, no fast-math, no TF32.
//
// Blocked: each block is at most B output frames (engine option "pvoc_block_frames") and at most B + 2 input frames.
// The forward STFT runs over the block's input frames only; phase_acc [1025] and the last three inverse-DFT frames
// (the overlap-add tail) carry over to the next block.  Every bin's accumulation is one sequence, every GEMM row is
// computed alone and every sample sums its <= 4 frames in frame order, so the result is the same for every B.  The
// waveform itself sits whole on the device until it is peak-normalised.
#include <cfloat>
#include <cmath>
#include <stdexcept>

#include "cond.h"

namespace xtts {
namespace {

constexpr int kFft = 2048, kHop = 512, kBins = kFft / 2 + 1;
constexpr double kTwoPi = 2.0 * kPi;          // numpy's 2.0 * np.pi

// mag[r][k] = |D|, ang[r][k] = angle(D) of input frame j0 + r, each in fp64 and rounded to fp32 (numpy's hypotf /
// atan2f, correctly rounded); frames >= T are librosa's zero padding: 0, 0.  D [rows][re 1025 | im 1025].
__global__ void pv_polar_kernel(const float* __restrict__ D, int rows, int64_t j0, int64_t T, float* __restrict__ mag,
                                float* __restrict__ ang) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * kBins) return;
    const int r = (int)(i / kBins), k = (int)(i % kBins);
    float m = 0.f, a = 0.f;
    if (j0 + r < T) {
        const double re = D[(size_t)r * 2 * kBins + k], im = D[(size_t)r * 2 * kBins + kBins + k];
        m = (float)sqrt(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));      // both squares exact in fp64
        a = (float)atan2(im, re);
    }
    mag[i] = m; ang[i] = a;
}

// dph[r][k]: the wrapped phase advance from input frame j0 + r to j0 + r + 1.  Depends on the input frame only, so it
// is computed for every frame in parallel.
__global__ void pv_dphase_kernel(const float* __restrict__ ang, int rows, const double* __restrict__ phi,
                                 double* __restrict__ dph) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * kBins) return;
    const int k = (int)(i % kBins);
    const float d32 = __fsub_rn(ang[i + kBins], ang[i]);                    // float32 - float32 stays float32
    const double d = __dsub_rn((double)d32, phi[k]);
    dph[i] = __dsub_rn(d, __dmul_rn(kTwoPi, rint(__ddiv_rn(d, kTwoPi))));   // np.round: half to even
}

// One thread per bin walks output frames t0 .. t0 + nt - 1 in order: phase[i][k] = the accumulator before step t0 + i,
// then acc = f32(f64(acc) + (phi + dph[int((t0 + i) * rate)])).  The per-step float32 rounding is numpy's, so the walk
// cannot be turned into a scan.  acc[k] carries the accumulator between blocks; the first block starts it at angle(D[0]).
__global__ void pv_accumulate_kernel(const double* __restrict__ dph, const float* __restrict__ ang, int64_t j0, int64_t t0,
                                     int nt, double rate, const double* __restrict__ phi, float* __restrict__ acc,
                                     float* __restrict__ phase) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= kBins) return;
    float a = t0 == 0 ? ang[k] : acc[k];                                     // (j0 == 0 in the first block)
    const double pk = phi[k];
#pragma unroll 4
    for (int i = 0; i < nt; ++i) {
        phase[(size_t)i * kBins + k] = a;
        const int64_t j = (int64_t)__dmul_rn((double)(t0 + i), rate);
        a = (float)__dadd_rn((double)a, __dadd_rn(pk, dph[(size_t)(j - j0) * kBins + k]));
    }
    acc[k] = a;
}

// Output frames t0 .. t0 + nt - 1 as the inverse-DFT GEMM's A operand S [nt][re 1025 | im 1025]:
// mag * (cos, sin)(phase), the cosine and sine rounded to float32, each product formed in fp64 and rounded to float32.
__global__ void pv_stretch_kernel(const float* __restrict__ mag, int64_t j0, int64_t t0, int nt, double rate,
                                  const float* __restrict__ phase, float* __restrict__ S) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)nt * kBins) return;
    const int r = (int)(i / kBins), k = (int)(i % kBins);
    const double step = __dmul_rn((double)(t0 + r), rate);
    const int64_t j = (int64_t)step;
    const double alpha = __dsub_rn(step, (double)j);                         // np.mod(step, 1.0), exact
    const float* m = mag + (size_t)(j - j0) * kBins + k;
    const double mg = __dadd_rn(__dmul_rn(__dsub_rn(1.0, alpha), (double)m[0]), __dmul_rn(alpha, (double)m[kBins]));
    const double p = (double)phase[i];
    const float c = (float)cos(p), s = (float)sin(p);
    S[(size_t)r * 2 * kBins + k] = (float)__dmul_rn((double)c, mg);
    S[(size_t)r * 2 * kBins + kBins + k] = (float)__dmul_rn((double)s, mg);
}

// peak = max |y| as its bit pattern (non-negative floats order like their bits: the order-preserving map enhance.cu
// uses, restricted to |y|); bad |= a non-finite sample
__global__ void pv_peak_kernel(const float* __restrict__ y, int64_t n, unsigned* __restrict__ peak, int* __restrict__ bad) {
    unsigned m = 0;
    int nf = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = fabsf(y[i]);
        if (isfinite(v)) m = max(m, __float_as_uint(v)); else nf = 1;
    }
    m = __reduce_max_sync(0xffffffffu, m);
    nf = __reduce_or_sync(0xffffffffu, (unsigned)nf);
    if ((threadIdx.x & 31) == 0) {
        atomicMax(peak, m);
        if (nf) atomicOr(bad, 1);
    }
}
// y /= peak as an IEEE division (librosa divides by the float64 max and stores float32: the same correctly rounded
// quotient); a peak below float32 tiny leaves y as it is
__global__ void pv_normalize_kernel(float* __restrict__ y, int64_t n, const unsigned* __restrict__ peak) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float mx = __uint_as_float(*peak);
    if (mx >= FLT_MIN) y[i] = __fdiv_rn(y[i], mx);
}

void invalid(const std::string& s) { throw std::invalid_argument("change_speed: " + s); }

constexpr int64_t kMaxIn = (int64_t)1 << 30;           // samples in (frame offsets stay in int)
constexpr int64_t kMaxOutFrames = (int64_t)1 << 22;   // 2^31 samples out

int64_t out_frames(int64_t n, double rate) {
    return (int64_t)std::ceil((double)(1 + n / kHop) / rate);
}

}  // namespace

struct PhaseVocoder::Impl {
    cudaStream_t st;
    DBuf<float> hann, win2, basis, ibasis, x, y, F, D, mag, ang, phase, Y, acc;
    DBuf<double> phi, dph;
    DBuf<unsigned> peak;
    DBuf<int> bad;

    void lazy_init() {
        if (basis.p) return;
        std::vector<float> w, w2, ib;
        stft_tables(w, w2, ib);
        hann.up(w, st); win2.up(w2, st);
        basis.up(dft_basis(kFft, kFft, 0), st);
        ibasis.up(ib, st);
        // phi_advance = hop * np.fft.rfftfreq(n_fft, d = 1 / (2 pi)) = 512 * (k * (1 / (n_fft * d)))
        const double val = 1.0 / ((double)kFft * (1.0 / kTwoPi));
        std::vector<double> p(kBins);
        for (int k = 0; k < kBins; ++k) p[k] = (double)kHop * ((double)k * val);
        phi.up(p, st);
        acc.alloc(kBins); peak.alloc(1); bad.alloc(1);
    }
};

PhaseVocoder::PhaseVocoder(cudaStream_t st) : impl(new Impl()) { impl->st = st; }
PhaseVocoder::~PhaseVocoder() = default;

int64_t PhaseVocoder::out_len(int64_t n, double rate) {
    if (!std::isfinite(rate) || rate <= 0 || n < 0) return 0;
    const double f = std::ceil((double)(1 + n / kHop) / rate);
    return f > (double)kMaxOutFrames ? 0 : (int64_t)kHop * ((int64_t)f - 1);
}

int64_t PhaseVocoder::run(const float* wav, int64_t n, double rate, float* out, int64_t cap, int block_frames) {
    Impl& m = *impl;
    cudaStream_t st = m.st;
    if (!std::isfinite(rate) || rate <= 0) invalid("the speed factor must be finite and positive");
    if (n < 0 || (n > 0 && !wav)) invalid("no input");
    if (n > kMaxIn) invalid("input longer than 2^30 samples");
    if (block_frames < 1) invalid("block_frames < 1");
    for (int64_t i = 0; i < n; ++i)
        if (!std::isfinite(wav[i])) invalid("input is not finite");
    const int64_t T = 1 + n / kHop;
    if ((double)T / rate > (double)kMaxOutFrames) invalid("result longer than 2^31 samples");
    const int64_t To = out_frames(n, rate);
    const int64_t n_out = (int64_t)kHop * (To - 1);
    if (n_out <= 0) invalid("empty result (the speed factor leaves one STFT frame)");
    if (cap < n_out || !out) invalid("output buffer too small");

    m.lazy_init();
    const int B = block_frames, J = block_frames + 2;                        // output / input frames per block
    m.x.ensure((size_t)std::max<int64_t>(n, 1)); m.y.ensure((size_t)n_out);
    m.F.ensure((size_t)J * kFft); m.D.ensure((size_t)J * 2 * kBins);
    m.mag.ensure((size_t)J * kBins); m.ang.ensure((size_t)J * kBins); m.dph.ensure((size_t)J * kBins);
    m.phase.ensure((size_t)B * kBins); m.Y.ensure((size_t)(B + 3) * kFft);
    if (n > 0) CUDA_CHECK(cudaMemcpyAsync(m.x.p, wav, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));

    auto jlast = [&](int64_t t) { return (int64_t)((double)t * rate); };     // int(time_steps[t])
    for (int64_t t0 = 0; t0 < To;) {
        const int64_t j0 = jlast(t0);
        // the longest run of output frames t0 .. t1-1 within B frames whose input frames j0 .. jlast(t1-1)+1 fit in J
        int64_t lo = t0 + 1, hi = std::min<int64_t>(To, t0 + B);
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) / 2;
            if (jlast(mid - 1) + 2 - j0 <= J) lo = mid; else hi = mid - 1;
        }
        const int64_t t1 = lo;
        const int nt = (int)(t1 - t0), rows = (int)(jlast(t1 - 1) + 2 - j0);
        const int real = (int)std::max<int64_t>(0, std::min<int64_t>(rows, T - j0));   // frames of the signal itself
        if (real > 0) {
            frame_window_kernel<<<real, 256, 0, st>>>(m.x.p, (int)n, m.hann.p, kFft, kHop, (int)(j0 * kHop), kFft / 2,
                                                      PAD_ZERO, m.F.p, real);
            COUNT_LAUNCH(); KERNEL_CHECK();
            launch_gemm_f32(m.F.p, m.basis.p, nullptr, nullptr, m.D.p, real, 2 * kBins, kFft, 0, st);
        }
        pv_polar_kernel<<<nblk((size_t)rows * kBins), 256, 0, st>>>(m.D.p, rows, j0, T, m.mag.p, m.ang.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        pv_dphase_kernel<<<nblk((size_t)(rows - 1) * kBins), 256, 0, st>>>(m.ang.p, rows - 1, m.phi.p, m.dph.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        pv_accumulate_kernel<<<nblk(kBins, 128), 128, 0, st>>>(m.dph.p, m.ang.p, j0, t0, nt, rate, m.phi.p, m.acc.p, m.phase.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        pv_stretch_kernel<<<nblk((size_t)nt * kBins), 256, 0, st>>>(m.mag.p, j0, t0, nt, rate, m.phase.p, m.D.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        // rows 0..2 of Y hold frames t0-3 .. t0-1 (the previous block's tail), rows 3.. this block's frames
        launch_gemm_f32(m.D.p, m.ibasis.p, nullptr, nullptr, m.Y.p + (size_t)3 * kFft, nt, kFft, 2 * kBins, 0, st);
        // samples m in [t0 * 512, t1 * 512) have all their frames in Y (the last block: up to the end of the signal)
        const int64_t mA = std::max<int64_t>(kFft / 2, t0 * kHop), mB = t1 == To ? (int64_t)kHop * To + kHop : t1 * kHop;
        if (mB > mA) {
            ola_kernel<<<nblk((size_t)(mB - mA)), 256, 0, st>>>(m.Y.p, (int)(t0 - 3), (int)To, m.win2.p,
                                                                 m.y.p + (mA - kFft / 2), mA, mB - mA);
            COUNT_LAUNCH(); KERNEL_CHECK();
        }
        for (int r = 0; r < 3; ++r)                       // row by row, in order: rows nt + r and r never overlap
            CUDA_CHECK(cudaMemcpyAsync(m.Y.p + (size_t)r * kFft, m.Y.p + (size_t)(nt + r) * kFft, kFft * sizeof(float),
                                       cudaMemcpyDeviceToDevice, st));
        t0 = t1;
    }

    CUDA_CHECK(cudaMemsetAsync(m.peak.p, 0, sizeof(unsigned), st));
    CUDA_CHECK(cudaMemsetAsync(m.bad.p, 0, sizeof(int), st));
    pv_peak_kernel<<<std::min(nblk((size_t)n_out), 4 * sm_count()), 256, 0, st>>>(m.y.p, n_out, m.peak.p, m.bad.p);
    COUNT_LAUNCH(); KERNEL_CHECK();
    pv_normalize_kernel<<<nblk((size_t)n_out), 256, 0, st>>>(m.y.p, n_out, m.peak.p);
    COUNT_LAUNCH(); KERNEL_CHECK();
    CUDA_CHECK(cudaMemcpyAsync(out, m.y.p, (size_t)n_out * sizeof(float), cudaMemcpyDeviceToHost, st));
    int bad = 0;
    CUDA_CHECK(cudaMemcpyAsync(&bad, m.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (bad) invalid("the stretched audio is not finite");
    return n_out;
}

}  // namespace xtts
