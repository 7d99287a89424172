// Speaker conditioning on the GPU: reference wav -> (GPT conditioning latents [32,H], d-vector [proj]).
// Replaces get_conditioning_latents (XTTSv2.py:409-468): wav_to_mel_cloning -> ConditioningEncoder ->
// PerceiverResampler (per 4 s piece, averaged) and ResNetSpeakerEncoder (SURVEY.md §2.4 K18-K21, §8a a15-a16).
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/xtts_b200.h"
#include "kernels.h"

namespace xtts {

constexpr double kPi = 3.14159265358979323846;

inline int nblk(size_t n, int t = 256) { return (int)((n + t - 1) / t); }

// ---- STFT front-end shared by the conditioner (cond.cu) and the reference enhancer (enhance.cu)
enum : int { PAD_REFLECT = 0, PAD_ZERO = 1 };
// F[t][i] = win[i] * xp[t*hop + off + i] with xp the padded signal (PAD_ZERO also maps NaN/inf samples to 0)
__global__ void frame_window_kernel(const float* __restrict__ x, int n, const float* __restrict__ win, int wlen, int hop,
                                    int off, int pad, int pad_mode, float* __restrict__ F, int frames);
// P[t][k] = re^2 + im^2 from D [frames, 2*nb] (re columns, then im columns)
__global__ void power_kernel(const float* __restrict__ D, float* __restrict__ P, int frames, int nb);
// [(2*nb)][wlen] forward DFT basis restricted to taps off..off+wlen-1 of an n_fft frame: cos rows then -sin rows
std::vector<float> dft_basis(int n_fft, int wlen, int off);
// torchaudio.functional.melscale_fbanks (htk mel scale; slaney-normalised when `slaney`), as [n_mels][n_freqs]
std::vector<float> mel_fb_t(int n_freqs, double f_min, double f_max, int n_mels, int sr, bool slaney);

// ---- librosa's iSTFT at n_fft 2048, hop 512 (enhance.cu), shared by the enhancer and the phase vocoder (pvoc.cu)
// Periodic Hann window, its square, and irfft x window as an NT GEMM operand [2048][re 1025 | im 1025].
void stft_tables(std::vector<float>& hann, std::vector<float>& win2, std::vector<float>& ibasis);
// y[s] = overlap-add sample m = m0 + s of frames 0 .. T-1 (windowed, [.][2048], frame t in row t - t_base), divided by
// the squared-window sum where that exceeds float32 tiny; m0 = 1024 drops librosa's centring pad.  Frames in ascending
// order, so a sample's sum does not depend on which rows hold its frames.
__global__ void ola_kernel(const float* __restrict__ Y, int t_base, int T, const float* __restrict__ win2,
                           float* __restrict__ y, int64_t m0, int64_t ns);

struct HostTensorView {
    const float* data;
    std::vector<int64_t> shape;
    size_t numel() const { size_t n = 1; for (auto s : shape) n *= (size_t)s; return n; }
};

class Conditioner {
public:
    // `get` returns the checkpoint tensor of that name or throws
    Conditioner(const xtts_config& cfg, const std::function<HostTensorView(const std::string&)>& get, cudaStream_t st);
    ~Conditioner();
    // writes cond [n_cond*H] and g [spk_proj] (device pointers)
    void run(const float* wav22k_host, int64_t n22, const float* wav16k_host, int64_t n16, int cond_len_s,
             int chunk_len_s, float* cond_dev, float* g_dev);
    // one front-end on device data, as run() applies it (xtts_debug_cond): op XTTS_COND_MEL22, x [n] -> [1 + n/256][n_mels];
    // XTTS_COND_MEL16, x [n] -> [spk_mels][1 + n/160].  Throws before any launch when the output exceeds cap floats.
    void frontend(int op, const float* x_dev, int n, float* out_dev, size_t cap);
    int n_mels() const;
    int spk_mels() const;

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// xtts_debug_cond (include/xtts_b200.h): one conditioning kernel (or front-end, through `cnd`, which may be NULL for the
// single-kernel ops) on host data, with the launch Conditioner::run uses.  Throws before any launch on a bad argument, and
// after it when the kernel wrote into the guard words around `out`.
void cond_debug(Conditioner* cnd, int op, const int32_t* dims, int n_dims, const float* scal, int n_scal, const float* const* in,
                const int64_t* in_len, int n_in, float* out, int64_t out_len, cudaStream_t st);

// Reference-audio enhancer (enhance.cu): the reference's EnhancedAudioProcessor.process followed by a 16-bit PCM
// write/read, on the GPU.  Needs no weights; its STFT basis and mel filterbanks are built on first use.
class Enhancer {
public:
    explicit Enhancer(cudaStream_t st);
    ~Enhancer();
    // Output length for n input samples (the gating and clarity inverse STFTs drop the tail past 512 * (n / 512)).
    static int64_t out_len(int64_t n, const xtts_enhance_config& c);
    // wav: host, n samples at c.sample_rate.  Writes out_len(n, c) samples to `out` (host).  Throws std::invalid_argument
    // for a bad config and where the reference's enhancer raises (too short, non-finite input or result).
    int64_t run(const float* wav, int64_t n, const xtts_enhance_config& c, float* out, int64_t cap);

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// Phase vocoder (pvoc.cu): the reference's TTSOutput.change_speed — librosa.stft (n_fft 2048, hop 512),
// librosa.phase_vocoder, librosa.istft, librosa.util.normalize(norm=inf) — on the GPU.  Needs no weights.  Works in
// blocks of at most `block_frames` output frames, so its spectral workspace does not grow with the input.
class PhaseVocoder {
public:
    explicit PhaseVocoder(cudaStream_t st);
    ~PhaseVocoder();
    // Output length for n input samples at `rate` (> 0, finite): 512 * (ceil((1 + n / 512) / rate) - 1).
    static int64_t out_len(int64_t n, double rate);
    // wav: host, n samples.  Writes out_len(n, rate) samples to `out` (host).  Throws std::invalid_argument where the
    // reference raises (rate not finite or <= 0, a non-finite sample, an empty or non-finite result) or cap is too small.
    // The result does not depend on block_frames.
    int64_t run(const float* wav, int64_t n, double rate, float* out, int64_t cap, int block_frames);

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// Resampler (resample.cu): torchaudio.functional.resample with its defaults (sinc_interp_hann, lowpass_filter_width 6,
// rolloff 0.99) on float32 mono audio, for speaker references, conditioning and TTSOutput.resample.  Needs no weights.
// Evaluates only the taps inside the filter's window, from a band table cached for the last rate pair, and works in
// passes of at most `block_samples` outputs, so its workspace does not grow with the input.
class Resampler {
public:
    explicit Resampler(cudaStream_t st);
    ~Resampler();
    // ceil(M n / L) (n when orig == new_sr); 0 for a rate outside 1 .. 2^20 - 1 or n outside 0 .. 2^40.
    static int64_t out_len(int64_t n, int orig, int new_sr);
    // wav: host, n samples at orig Hz.  Writes out_len(n, orig, new_sr) samples at new_sr Hz to `out` (host).  Throws
    // std::invalid_argument for a rate out of range, n < 0, a NULL pointer, cap too small or a non-finite sample
    // (orig == new_sr copies the samples as they are).  The result does not depend on block_samples.
    int64_t run(const float* wav, int64_t n, int orig, int new_sr, float* out, int64_t cap, int block_samples);

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// FLAC encoder (flac.cu): mono 16-bit PCM -> a complete lossless FLAC stream (RFC 9639), for TTSOutput.to_bytes("flac").
// Needs no weights.  Works in batches of at most `batch_frames` 4096-sample frames, so its device memory does not grow
// with the input; only the host holds the whole input and stream.
class FlacEncoder {
public:
    explicit FlacEncoder(cudaStream_t st);
    ~FlacEncoder();
    // The most bytes a stream of n samples can take: 42 + ceil(n / 4096) * 8211.
    static int64_t max_bytes(int64_t n);
    // pcm: host, n samples.  md5: 16 bytes or NULL (zeros).  Writes the stream to `out` (host) and its length to
    // *n_out, which is always set (the needed length when cap is too small).  Throws std::invalid_argument for a sample
    // rate outside 1 .. 2^20 - 1, n < 0, a NULL input with n > 0, or cap < *n_out.  The bytes do not depend on
    // batch_frames.
    int64_t run(const int16_t* pcm, int64_t n, int sample_rate, const uint8_t* md5, uint8_t* out, int64_t cap,
                int batch_frames, int64_t* n_out);

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// FLAC decoder (flac.cu): a FLAC stream (RFC 9639: 1-8 channels, 4-32 bits, fixed or variable blocking, every
// subframe and residual coding) -> planar int32 samples, for speaker references and TTSOutput.from_file.  Frame
// headers are found by a scan of every byte position on the device; frames are decoded in parallel, in batches of at
// most `batch_frames` frames and batch_frames * 4096 samples (all channels; one larger frame is a batch alone).
class FlacDecoder {
public:
    explicit FlacDecoder(cudaStream_t st);
    ~FlacDecoder();
    // data: host, n bytes.  Fills *info as soon as STREAMINFO parses (total_samples: STREAMINFO's once the data can
    // hold it, the decoded count at the end).
    // Writes [channels][total] int32 to `out` (host) and returns total.  Throws std::invalid_argument for a stream
    // that breaks the format or fails a check, and for cap < channels * total.  The samples do not depend on
    // batch_frames.
    int64_t run(const uint8_t* data, int64_t n, int32_t* out, int64_t cap, int batch_frames, xtts_flac_info* info);

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

}  // namespace xtts
