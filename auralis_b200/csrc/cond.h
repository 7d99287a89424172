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

// device buffer (the conditioner's and the enhancer's workspaces)
template <typename T>
struct Dev {
    T* p = nullptr; size_t n = 0;
    ~Dev() { if (p) cudaFree(p); }
    void alloc(size_t c) { if (p) cudaFree(p); p = nullptr; n = c; if (c) CUDA_CHECK(cudaMalloc(&p, c * sizeof(T))); }
    void ensure(size_t c) { if (c > n) alloc(c); }
    void up(const std::vector<T>& h, cudaStream_t st) { alloc(h.size()); CUDA_CHECK(cudaMemcpyAsync(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st)); CUDA_CHECK(cudaStreamSynchronize(st)); }
};

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
    // stage taps for parity tests (host copies of the last run)
    std::vector<float> last_mel;       // [frames,80] of the first piece
    int last_mel_frames = 0;

private:
    struct Impl;
    std::unique_ptr<Impl> impl;
};

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

}  // namespace xtts
