// Engine: weights, paged-KV slots, continuous-batching scheduler thread, vocoder driver and the C ABI
// (include/xtts_b200.h).  Host orchestration that stands in for XTTSv2Engine + vLLM's engine loop
// (XTTSv2.py:690-814, SURVEY.md §3.2); every tensor op below it is one of the kernels in this directory.
#include "../../include/xtts_b200.h"
#include "kernels.h"
#include "cond.h"
#include "harness.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <tuple>
#include <unordered_map>
#include <vector>

namespace xtts {

static thread_local std::string t_last_error;
static std::string g_last_error;
static std::mutex g_err_mu;

static void set_error(const std::string& s) {
    t_last_error = s;
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_last_error = s;
}

// a request the engine cannot take in its current state (XTTS_ERR_STATE), e.g. a KV format switch with work in flight
struct StateError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

static double now_s() {
    using namespace std::chrono;
    return duration<double>(steady_clock::now().time_since_epoch()).count();
}

// ------------------------------------------------------------------------------------------------
struct HostTensor {
    std::vector<float> data;
    std::vector<int64_t> shape;
    size_t numel() const { size_t n = 1; for (auto s : shape) n *= (size_t)s; return n; }
};

// weight matrix usable as the B operand of either GEMM path
struct Linear {
    DBuf<float> w32;              // [N,K] fp32   (precision fp32)
    DBuf<__nv_bfloat16> w16;      // [N,K] bf16   (precision bf16)
    DBuf<float> b;                // [N]
    int N = 0, K = 0;
};

struct ConvW {
    DBuf<float> wt;               // [Cin][K][Cout]      (CUDA-core path)
    DBuf<__half> blob;            // wgmma tile blob     (fast mode, Conv1d only)
    ConvTcPlan plan{};
    bool tc = false;
    DBuf<float> b;                // [Cout]
    int Cin = 0, Cout = 0, K = 0;
};

struct Sequence {
    uint64_t id = 0;
    std::vector<int32_t> text_ids;
    int speaker = 0;
    xtts_sampling sp{};
    float speed = 1.f;            // speaking rate (xtts_submit_speed): time-scales the latents before the vocoder
    xtts_beam beam{1, 1.f, 0};    // xtts_submit_beams: num_beams > 1 decodes the chunk as a beam-search group
    std::vector<int> beam_slots;  // the group's slots, beam j in beam_slots[j]; beam_slots[0] == slot (the primary)
    int slot = -1;
    int n_prompt = 0;
    int max_tok = 0;              // min(sp.max_tokens, max_audio_tokens)
    int steps = 0;                // decode steps issued so far (host-side mirror of n_gen - 1)
    std::vector<int> pages;
    double t_submit = 0, t_first = 0, t_done = 0;
    bool cancelled = false;
    // results: written on the vocoder stream, valid once the job that wrote them has completed
    int n_tokens = 0;             // final token count (0 while decoding)
    int32_t* tok_host = nullptr;  // pinned [max_tok]
    size_t tok_cap = 0;
    float* wav_host = nullptr;    // pinned, the whole chunk's samples (option d2h_wav = 1)
    size_t wav_cap = 0;
    float* wav_dev = nullptr;     // pooled device buffer instead (d2h_wav = 0)
    size_t wav_dev_cap = 0;
    float* lat_dev = nullptr;     // [n_tokens, H] snapshot of the latent ring (pooled device buffer)
    size_t lat_dev_cap = 0;
    // vocoder progress: the chunk's audio is produced window by window while it is still decoding
    int next_boundary = 0;        // tokens: the next window is cut here (0 = no further cut, the rest goes out at the end)
    int seg_next = 0;             // distance of the cuts after the first (0 = none)
    bool stream_pieces = false;   // windows are handed to the completion queue as partial results (sp.early_tokens > 0)
    int voc_z_done = 0;           // z-frames whose samples are produced or in flight
    int tok_delivered = 0, samp_delivered = 0;   // covered by partial results already queued
};

// one entry of the completion queue: a partial piece of a chunk (status 1) or its final result (status <= 0)
struct Piece {
    std::shared_ptr<Sequence> s;
    int status = 0;
    int tok0 = 0, tok1 = 0;       // tokens [tok0, tok1) of s->tok_host
    int samp0 = 0, nsamp = 0;     // samples [samp0, samp0 + nsamp) of the chunk's waveform buffer
    double t_done = 0;
    bool final = false;
};

// one window of one chunk on its way through the vocoder: z-frames [zw0, zw1) are computed, the samples of [zk0, zk1) kept
// (the margins are the vocoder's receptive field, so kept samples equal those of the unsplit chunk)
struct VocJob {
    std::shared_ptr<Sequence> s;
    int T_clamp = 0;              // latent frames the interpolation may touch
    int zw0 = 0, zw1 = 0, zk0 = 0, zk1 = 0;
    int tok_upto = 0;             // tokens [0, tok_upto) are final and copied out with this job
    bool final = false;
    bool internal = false;        // a leading window of a finished chunk too long for one window: never a partial piece
    int fail_status = 0;          // final job of a cancelled / failed chunk: no vocoder work, this status is delivered
};
struct VocBatch {
    std::vector<VocJob> jobs;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

class Engine {
public:
    explicit Engine(const xtts_config& c);
    ~Engine();
    // binds this engine's launcher state (launch counter, profiler, knobs) to the calling thread for one API call
    struct Bind {
        KernelCtx* prev;
        explicit Bind(Engine* e) : prev(t_kctx) { t_kctx = &e->kctx_; }
        ~Bind() { t_kctx = prev; }
    };

    void load_weight(const char* name, const float* data, const int64_t* shape, int ndim);
    void finalize_weights();
    void set_speaker(int slot, const float* cond, const float* g);
    void get_speaker(int slot, float* cond, float* g);
    void condition(int slot, const float* w22, int64_t n22, const float* w16, int64_t n16, int cond_len, int chunk_len);
    int64_t enhance(const float* wav, int64_t n, const xtts_enhance_config& c, float* out, int64_t cap);
    int64_t change_speed(const float* wav, int64_t n, double rate, float* out, int64_t cap);
    int64_t resample(const float* wav, int64_t n, int orig_sr, int new_sr, float* out, int64_t cap);
    int64_t encode_flac(const int16_t* pcm, int64_t n, int sample_rate, const uint8_t* md5, uint8_t* out, int64_t cap,
                        int64_t* n_out);
    int64_t decode_flac(const uint8_t* data, int64_t n, int32_t* out, int64_t cap, xtts_flac_info* info);
    void submit(uint64_t id, const int32_t* text, int n_text, int speaker, const xtts_sampling& sp, float speed,
                const xtts_beam* beam = nullptr);
    void cancel(uint64_t id);
    int poll(xtts_result* out, int timeout_ms);
    void fetch(uint64_t id, int32_t* tokens, float* wav, float* latents);
    void set_option(const std::string& k, int64_t v);
    void get_stats(xtts_stats* s);
    void sync_idle();
    void kernel_profile(xtts_kernel_profile* out);
    void device_timer(int op, double* ms);
    int trace(int op, uint64_t* out, int cap);

    void vocode_sync(const float* latents, int T, int speaker, float* wav, int* n_out, const char* stage,
                     float* stage_out, int64_t stage_cap);
    void vocode_window_sync(const float* latents, int T, int speaker, int z0, int nz, float* wav);
    void vocode_speed_sync(const float* latents, int T, int speaker, float speed, int z0, int nz, float* wav, int* n_out);
    void gpt_prefill_sync(const int32_t* text, int n_text, int speaker, const int32_t* audio, int n_audio,
                          float* hidden_out, float* logits_out, float* latents_out);
    void gpt_teacher_forced_sync(const int32_t* text, int n_text, int speaker, const int32_t* forced, int n,
                                 const xtts_sampling& sp, float* logits_out, float* latents_out, int32_t* sampled_out);
    // runs f with this engine's stream and options under its API lock; throws unless the engine is idle
    void run_idle(const std::function<void(const HarnessCtx&)>& f);

private:
    KernelCtx kctx_;
    // ---- geometry
    xtts_config cfg;
    int H, L, NH, FF, V, Vpad, B, NSLOT, CAP, MAXP, max_pages, SEENW, S;
    int prefill_rows_cap;
    bool bf16;                    // 16-bit fast mode (wgmma GEMMs, 16-bit KV): bf16 operands, or IEEE fp16 when `f16`
    bool f16 = false;             // precision fp16: same kernels, fp16 operands (3 more mantissa bits than bf16, range is ample here)
    int gflag = 0;                // GEMM_F16 in fp16 mode
    cudaStream_t st = nullptr;
    cudaStream_t st_voc = nullptr;                       // the vocoder's own (low-priority) stream: runs beside the decode step
    static constexpr int kMaxMicro = 4;
    cudaStream_t st_mb[kMaxMicro] = {nullptr, nullptr, nullptr, nullptr};   // [0] == st; decode micro-batch branches
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;       // xtts_device_timer
    bool timer_armed = false;
    cudaEvent_t ev_fork = nullptr, ev_join[kMaxMicro] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_vjoin = nullptr;

    // ---- weights
    std::map<std::string, HostTensor> raw;
    std::atomic<bool> finalized{false};
    DBuf<float> text_emb, text_pos, wte, wpe;
    struct Layer { DBuf<float> ln1w, ln1b, ln2w, ln2b; Linear qkv, o, fc, proj; };
    std::vector<std::unique_ptr<Layer>> layers;
    DBuf<float> lnfw, lnfb, fnw, fnb;
    Linear mel_head;
    ConvW conv_pre;
    std::vector<std::unique_ptr<ConvW>> ups;
    struct RB { std::unique_ptr<ConvW> c1[4], c2[4]; };
    std::vector<std::unique_ptr<RB>> rbs;
    DBuf<float> conv_post_w;
    int post_cin = 0;
    struct CondLin { DBuf<float> w, b; int rows = 0; };
    CondLin cond_layer;
    std::vector<std::unique_ptr<CondLin>> conds;
    uint64_t weight_bytes = 0;
    std::unique_ptr<Conditioner> conditioner;
    std::unique_ptr<Enhancer> enhancer;          // built on the first xtts_enhance
    std::unique_ptr<PhaseVocoder> pvoc;          // built on the first xtts_change_speed
    int pvoc_block_frames = 4096;                // option "pvoc_block_frames"
    std::unique_ptr<Resampler> resampler;        // built on the first xtts_resample
    int resample_block_samples = 1 << 22;        // option "resample_block_samples"
    std::unique_ptr<FlacEncoder> flac;           // built on the first xtts_encode_flac
    std::unique_ptr<FlacDecoder> flac_dec;       // built on the first xtts_decode_flac
    int flac_batch_frames = 8192;                // option "flac_batch_frames" (encoder and decoder)

    // ---- speakers
    DBuf<float> spk_cond, spk_g, spk_cbias;
    int cbias_stride = 0;
    std::vector<int> cbias_off;
    std::vector<char> spk_valid;

    // ---- slot state (device)
    DBuf<int> d_last_tok, d_n_gen, d_ctx_len, d_finished, d_tokens, d_sampled, d_forced, d_top_k, d_max_tokens,
        d_stop, d_seq_seed, d_block_tables, d_active, d_rowidx, d_row_slot, d_row_pos, d_lat_pos;
    DBuf<unsigned> d_seen;
    DBuf<float> d_temp, d_top_p, d_pen;
    DBuf<unsigned long long> d_seed;
    DBuf<int> d_beam_flag;        // [NSLOT] SampleState::beam
    // beam search (beam.cu): per-group state, history and page pool indexed by the primary slot, scores per slot
    DBuf<BeamState> d_beam_state;
    DBuf<int2> d_beam_hist;
    DBuf<int> d_beam_pool;
    DBuf<float> d_beam_scores;
    DBuf<BeamDesc> d_beam_desc;
    BeamDesc* h_beam_desc = nullptr;               // pinned [NSLOT]
    BeamState* h_beam_init = nullptr;              // pinned [NSLOT]: initial state of the groups of an admission wave
    int* h_beam_pool = nullptr;                    // pinned [NSLOT][beam_pool_cap]: their page pools
    DBuf<void*> d_kv_ptrs;                          // [2][L] K then V pool of each layer
    int beam_pool_cap = 0;
    DBuf<float> d_latents;
    DBuf<RowDesc> d_rows;
    DBuf<AttnSeq> d_attnseq;
    bool use_forced = false;
    // KV pools, one pair per layer, in one format: fp32 (parity mode), 16-bit, or fp8 (option "kv_fp8", kv_fp8.cuh)
    std::vector<std::unique_ptr<DBuf<float>>> k32, v32;
    std::vector<std::unique_ptr<DBuf<__nv_bfloat16>>> k16, v16;
    std::vector<std::unique_ptr<DBuf<uint8_t>>> k8, v8;
    bool kv_fp8 = false;
    std::vector<int> free_pages;
    void alloc_kv();              // the pools in the current format, d_kv_ptrs, every page free
    __nv_fp8_e4m3* k8p(int l) const { return reinterpret_cast<__nv_fp8_e4m3*>(k8[l]->p); }
    __nv_fp8_e4m3* v8p(int l) const { return reinterpret_cast<__nv_fp8_e4m3*>(v8[l]->p); }
    // GPT workspace
    DBuf<float> wX, wQKV, wLOG, wPART;
    DBuf<float> wXn32, wATT32, wFF32, wY32;
    DBuf<__nv_bfloat16> wXn16, wATT16, wFF16, wY16;
    // pinned staging
    int* h_finished = nullptr;       // [2][NSLOT]: finished flags, then n_gen, read back after every step
    SlotInit* h_slot_init = nullptr; // [B + 1] admission wave
    int* h_slot_pages = nullptr;     // [B + 1][max_pages]
    DBuf<SlotInit> d_slot_init;
    DBuf<int> d_slot_pages;
    // vocoder workspace (used on st_voc only)
    DBuf<float> vz, vpre, vb[5], vwav, vcb;
    DBuf<__half> vz16, va16[5];   // fp16 operand atoms of the tensor-core vocoder path
    bool tc_vocoder_ready = false;
    int voc_max_T = 0, voc_max_Tz = 0;
    size_t voc_cap_z = 0;         // z-frames a batch may hold: items x longest window
    size_t vz16_halves = 0, va16_halves = 0;
    int voc_hz = 16;              // receptive field of the vocoder in z-frames (window margin), from the geometry
    int voc_hop = 1;              // samples per z-frame
    std::vector<int> stage_ch;

    // ---- scheduler
    // Two locks so that submit/poll never wait behind a GPU step:
    //   q_mu   — pending / done queues, inflight counter (short critical sections)
    //   mu     — all GPU state and work issue: held by the scheduler thread for one iteration at a time and by
    //            the synchronous entry points (weights, speakers, debug calls)
    std::mutex mu, q_mu, pin_mu;
    // std::mutex is not fair: the scheduler thread re-takes `mu` a few hundred nanoseconds after releasing it and would
    // starve a synchronous API call (stats, set_speaker, options) for as long as the engine stays busy.  API calls
    // announce themselves; the scheduler waits for them between two iterations.
    std::atomic<int> api_waiting{0};
    struct ApiLock {
        Engine* e; std::unique_lock<std::mutex> lk;
        explicit ApiLock(Engine* en) : e(en) { e->api_waiting.fetch_add(1); lk = std::unique_lock<std::mutex>(e->mu); e->api_waiting.fetch_sub(1); }
    };
    std::condition_variable cv_work, cv_done;
    std::deque<std::shared_ptr<Sequence>> pending;      // q_mu
    std::deque<std::shared_ptr<Sequence>> waiting;      // scheduler thread only: accepted, not yet admitted
    std::vector<std::shared_ptr<Sequence>> running;     // index = position in active list
    std::vector<int> free_slots;
    std::deque<std::shared_ptr<Piece>> done_q;                                  // q_mu
    std::unordered_map<uint64_t, std::deque<std::shared_ptr<Piece>>> done_map;  // q_mu: unfetched pieces per id, oldest first
    std::vector<uint64_t> cancel_req;                                           // q_mu
    std::deque<VocJob> voc_pending;          // scheduler thread only
    std::deque<VocBatch> voc_inflight;       // scheduler thread only (stream order = queue order)
    int voc_segment = 0;          // option "voc_segment": tokens per vocoder window while a chunk decodes (0 = whole chunks at the end)
    int voc_sms = 0;              // option "voc_sms": SMs the conv kernels may take while a decode step is in flight (0 = all)
    int voc_max_items = kVocMaxItems;   // option "voc_batch": windows per vocoder launch
    std::thread worker;
    std::atomic<bool> stop{false};
    int inflight = 0;
    bool d2h_wav = true;
    bool use_splitk = true;       // option "splitk"
    bool use_pdl = true;          // option "pdl" (programmatic dependent launch along the decode chain)
    bool use_graphs = true;       // option "cuda_graphs"
    std::atomic<bool> hold_admission{false};   // option "hold_admission": queue submissions, admit nothing (batch submit)
    std::map<int, std::pair<cudaGraphExec_t, KernelProfiler::GraphRecs*>> prof_graphs;   // decode graphs with event-record nodes (option "profile")
    KernelProfiler::GraphRecs* last_prof = nullptr;     // recs of the profiled graph launched by the current step
    void drop_graphs();
    DBuf<unsigned long long> d_trace; DBuf<unsigned> d_trace_n;      // debug timeline (xtts_debug_trace)
    int n_micro = 2;              // option "microbatches": decode rows are split into this many concurrent branches
    int micro_min_rows = 48;      // option "microbatch_min_rows": below this many active rows the step stays single-branch
    int eager_steps_done = 0;
    std::map<int, cudaGraphExec_t> decode_graphs;
    std::map<int, unsigned long long> graph_kernels;
    bool use_tc_vocoder = true;   // fast mode only; option "tc_vocoder" switches back to the fp32 CUDA-core convs
    bool use_resblock_tc = true;  // test / A-B switch "tc_resblock": 0 runs every resblock as its six conv1d_tc launches (same bits)
    std::vector<std::pair<float*, size_t>> pinned_pool;
    // stats
    double decode_ctx_sum = 0;
    uint64_t st_decode_steps = 0, st_prefill_rows = 0, st_tokens = 0, st_samples = 0;
    double st_gpt_ms = 0, st_voc_ms = 0, st_cond_ms = 0;
    unsigned long long launch_base = 0;

    // ---- helpers
    const HostTensor& need(const std::string& name) const;
    void up(DBuf<float>& d, const std::vector<float>& h) { d.alloc(h.size()); d.upload(h.data(), h.size(), st); weight_bytes += h.size() * 4; }
    void make_linear(Linear& lin, const std::string& wname, const std::string& bname, bool conv1d_layout, int pad_n = 0);
    void make_conv(ConvW& c, const std::string& prefix, bool transposed, bool has_bias);
    struct VocItem { const float* lat; int T; int z0, nz; int speaker; float speed = 1.f; };
    InterpItem interp_item(const VocItem& v) const;
    bool speed_stage(int T, float speed) const;
    struct VocSpan { int zw0, zw1, zk0, zk1; };
    std::vector<VocSpan> split_windows(int zk0, int Tz) const;
    void run_vocoder_tc(const VocItem* it, int nb, int Lz, float* wav_dev_out, const char* stage, float* stage_out,
                        int64_t stage_cap);
    void run_vocoder_f32(const VocItem* it, int nb, int Lz, float* wav_dev_out, const char* stage, float* stage_out,
                         int64_t stage_cap);
    bool voc_fits(int nb, int Lz) const;
    void compute_voc_margin(int pre_k);
    int z_frames(int T, float speed = 1.f) const;
    int z_avail(int n, float speed = 1.f) const;
    std::vector<float> folded(const std::string& prefix) const;
    GptTables tables() const {
        GptTables t; t.text_emb = text_emb.p; t.text_pos = text_pos.p; t.wte = wte.p; t.wpe = wpe.p;
        t.spk_cond = spk_cond.p; t.H = H; t.n_cond = cfg.n_cond_latents; return t;
    }
    SampleState sample_state() const;
    void finish_speaker(int slot);
    void gemm(const void* A, const Linear& lin, const float* resid, void* out, int M, int flags, bool pdl = false);
    void layers_forward(int M, bool prefill, int nseq, int max_nq);
    void head_and_sample(int M, const int* row_index, const int* slots_dev, const int* lat_pos, int advance_ctx, bool do_sample,
                         bool pdl_first = true);
    void decode_layers_rows(int r0, int Mi, cudaStream_t s, bool pdl_first, double ctx_sum);
    // split-K reduction + bias + residual + LayerNorm into the 16-bit operand buffer, in the engine's 16-bit format
    void reduce_ln16(float* X, const float* part, int splits, const float* bias, const float* w, const float* b, __nv_bfloat16* Y, int M,
                     cudaStream_t s, bool pdl) {
        if (f16) launch_residual_reduce_layernorm<__half>(X, part, splits, bias, w, b, reinterpret_cast<__half*>(Y), M, H, cfg.ln_eps, s, pdl);
        else launch_residual_reduce_layernorm<__nv_bfloat16>(X, part, splits, bias, w, b, Y, M, H, cfg.ln_eps, s, pdl);
    }
    void init_slots(const std::vector<Sequence*>& seqs, const int32_t* forced, int n_forced);
    void release_pages(Sequence& s);
    void release_slot(Sequence& s);
    void free_seq_buffers(Sequence& s);
    void recycle_seq_buffers(Sequence& s);
    int build_prefill(const std::vector<Sequence*>& seqs, const std::vector<std::vector<int32_t>>& audio,
                      std::vector<int>& last_rows, int& max_nq);
    void prefill(const std::vector<Sequence*>& seqs);
    void beam_step(const std::vector<Sequence*>& groups, const std::vector<int>& rows0, bool first);
    void decode_step(const std::vector<int>& active);
    void run_vocoder(const VocItem* it, int nb, float* wav_dev_out, const char* stage, float* stage_out, int64_t stage_cap);
    int samples_for(int T, float speed = 1.f) const;
    void on_finished(std::shared_ptr<Sequence> s, int n_tokens, int fail_status);
    void maybe_cut_window(std::shared_ptr<Sequence>& s);
    void dispatch_ready(bool decode_active);
    void dispatch_batch(std::vector<VocJob>& jobs, bool decode_active);
    void reap(bool block);
    void complete_batch(VocBatch& b);
    void deliver(std::shared_ptr<Piece> p, bool ends_sequence);
    void fail_unadmitted(std::shared_ptr<Sequence> s, int code, const char* what);
    void process_cancels(const std::vector<uint64_t>& ids);
    float* pinned_get(size_t n, size_t* cap);
    void pinned_put(float* p, size_t cap);
    float* dev_get(size_t n, size_t* cap);           // device buffer pool (no cudaMalloc/cudaFree per chunk)
    void dev_put(float* p, size_t cap);
    std::vector<std::pair<float*, size_t>> dev_pool;
    void loop();
    void require_finalized() const { if (!finalized) throw std::runtime_error("weights not finalized: call xtts_finalize_weights first"); }
    void require_idle() const {
        if (!running.empty() || !waiting.empty() || !voc_pending.empty() || !voc_inflight.empty())
            throw std::runtime_error("debug entry points need an idle engine");
    }
};

// ================================================================================================
// construction
// ================================================================================================
Engine::Engine(const xtts_config& c) : cfg(c) {
    Bind bind_ctx(this);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        (void)cudaGetLastError();
        throw std::runtime_error("libxtts_b200: no CUDA device visible — this library has no CPU fallback");
    }
    if (c.device < 0 || c.device >= ndev) throw std::runtime_error("invalid CUDA device ordinal");
    CUDA_CHECK(cudaSetDevice(c.device));
    cudaDeviceProp prop{};
    CUDA_CHECK(cudaGetDeviceProperties(&prop, c.device));
    if (prop.major != 9 || prop.minor != 0) {
        throw std::runtime_error(std::string("libxtts_b200 is built for sm_90a only; found ") + prop.name + " (sm_" +
                                 std::to_string(prop.major) + std::to_string(prop.minor) + ")");
    }
    H = c.hidden; L = c.layers; NH = c.heads; FF = c.ff; V = c.n_audio_tokens;
    if (H != NH * kHeadDim) throw std::runtime_error("hidden must equal heads * 64");
    if (H % 64 != 0 || FF % 64 != 0) throw std::runtime_error("hidden and ff must be multiples of 64");
    if (V > 2048) throw std::runtime_error("n_audio_tokens > 2048 unsupported");
    Vpad = ceil_div(V, 32) * 32;
    B = c.max_batch; NSLOT = B + 1;     // last slot is reserved for the synchronous debug entry points
    CAP = c.max_audio_tokens;
    MAXP = c.n_cond_latents + (c.max_text_tokens + 2) + 1;
    max_pages = ceil_div(MAXP + CAP, kPageTokens);
    SEENW = ceil_div(V, 32);
    S = std::max(1, c.max_speakers);
    bf16 = c.precision == XTTS_PRECISION_BF16 || c.precision == XTTS_PRECISION_FP16;
    f16 = c.precision == XTTS_PRECISION_FP16;
    gflag = f16 ? GEMM_F16 : 0;
    if (c.precision != XTTS_PRECISION_FP32 && !bf16) throw std::runtime_error("unknown precision");
    if (bf16) { std::string err; if (!gemm_tc_init(&err)) throw std::runtime_error(err); }
    // the decode step is a chain of short dependent kernels: its streams get the highest priority, the vocoder (long
    // throughput kernels on its own stream) the lowest, so a decode kernel never queues behind vocoder CTAs that have
    // not started yet
    int prio_lo = 0, prio_hi = 0;
    CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    CUDA_CHECK(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio_hi));
    st_mb[0] = st;
    for (int i = 1; i < kMaxMicro; ++i) CUDA_CHECK(cudaStreamCreateWithPriority(&st_mb[i], cudaStreamNonBlocking, prio_hi));
    CUDA_CHECK(cudaStreamCreateWithPriority(&st_voc, cudaStreamNonBlocking, prio_lo));
    CUDA_CHECK(cudaEventCreateWithFlags(&ev_vjoin, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    for (int i = 1; i < kMaxMicro; ++i) CUDA_CHECK(cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming));

    // speakers
    spk_cond.alloc((size_t)S * c.n_cond_latents * H);
    spk_g.alloc((size_t)S * c.d_vector);
    spk_valid.assign(S, 0);
    cbias_off.clear();
    int off = 0;
    cbias_off.push_back(off); off += c.voc_init_ch;
    stage_ch.clear();
    for (int i = 0; i < c.voc_n_up; ++i) {
        const int ch = c.voc_init_ch >> (i + 1);
        stage_ch.push_back(ch);
        cbias_off.push_back(off); off += ch;
    }
    cbias_stride = off;
    spk_cbias.alloc((size_t)S * cbias_stride);

    // slot state
    d_last_tok.alloc(NSLOT); d_n_gen.alloc(NSLOT); d_ctx_len.alloc(NSLOT); d_finished.alloc(NSLOT);
    d_tokens.alloc((size_t)NSLOT * CAP); d_sampled.alloc((size_t)NSLOT * CAP); d_forced.alloc((size_t)NSLOT * CAP);
    d_top_k.alloc(NSLOT); d_max_tokens.alloc(NSLOT); d_stop.alloc(NSLOT); d_seq_seed.alloc(NSLOT);
    d_temp.alloc(NSLOT); d_top_p.alloc(NSLOT); d_pen.alloc(NSLOT); d_seed.alloc(NSLOT);
    d_seen.alloc((size_t)NSLOT * SEENW);
    d_block_tables.alloc((size_t)NSLOT * max_pages);
    d_active.alloc(NSLOT);
    d_beam_flag.alloc(NSLOT); d_beam_flag.zero(st);
    beam_pool_cap = kMaxBeams * max_pages;
    d_beam_state.alloc(NSLOT); d_beam_hist.alloc((size_t)NSLOT * CAP * kMaxBeams); d_beam_pool.alloc((size_t)NSLOT * beam_pool_cap);
    d_beam_desc.alloc(NSLOT);
    CUDA_CHECK(cudaMallocHost(&h_beam_desc, NSLOT * sizeof(BeamDesc)));
    CUDA_CHECK(cudaMallocHost(&h_beam_init, NSLOT * sizeof(BeamState)));
    CUDA_CHECK(cudaMallocHost(&h_beam_pool, (size_t)NSLOT * beam_pool_cap * sizeof(int)));
    beam_init_device();
    d_latents.alloc((size_t)NSLOT * CAP * H);
    d_finished.zero(st); d_n_gen.zero(st); d_ctx_len.zero(st); d_last_tok.zero(st);
    CUDA_CHECK(cudaMallocHost(&h_finished, 2 * NSLOT * sizeof(int)));
    std::memset(h_finished, 0, 2 * NSLOT * sizeof(int));
    CUDA_CHECK(cudaMallocHost(&h_slot_init, NSLOT * sizeof(SlotInit)));
    CUDA_CHECK(cudaMallocHost(&h_slot_pages, (size_t)NSLOT * max_pages * sizeof(int)));
    d_slot_init.alloc(NSLOT); d_slot_pages.alloc((size_t)NSLOT * max_pages);

    // prefill row budget: whole prompts of up to 8 sequences at the maximum prompt length, >= one debug pass
    prefill_rows_cap = std::max(8 * MAXP, MAXP + CAP);
    d_rows.alloc(prefill_rows_cap); d_row_slot.alloc(prefill_rows_cap); d_row_pos.alloc(prefill_rows_cap);
    d_rowidx.alloc(prefill_rows_cap); d_lat_pos.alloc(prefill_rows_cap);
    d_attnseq.alloc(NSLOT);
    const size_t Mmax = (size_t)std::max(prefill_rows_cap, NSLOT);
    wX.alloc(Mmax * H); wQKV.alloc(Mmax * 3 * H); wLOG.alloc((size_t)std::max(NSLOT, CAP + 1) * Vpad);
    d_beam_scores.alloc((size_t)NSLOT * Vpad);
    if (bf16) wPART.alloc((size_t)8 * NSLOT * H);
    if (bf16) { wXn16.alloc(Mmax * H); wATT16.alloc(Mmax * H); wFF16.alloc(Mmax * FF); wY16.alloc((size_t)std::max(NSLOT, CAP + 1) * H); }
    else { wXn32.alloc(Mmax * H); wATT32.alloc(Mmax * H); wFF32.alloc(Mmax * FF); wY32.alloc((size_t)std::max(NSLOT, CAP + 1) * H); }

    alloc_kv();
    for (int s = B - 1; s >= 0; --s) free_slots.push_back(s);

    // vocoder workspace: a batch is up to kVocMaxItems windows, nb x (longest window) <= voc_cap_z z-frames
    // (8 whole chunks of the maximum length, or more, shorter windows)
    voc_max_T = CAP;
    {
        voc_hop = 1;
        for (int i = 0; i < c.voc_n_up; ++i) voc_hop *= c.voc_up_rates[i];
        voc_max_Tz = z_frames(voc_max_T);
        const int nfull = std::max(1, std::min(8, B));
        voc_cap_z = (size_t)nfull * voc_max_Tz;
        vz.alloc(voc_cap_z * c.voc_in_dim);
        vpre.alloc(voc_cap_z * c.voc_init_ch);
        size_t mx = 0; size_t rate = 1;
        for (int i = 0; i < c.voc_n_up; ++i) { rate *= c.voc_up_rates[i]; mx = std::max(mx, (size_t)stage_ch[i] * rate); }
        for (auto& b : vb) b.alloc(voc_cap_z * mx);
        vwav.alloc(voc_cap_z * voc_hop);
        vcb.alloc((size_t)kVocMaxItems * cbias_stride);
        compute_voc_margin(7);
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
    launch_base = g_launch_count;
    worker = std::thread([this] { this->loop(); });
}

// KV pools of every layer in the current format (the old ones are freed first, so a switch never holds both), their base
// pointers for the beam kernels, and a free list of every page
void Engine::alloc_kv() {
    k32.clear(); v32.clear(); k16.clear(); v16.clear(); k8.clear(); v8.clear();
    const int total_pages = NSLOT * max_pages;
    const size_t page_elems = (size_t)NH * kPageTokens * kHeadDim;
    std::vector<void*> kv(2 * L);
    for (int l = 0; l < L; ++l) {
        if (kv_fp8) {
            k8.emplace_back(new DBuf<uint8_t>()); v8.emplace_back(new DBuf<uint8_t>());
            k8.back()->alloc(total_pages * NH * kv_block_bytes(1)); v8.back()->alloc(total_pages * NH * kv_block_bytes(1));
            kv[l] = k8[l]->p; kv[L + l] = v8[l]->p;
        } else if (bf16) {
            k16.emplace_back(new DBuf<__nv_bfloat16>()); v16.emplace_back(new DBuf<__nv_bfloat16>());
            k16.back()->alloc(total_pages * page_elems); v16.back()->alloc(total_pages * page_elems);
            kv[l] = k16[l]->p; kv[L + l] = v16[l]->p;
        } else {
            k32.emplace_back(new DBuf<float>()); v32.emplace_back(new DBuf<float>());
            k32.back()->alloc(total_pages * page_elems); v32.back()->alloc(total_pages * page_elems);
            kv[l] = k32[l]->p; kv[L + l] = v32[l]->p;
        }
    }
    d_kv_ptrs.alloc(2 * L); d_kv_ptrs.upload(kv.data(), 2 * L, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    free_pages.clear();
    for (int p = total_pages - 1; p >= 0; --p) free_pages.push_back(p);
}

// receptive field of the generator in z-frames: conv_pre, per stage the transposed conv (1.5 input frames) and the widest
// resblock chain (sum over its dilations of the two convs' half-widths), conv_post (k = 7); + 2 frames of margin
void Engine::compute_voc_margin(int pre_k) {
    const auto& c = cfg;
    double rf = (pre_k - 1) / 2, rt = 1.0;
    for (int i = 0; i < c.voc_n_up; ++i) {
        rf += 1.5 / rt;
        rt *= c.voc_up_rates[i];
        double widest = 0;
        for (int j = 0; j < c.voc_n_rb; ++j) {
            const int hk = (c.voc_rb_kernels[j] - 1) / 2;
            double w = 0;
            for (int t = 0; t < 3; ++t) w += hk * c.voc_rb_dilations[t] + hk;
            widest = std::max(widest, w);
        }
        rf += widest / rt;
    }
    rf += 3.0 / rt;
    voc_hz = (int)std::ceil(rf) + 2;
}

Engine::~Engine() {
    {
        std::lock_guard<std::mutex> lk(q_mu);
        stop = true;
    }
    cv_work.notify_all();
    if (worker.joinable()) worker.join();
    cudaSetDevice(cfg.device);
    cudaStreamSynchronize(st);
    if (st_voc) cudaStreamSynchronize(st_voc);
    drop_graphs();
    // buffers of every chunk still in the pipeline or never fetched
    for (auto& s : running) free_seq_buffers(*s);
    for (auto& j : voc_pending) free_seq_buffers(*j.s);
    for (auto& b : voc_inflight) {
        for (auto& j : b.jobs) free_seq_buffers(*j.s);
        if (b.ev0) cudaEventDestroy(b.ev0);
        if (b.ev1) cudaEventDestroy(b.ev1);
    }
    for (auto& kv : done_map) for (auto& pc : kv.second) if (pc->s) free_seq_buffers(*pc->s);
    for (auto& pr : pinned_pool) cudaFreeHost(pr.first);
    for (auto& pr : dev_pool) cudaFree(pr.first);
    if (h_finished) cudaFreeHost(h_finished);
    if (h_slot_init) cudaFreeHost(h_slot_init);
    if (h_slot_pages) cudaFreeHost(h_slot_pages);
    if (h_beam_desc) cudaFreeHost(h_beam_desc);
    if (h_beam_init) cudaFreeHost(h_beam_init);
    if (h_beam_pool) cudaFreeHost(h_beam_pool);
    for (int i = 1; i < kMaxMicro; ++i) { if (st_mb[i]) cudaStreamDestroy(st_mb[i]); if (ev_join[i]) cudaEventDestroy(ev_join[i]); }
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_vjoin) cudaEventDestroy(ev_vjoin);
    if (ev_t0) cudaEventDestroy(ev_t0);
    if (ev_t1) cudaEventDestroy(ev_t1);
    if (st_voc) cudaStreamDestroy(st_voc);
    if (st) cudaStreamDestroy(st);
}

// ================================================================================================
// weights
// ================================================================================================
void Engine::load_weight(const char* name, const float* data, const int64_t* shape, int ndim) {
    ApiLock lk(this);
    if (finalized) throw std::runtime_error("weights already finalized");
    HostTensor t;
    t.shape.assign(shape, shape + ndim);
    const size_t n = t.numel();
    t.data.assign(data, data + n);
    raw[name] = std::move(t);
}

const HostTensor& Engine::need(const std::string& name) const {
    auto it = raw.find(name);
    if (it == raw.end()) throw std::runtime_error("missing weight: " + name);
    return it->second;
}

// [K,N] (HF Conv1D, in x out) or [N,K] (nn.Linear) -> device [Npad,K] in the engine precision
void Engine::make_linear(Linear& lin, const std::string& wname, const std::string& bname, bool conv1d_layout, int pad_n) {
    const HostTensor& w = need(wname);
    if (w.shape.size() != 2) throw std::runtime_error("expected 2-D weight: " + wname);
    const int d0 = (int)w.shape[0], d1 = (int)w.shape[1];
    const int N = conv1d_layout ? d1 : d0, K = conv1d_layout ? d0 : d1;
    const int Np = pad_n > 0 ? pad_n : N;
    std::vector<float> t((size_t)Np * K, 0.f);
    if (conv1d_layout) {
        const int BL = 32;                                  // blocked transpose (vllm_mm_gpt.py:723-725)
        for (int k0 = 0; k0 < K; k0 += BL)
            for (int n0 = 0; n0 < N; n0 += BL)
                for (int k = k0; k < std::min(K, k0 + BL); ++k)
                    for (int n = n0; n < std::min(N, n0 + BL); ++n) t[(size_t)n * K + k] = w.data[(size_t)k * N + n];
    } else {
        std::memcpy(t.data(), w.data.data(), (size_t)N * K * sizeof(float));
    }
    lin.N = Np; lin.K = K;
    std::vector<float> bias(Np, 0.f);
    if (!bname.empty()) { const HostTensor& b = need(bname); std::copy(b.data.begin(), b.data.end(), bias.begin()); }
    lin.b.alloc(Np); lin.b.upload(bias.data(), Np, st);
    lin.w32.alloc(t.size()); lin.w32.upload(t.data(), t.size(), st);
    if (bf16) {
        lin.w16.alloc(t.size());
        if (f16) launch_f32_to_f16(lin.w32.p, reinterpret_cast<__half*>(lin.w16.p), t.size(), st);
        else launch_f32_to_bf16(lin.w32.p, lin.w16.p, t.size(), st);
        CUDA_CHECK(cudaStreamSynchronize(st));
        lin.w32.release();
        weight_bytes += t.size() * 2;
    } else {
        CUDA_CHECK(cudaStreamSynchronize(st));
        weight_bytes += t.size() * 4;
    }
}

// weight-norm fold (torch parametrizations.weight.original0/1, dim 0) — hifigan_decoder.py:44-73,189-202
std::vector<float> Engine::folded(const std::string& prefix) const {
    auto it = raw.find(prefix + ".weight");
    if (it != raw.end()) return it->second.data;
    const HostTensor& g = need(prefix + ".parametrizations.weight.original0");
    const HostTensor& v = need(prefix + ".parametrizations.weight.original1");
    const size_t d0 = (size_t)v.shape[0];
    const size_t inner = v.numel() / d0;
    std::vector<float> w(v.numel());
    for (size_t i = 0; i < d0; ++i) {
        double ss = 0;
        for (size_t j = 0; j < inner; ++j) { const double x = v.data[i * inner + j]; ss += x * x; }
        const float scale = g.data[i] / (float)std::sqrt(ss);
        for (size_t j = 0; j < inner; ++j) w[i * inner + j] = v.data[i * inner + j] * scale;
    }
    return w;
}

// Conv1d weight [Cout,Cin,K] or ConvTranspose1d weight [Cin,Cout,K] -> [Cin][K][Cout]
void Engine::make_conv(ConvW& c, const std::string& prefix, bool transposed, bool has_bias) {
    const std::vector<float> w = folded(prefix);
    const HostTensor& ref = raw.count(prefix + ".weight") ? need(prefix + ".weight")
                                                          : need(prefix + ".parametrizations.weight.original1");
    const int d0 = (int)ref.shape[0], d1 = (int)ref.shape[1], K = (int)ref.shape[2];
    const int Cin = transposed ? d0 : d1, Cout = transposed ? d1 : d0;
    std::vector<float> t((size_t)Cin * K * Cout);
    for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
            for (int j = 0; j < K; ++j) {
                const float x = transposed ? w[((size_t)ci * Cout + co) * K + j] : w[((size_t)co * Cin + ci) * K + j];
                t[((size_t)ci * K + j) * Cout + co] = x;
            }
    c.Cin = Cin; c.Cout = Cout; c.K = K;
    up(c.wt, t);
    if (has_bias) up(c.b, need(prefix + ".bias").data);
    if (bf16 && transposed && K % 2 == 0 && Cout % 32 == 0) {      // fast mode: ConvTranspose1d as u two-tap phases
        const int u = K / 2;
        c.plan = conv1d_tc_plan(Cin, u * Cout, 2);
        if (c.plan.ok) {
            std::vector<__half> blob(c.plan.blob_halves);
            convT_tc_pack(w.data(), Cin, Cout, u, c.plan, blob.data());
            c.blob.alloc(blob.size());
            c.blob.upload(blob.data(), blob.size(), st);
            CUDA_CHECK(cudaStreamSynchronize(st));
            c.tc = true;
            weight_bytes += blob.size() * 2;
        }
    }
    if (bf16 && !transposed) {               // fast mode: fp16 tensor-core tiles for every Conv1d that fits the plan
        c.plan = conv1d_tc_plan(Cin, Cout, K);
        if (c.plan.ok) {
            std::vector<__half> blob(c.plan.blob_halves);
            conv1d_tc_pack(w.data(), Cin, Cout, K, c.plan, blob.data());
            c.blob.alloc(blob.size());
            c.blob.upload(blob.data(), blob.size(), st);
            CUDA_CHECK(cudaStreamSynchronize(st));
            c.tc = true;
            weight_bytes += blob.size() * 2;
        }
    }
}

void Engine::finalize_weights() {
    ApiLock lk(this);
    if (finalized) return;
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const auto& c = cfg;
    // ---- GPT (names: checkpoint_converter.py:230-272)
    up(text_emb, need("text_embedding.weight").data);
    up(text_pos, need("text_pos_embedding.emb.weight").data);
    up(wte, need("gpt.wte.weight").data);
    up(wpe, need("gpt.wpe.emb.weight").data);
    if ((int)need("gpt.wpe.emb.weight").shape[0] < c.max_audio_tokens + 1) throw std::runtime_error("wpe table too short");
    for (int i = 0; i < L; ++i) {
        const std::string p = "gpt.h." + std::to_string(i) + ".";
        std::unique_ptr<Layer> ly(new Layer());
        up(ly->ln1w, need(p + "ln_1.weight").data); up(ly->ln1b, need(p + "ln_1.bias").data);
        up(ly->ln2w, need(p + "ln_2.weight").data); up(ly->ln2b, need(p + "ln_2.bias").data);
        make_linear(ly->qkv, p + "attn.c_attn.weight", p + "attn.c_attn.bias", true);
        make_linear(ly->o, p + "attn.c_proj.weight", p + "attn.c_proj.bias", true);
        make_linear(ly->fc, p + "mlp.c_fc.weight", p + "mlp.c_fc.bias", true);
        make_linear(ly->proj, p + "mlp.c_proj.weight", p + "mlp.c_proj.bias", true);
        if (ly->qkv.N != 3 * H || ly->qkv.K != H || ly->fc.N != FF || ly->proj.K != FF) throw std::runtime_error("GPT weight shape mismatch at layer " + std::to_string(i));
        layers.push_back(std::move(ly));
        // free host copies early (1.5 GB for the full model)
        for (const char* nm : {"attn.c_attn.weight", "attn.c_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight"}) raw.erase(p + nm);
    }
    up(lnfw, need("gpt.ln_f.weight").data); up(lnfb, need("gpt.ln_f.bias").data);
    up(fnw, need("final_norm.weight").data); up(fnb, need("final_norm.bias").data);
    make_linear(mel_head, "mel_head.weight", "mel_head.bias", false, Vpad);
    // ---- vocoder (names: XTTSv2Engine.state_dict(), hifigan_decoder.*)
    const std::string w = "hifigan_decoder.waveform_decoder.";
    make_conv(conv_pre, w + "conv_pre", false, true);
    {
        const HostTensor& cw = need(w + "cond_layer.weight");
        cond_layer.rows = (int)cw.shape[0];
        up(cond_layer.w, cw.data); up(cond_layer.b, need(w + "cond_layer.bias").data);
    }
    const int nk = c.voc_n_rb;
    for (int i = 0; i < c.voc_n_up; ++i) {
        std::unique_ptr<ConvW> u(new ConvW());
        make_conv(*u, w + "ups." + std::to_string(i), true, true);
        ups.push_back(std::move(u));
        std::unique_ptr<CondLin> cl(new CondLin());
        const HostTensor& cw = need(w + "conds." + std::to_string(i) + ".weight");
        cl->rows = (int)cw.shape[0];
        up(cl->w, cw.data); up(cl->b, need(w + "conds." + std::to_string(i) + ".bias").data);
        conds.push_back(std::move(cl));
        for (int j = 0; j < nk; ++j) {
            std::unique_ptr<RB> rb(new RB());
            const std::string rp = w + "resblocks." + std::to_string(i * nk + j) + ".";
            for (int t = 0; t < 3; ++t) {
                rb->c1[t].reset(new ConvW()); rb->c2[t].reset(new ConvW());
                make_conv(*rb->c1[t], rp + "convs1." + std::to_string(t), false, true);
                make_conv(*rb->c2[t], rp + "convs2." + std::to_string(t), false, true);
            }
            rbs.push_back(std::move(rb));
        }
    }
    {
        const HostTensor& pw = need(w + "conv_post.weight");
        post_cin = (int)pw.shape[1];
        up(conv_post_w, pw.data);
    }
    if (bf16) {
        bool all_tc = conv_pre.tc;
        for (auto& u : ups) all_tc = all_tc && u->tc && (u->K == 2 * c.voc_up_rates[&u - &ups[0]]);
        for (auto& rb : rbs) for (int t = 0; t < 3; ++t) all_tc = all_tc && rb->c1[t]->tc && rb->c2[t]->tc;
        for (int ch : stage_ch) all_tc = all_tc && (ch % 16 == 0);
        if (all_tc) {
            // atoms carry up to 640 pad rows per plane, which weighs more the shorter the windows: size the buffers for the
            // three batch shapes the scheduler forms most (n whole chunks, 2n half-length, 4n quarter-length windows)
            const int nfull = (int)(voc_cap_z / voc_max_Tz);
            vz16_halves = va16_halves = 0;
            for (int f = 1; f <= 4; f *= 2) {
                const int nb = std::min(nfull * f, kVocMaxItems), Lz = ceil_div(voc_max_Tz, f);
                vz16_halves = std::max(vz16_halves, (size_t)nb * c.voc_in_dim * atoms_lpad(Lz));
                size_t mx = (size_t)c.voc_init_ch * atoms_lpad(Lz); int len = Lz;
                for (int i = 0; i < c.voc_n_up; ++i) { len *= c.voc_up_rates[i]; mx = std::max(mx, (size_t)stage_ch[i] * atoms_lpad(len)); }
                va16_halves = std::max(va16_halves, (size_t)nb * mx);
            }
            vz16.alloc(vz16_halves);
            for (auto& b : va16) b.alloc(va16_halves);
            tc_vocoder_ready = true;
        }
    }
    compute_voc_margin(conv_pre.K);
    CUDA_CHECK(cudaStreamSynchronize(st));
    // ---- speaker conditioning stack (optional in a checkpoint: without it only xtts_set_speaker works)
    if (raw.count("conditioning_encoder.init.weight") && raw.count("hifigan_decoder.speaker_encoder.conv1.weight")) {
        auto get = [this](const std::string& n) {
            const HostTensor& t = need(n);
            return HostTensorView{t.data.data(), t.shape};
        };
        conditioner.reset(new Conditioner(cfg, get, st));
    }
    raw.clear();
    finalized = true;
}

// ================================================================================================
// speakers
// ================================================================================================
void Engine::set_speaker(int slot, const float* cond, const float* g) {
    ApiLock lk(this);
    require_finalized();
    if (slot < 0 || slot >= S) throw std::runtime_error("speaker slot out of range");
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const size_t nc = (size_t)cfg.n_cond_latents * H;
    spk_cond.upload(cond, nc, st, (size_t)slot * nc);
    spk_g.upload(g, cfg.d_vector, st, (size_t)slot * cfg.d_vector);
    // speaker-conditioning biases: cond_layer(g), conds[i](g)  (hifigan_decoder.py:244-251)
    finish_speaker(slot);
}

void Engine::finish_speaker(int slot) {
    const float* gd = spk_g.p + (size_t)slot * cfg.d_vector;
    float* cb = spk_cbias.p + (size_t)slot * cbias_stride;
    launch_gemv(cond_layer.w.p, cond_layer.b.p, gd, cb + cbias_off[0], cond_layer.rows, cfg.d_vector, st);
    for (int i = 0; i < cfg.voc_n_up; ++i)
        launch_gemv(conds[i]->w.p, conds[i]->b.p, gd, cb + cbias_off[i + 1], conds[i]->rows, cfg.d_vector, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    spk_valid[slot] = 1;
}

// get_conditioning_latents (XTTSv2.py:409-468) on the GPU
void Engine::condition(int slot, const float* w22, int64_t n22, const float* w16, int64_t n16, int cond_len, int chunk_len) {
    ApiLock lk(this);
    require_finalized();
    if (!conditioner) throw std::runtime_error("checkpoint has no conditioning encoder / speaker encoder weights");
    if (slot < 0 || slot >= S) throw std::runtime_error("speaker slot out of range");
    if (cfg.spk_proj != cfg.d_vector) throw std::runtime_error("speaker encoder projection != d_vector");
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    conditioner->run(w22, n22, w16, n16, cond_len, chunk_len, spk_cond.p + (size_t)slot * cfg.n_cond_latents * H,
                     spk_g.p + (size_t)slot * cfg.d_vector);
    finish_speaker(slot);
    st_cond_ms += (now_s() - t0) * 1e3;
}

// TTSRequest.enhance_speech (requests.py:199-248): the reference's audio enhancer, on the conditioning stream
int64_t Engine::enhance(const float* wav, int64_t n, const xtts_enhance_config& c, float* out, int64_t cap) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    if (!enhancer) enhancer.reset(new Enhancer(st));
    const int64_t n_out = enhancer->run(wav, n, c, out, cap);
    st_cond_ms += (now_s() - t0) * 1e3;
    return n_out;
}

// TTSOutput.change_speed (output.py:40-92): the reference's phase-vocoder time stretch, on the conditioning stream
int64_t Engine::change_speed(const float* wav, int64_t n, double rate, float* out, int64_t cap) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    if (!pvoc) pvoc.reset(new PhaseVocoder(st));
    const int64_t n_out = pvoc->run(wav, n, rate, out, cap, pvoc_block_frames);
    st_cond_ms += (now_s() - t0) * 1e3;
    return n_out;
}

// torchaudio.functional.resample (common/utilities.py:94, XTTSv2.py:322,362, TTSOutput.resample), on the conditioning stream
int64_t Engine::resample(const float* wav, int64_t n, int orig_sr, int new_sr, float* out, int64_t cap) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    if (!resampler) resampler.reset(new Resampler(st));
    const int64_t n_out = resampler->run(wav, n, orig_sr, new_sr, out, cap, resample_block_samples);
    st_cond_ms += (now_s() - t0) * 1e3;
    return n_out;
}

// TTSOutput.to_bytes("flac") (output.py:119-187): a lossless FLAC stream of 16-bit PCM, on the conditioning stream
int64_t Engine::encode_flac(const int16_t* pcm, int64_t n, int sample_rate, const uint8_t* md5, uint8_t* out,
                            int64_t cap, int64_t* n_out) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    if (!flac) flac.reset(new FlacEncoder(st));
    const int64_t n_bytes = flac->run(pcm, n, sample_rate, md5, out, cap, flac_batch_frames, n_out);
    st_cond_ms += (now_s() - t0) * 1e3;
    return n_bytes;
}

// FLAC input (engine.load_audio, TTSOutput.from_file): a FLAC stream -> planar int32 samples, on the conditioning stream
int64_t Engine::decode_flac(const uint8_t* data, int64_t n, int32_t* out, int64_t cap, xtts_flac_info* info) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const double t0 = now_s();
    if (!flac_dec) flac_dec.reset(new FlacDecoder(st));
    const int64_t total = flac_dec->run(data, n, out, cap, flac_batch_frames, info);
    st_cond_ms += (now_s() - t0) * 1e3;
    return total;
}

void Engine::get_speaker(int slot, float* cond, float* g) {
    ApiLock lk(this);
    if (slot < 0 || slot >= S || !spk_valid[slot]) throw std::runtime_error("speaker slot not set");
    CUDA_CHECK(cudaSetDevice(cfg.device));
    const size_t nc = (size_t)cfg.n_cond_latents * H;
    if (cond) spk_cond.download(cond, nc, st, (size_t)slot * nc);
    if (g) spk_g.download(g, cfg.d_vector, st, (size_t)slot * cfg.d_vector);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ================================================================================================
// GPT forward
// ================================================================================================
SampleState Engine::sample_state() const {
    SampleState s;
    s.last_tok = d_last_tok.p; s.n_gen = d_n_gen.p; s.ctx_len = d_ctx_len.p; s.finished = d_finished.p;
    s.tokens = d_tokens.p; s.sampled = d_sampled.p; s.forced = use_forced ? d_forced.p : nullptr;
    s.seen = d_seen.p; s.temperature = d_temp.p; s.top_p = d_top_p.p; s.top_k = d_top_k.p; s.penalty = d_pen.p;
    s.max_tokens = d_max_tokens.p; s.stop_token = d_stop.p; s.seed = d_seed.p; s.seq_seed = d_seq_seed.p;
    s.beam = d_beam_flag.p;
    s.tokens_cap = CAP; s.seen_words = SEENW;
    return s;
}

void Engine::gemm(const void* A, const Linear& lin, const float* resid, void* out, int M, int flags, bool pdl) {
    if (bf16)
        launch_gemm_bf16_tc(reinterpret_cast<const __nv_bfloat16*>(A), lin.w16.p, lin.b.p, resid, out, M, lin.N, lin.K, flags | gflag, st, pdl);
    else
        launch_gemm_f32(reinterpret_cast<const float*>(A), lin.w32.p, lin.b.p, resid, reinterpret_cast<float*>(out), M, lin.N, lin.K,
                        flags & ~GEMM_OUT_BF16, st);
}

// X [M,H] -> X after all blocks.  prefill: causal attention inside each sequence of d_attnseq, KV written at
// d_row_pos; decode: one row per active slot, KV appended at ctx_len, attention over the paged cache.
void Engine::layers_forward(int M, bool prefill, int nseq, int max_nq) {
    void* Xn = bf16 ? (void*)wXn16.p : (void*)wXn32.p;
    void* ATT = bf16 ? (void*)wATT16.p : (void*)wATT32.p;
    void* FFb = bf16 ? (void*)wFF16.p : (void*)wFF32.p;
    const int oflag = bf16 ? GEMM_OUT_BF16 : 0;
    // Decode-shaped steps in fast mode: the two N = hidden GEMMs (attention out-proj, MLP down-proj) expose only
    // N/BN CTAs, so they run split-K into fp32 partials and the reduction is fused with the residual add and the
    // following LayerNorm (fixed summation order => deterministic).
    const bool splitk = bf16 && !prefill && use_splitk && M <= NSLOT && (H / 64) % 4 == 0 && (FF / 64) % 8 == 0;
    const bool pdl = !prefill && use_pdl;            // decode chain: programmatic dependent launch
    auto ln = [&](const float* w, const float* b) {
        if (f16) launch_layernorm<__half>(wX.p, w, b, reinterpret_cast<__half*>(wXn16.p), M, H, cfg.ln_eps, st, pdl);
        else if (bf16) launch_layernorm<__nv_bfloat16>(wX.p, w, b, wXn16.p, M, H, cfg.ln_eps, st, pdl);
        else launch_layernorm<float>(wX.p, w, b, wXn32.p, M, H, cfg.ln_eps, st, pdl);
    };
    if (splitk) ln(layers[0]->ln1w.p, layers[0]->ln1b.p);
    for (int l = 0; l < L; ++l) {
        Layer& ly = *layers[l];
        if (!splitk) ln(ly.ln1w.p, ly.ln1b.p);
        gemm(Xn, ly.qkv, nullptr, wQKV.p, M, 0, pdl);
        if (prefill) {
            if (kv_fp8) launch_kv_write<__nv_fp8_e4m3>(wQKV.p, M, d_row_slot.p, d_row_pos.p, d_ctx_len.p, d_block_tables.p, max_pages, k8p(l), v8p(l), NH, st);
            else if (f16) launch_kv_write<__half>(wQKV.p, M, d_row_slot.p, d_row_pos.p, d_ctx_len.p, d_block_tables.p, max_pages, reinterpret_cast<__half*>(k16[l]->p), reinterpret_cast<__half*>(v16[l]->p), NH, st);
            else if (bf16) launch_kv_write<__nv_bfloat16>(wQKV.p, M, d_row_slot.p, d_row_pos.p, d_ctx_len.p, d_block_tables.p, max_pages, k16[l]->p, v16[l]->p, NH, st);
            else launch_kv_write<float>(wQKV.p, M, d_row_slot.p, d_row_pos.p, d_ctx_len.p, d_block_tables.p, max_pages, k32[l]->p, v32[l]->p, NH, st);
            AttnLayout A;
            A.q = wQKV.p; A.k = wQKV.p + H; A.v = wQKV.p + 2 * H;
            A.q_row_stride = 3 * H; A.kv_row_stride = 3 * H; A.q_head_stride = kHeadDim; A.kv_head_stride = kHeadDim;
            A.heads = NH; A.scale = 0.125f; A.causal = 1;
            if (f16) launch_attn_generic<__half>(A, d_attnseq.p, nseq, max_nq, reinterpret_cast<__half*>(wATT16.p), H, st);
            else if (bf16) launch_attn_generic<__nv_bfloat16>(A, d_attnseq.p, nseq, max_nq, wATT16.p, H, st);
            else launch_attn_generic<float>(A, d_attnseq.p, nseq, max_nq, wATT32.p, H, st);
        } else {
            // (the attention kernel appends this step's K/V to the cache itself)
            if (kv_fp8 && f16) launch_attn_decode<__nv_fp8_e4m3, __half>(wQKV.p, d_active.p, M, d_ctx_len.p, d_block_tables.p, max_pages, k8p(l), v8p(l), reinterpret_cast<__half*>(wATT16.p), NH, st, decode_ctx_sum, pdl);
            else if (kv_fp8) launch_attn_decode<__nv_fp8_e4m3, __nv_bfloat16>(wQKV.p, d_active.p, M, d_ctx_len.p, d_block_tables.p, max_pages, k8p(l), v8p(l), wATT16.p, NH, st, decode_ctx_sum, pdl);
            else if (f16) launch_attn_decode<__half, __half>(wQKV.p, d_active.p, M, d_ctx_len.p, d_block_tables.p, max_pages, reinterpret_cast<__half*>(k16[l]->p), reinterpret_cast<__half*>(v16[l]->p), reinterpret_cast<__half*>(wATT16.p), NH, st, decode_ctx_sum, pdl);
            else if (bf16) launch_attn_decode<__nv_bfloat16, __nv_bfloat16>(wQKV.p, d_active.p, M, d_ctx_len.p, d_block_tables.p, max_pages, k16[l]->p, v16[l]->p, wATT16.p, NH, st, decode_ctx_sum, pdl);
            else launch_attn_decode<float, float>(wQKV.p, d_active.p, M, d_ctx_len.p, d_block_tables.p, max_pages, k32[l]->p, v32[l]->p, wATT32.p, NH, st, decode_ctx_sum, pdl);
        }
        if (splitk) {
            launch_gemm_bf16_tc_splitk(wATT16.p, ly.o.w16.p, wPART.p, M, H, H, 4, st, pdl, gflag);
            reduce_ln16(wX.p, wPART.p, 4, ly.o.b.p, ly.ln2w.p, ly.ln2b.p, wXn16.p, M, st, pdl);
            gemm(Xn, ly.fc, nullptr, FFb, M, GEMM_GELU | oflag, pdl);
            launch_gemm_bf16_tc_splitk(wFF16.p, ly.proj.w16.p, wPART.p, M, H, FF, 8, st, pdl, gflag);
            const bool last = (l + 1 == L);
            reduce_ln16(wX.p, wPART.p, 8, ly.proj.b.p, last ? nullptr : layers[l + 1]->ln1w.p,
                        last ? nullptr : layers[l + 1]->ln1b.p, last ? nullptr : wXn16.p, M, st, pdl);
        } else {
            gemm(ATT, ly.o, wX.p, wX.p, M, GEMM_RESID, pdl);
            ln(ly.ln2w.p, ly.ln2b.p);
            gemm(Xn, ly.fc, nullptr, FFb, M, GEMM_GELU | oflag, pdl);
            gemm(FFb, ly.proj, wX.p, wX.p, M, GEMM_RESID, pdl);
        }
    }
}

// rows row_index[0..M) of X -> Y -> logits (wLOG[i]) ; latents captured ; optionally sample
void Engine::head_and_sample(int M, const int* row_index, const int* slots_dev, const int* lat_pos, int advance_ctx, bool do_sample,
                             bool pdl_first) {
    const bool pdl = advance_ctx && use_pdl;         // decode step only
    const bool pdl0 = pdl && pdl_first;              // (the first kernel after a stream join takes a full dependency)
    if (f16) launch_head_norms<__half>(wX.p, row_index, lnfw.p, lnfb.p, fnw.p, fnb.p, reinterpret_cast<__half*>(wY16.p), d_latents.p, slots_dev, lat_pos, d_n_gen.p, CAP, M, H, cfg.ln_eps, st, pdl0);
    else if (bf16) launch_head_norms<__nv_bfloat16>(wX.p, row_index, lnfw.p, lnfb.p, fnw.p, fnb.p, wY16.p, d_latents.p, slots_dev, lat_pos, d_n_gen.p, CAP, M, H, cfg.ln_eps, st, pdl0);
    else launch_head_norms<float>(wX.p, row_index, lnfw.p, lnfb.p, fnw.p, fnb.p, wY32.p, d_latents.p, slots_dev, lat_pos, d_n_gen.p, CAP, M, H, cfg.ln_eps, st, pdl0);
    gemm(bf16 ? (void*)wY16.p : (void*)wY32.p, mel_head, nullptr, wLOG.p, M, 0, pdl);
    if (do_sample) launch_sample(wLOG.p, Vpad, slots_dev, M, V, sample_state(), advance_ctx, st, pdl);
}

// Slot state of an admission wave: KV pages are taken here, everything the device needs goes up in one staged copy and
// one kernel (launch_init_slots).  `forced` (debug entry points, one sequence): teacher-forced token ids.
void Engine::init_slots(const std::vector<Sequence*>& seqs, const int32_t* forced, int n_forced) {
    if (seqs.empty()) return;
    int n = 0;
    for (auto* sq : seqs) n += std::max(1, (int)sq->beam_slots.size());
    if (n > NSLOT) throw std::runtime_error("init_slots: wave larger than the slot count");
    std::vector<std::pair<Sequence*, int>> groups;      // beam groups of the wave and their prompt pages
    for (int i = 0, r = 0; i < (int)seqs.size(); ++i) {
        Sequence& s = *seqs[i];
        s.n_prompt = cfg.n_cond_latents + (int)s.text_ids.size() + 1;
        s.max_tok = std::min<int>(s.sp.max_tokens > 0 ? s.sp.max_tokens : CAP, CAP);
        const int need_pages = ceil_div(s.n_prompt + s.max_tok, kPageTokens);
        const int nb = std::max(1, (int)s.beam_slots.size());
        // a beam group takes nb x need_pages at once: beam 0 starts with the prompt's pages, the rest form the group's pool
        const int n_pages = nb == 1 ? need_pages : ceil_div(s.n_prompt, kPageTokens);
        if ((int)free_pages.size() < nb * need_pages) throw std::runtime_error("out of KV pages");
        s.pages.clear();
        for (int k = 0; k < nb * need_pages; ++k) { s.pages.push_back(free_pages.back()); free_pages.pop_back(); }
        if (nb > 1) groups.emplace_back(&s, n_pages);
        for (int b = 0; b < nb; ++b, ++r) {
            int* pg = h_slot_pages + (size_t)r * max_pages;
            SlotInit& d = h_slot_init[r];
            d.slot = nb == 1 ? s.slot : s.beam_slots[b]; d.ctx_len = s.n_prompt; d.top_k = s.sp.top_k; d.max_tokens = s.max_tok;
            d.stop_token = s.sp.stop_token; d.seq_seed = s.sp.seq_seed; d.start_token = cfg.start_audio_token;
            d.n_pages = b == 0 ? n_pages : 0; d.beam = nb > 1;
            for (int k = 0; k < d.n_pages; ++k) pg[k] = s.pages[k];
            d.temperature = s.sp.temperature; d.top_p = s.sp.top_p; d.penalty = s.sp.repetition_penalty; d.seed = s.sp.seed;
        }
    }
    d_slot_init.upload(h_slot_init, n, st);
    d_slot_pages.upload(h_slot_pages, (size_t)n * max_pages, st);
    SlotArrays a{};
    a.last_tok = d_last_tok.p; a.n_gen = d_n_gen.p; a.ctx_len = d_ctx_len.p; a.finished = d_finished.p; a.seen = d_seen.p;
    a.temperature = d_temp.p; a.top_p = d_top_p.p; a.top_k = d_top_k.p; a.penalty = d_pen.p; a.max_tokens = d_max_tokens.p;
    a.stop_token = d_stop.p; a.seed = d_seed.p; a.seq_seed = d_seq_seed.p; a.block_tables = d_block_tables.p;
    a.beam = d_beam_flag.p;
    a.seen_words = SEENW; a.max_pages = max_pages;
    launch_init_slots(d_slot_init.p, d_slot_pages.p, n, a, st);
    for (size_t gi = 0; gi < groups.size(); ++gi) {
        // group state as transformers initialises it: no finished hypothesis (-1e9), heuristic unsatisfied
        Sequence& s = *groups[gi].first;
        BeamState& bs = h_beam_init[gi];
        bs = BeamState{};
        for (int j = 0; j < kMaxBeams; ++j) bs.fin_score[j] = -1e9f;
        bs.heur_unsat = 1;
        bs.n_pages[0] = groups[gi].second;
        bs.n_free = (int)s.pages.size() - groups[gi].second;
        int* pool = h_beam_pool + gi * beam_pool_cap;
        std::copy(s.pages.begin() + groups[gi].second, s.pages.end(), pool);
        d_beam_state.upload(&bs, 1, st, (size_t)s.slot);
        d_beam_pool.upload(pool, bs.n_free, st, (size_t)s.slot * beam_pool_cap);
    }
    if (forced) {
        std::vector<int> f(CAP, -1);
        for (int i = 0; i < std::min(n_forced, CAP); ++i) f[i] = forced[i];
        d_forced.upload(f.data(), CAP, st, (size_t)seqs[0]->slot * CAP);
        CUDA_CHECK(cudaStreamSynchronize(st));     // `f` goes out of scope
    }
    // (the pinned staging is reused by the next wave: prefill() synchronizes the stream before the scheduler gets there)
}

void Engine::release_pages(Sequence& s) {
    for (int p : s.pages) free_pages.push_back(p);
    s.pages.clear();
}

void Engine::release_slot(Sequence& s) {
    release_pages(s);
    for (size_t b = 1; b < s.beam_slots.size(); ++b) free_slots.push_back(s.beam_slots[b]);
    if (s.beam_slots.size() > 1) s.beam_slots.resize(1);
    if (s.slot >= 0 && s.slot < B) free_slots.push_back(s.slot);
    s.slot = -1;
}

// The beam kernels of one step for `groups` (running beam groups), after the prefill (first: every beam reads the
// group's prefill row rows0[g]) or after a decode step (beam j reads the row of its slot in d_active)
void Engine::beam_step(const std::vector<Sequence*>& groups, const std::vector<int>& rows0, bool first) {
    if (groups.empty()) return;
    for (size_t g = 0; g < groups.size(); ++g) {
        const Sequence& s = *groups[g];
        BeamDesc& d = h_beam_desc[g];
        d.primary = s.slot; d.nb = (int)s.beam_slots.size(); d.first = first; d.advance = first ? 0 : 1;
        d.do_sample = s.beam.do_sample != 0; d.length_penalty = s.beam.length_penalty;
        for (int j = 0; j < kMaxBeams; ++j) {
            d.slot[j] = j < d.nb ? s.beam_slots[j] : -1;
            d.row[j] = j < d.nb ? (first ? rows0[g] : rows0[g] + j) : 0;
        }
    }
    d_beam_desc.upload(h_beam_desc, groups.size(), st);
    BeamArgs a{};
    a.desc = d_beam_desc.p; a.n_groups = (int)groups.size(); a.state = d_beam_state.p; a.hist = d_beam_hist.p;
    a.pool = d_beam_pool.p; a.pool_cap = beam_pool_cap; a.scores = d_beam_scores.p; a.block_tables = d_block_tables.p;
    a.max_pages = max_pages; a.latents = d_latents.p; a.H = H;
    launch_beam_step(wLOG.p, Vpad, V, sample_state(), a, d_kv_ptrs.p, d_kv_ptrs.p + L, L, NH, kv_fp8 ? 1 : bf16 ? 2 : 4, st);
}

// builds row descriptors for [prompt ; optional forced audio rows] of each sequence; returns total rows
int Engine::build_prefill(const std::vector<Sequence*>& seqs, const std::vector<std::vector<int32_t>>& audio,
                          std::vector<int>& last_rows, int& max_nq) {
    std::vector<RowDesc> rows;
    std::vector<int> row_slot, row_pos;
    std::vector<AttnSeq> as;
    last_rows.clear();
    max_nq = 0;
    for (size_t si = 0; si < seqs.size(); ++si) {
        Sequence& s = *seqs[si];
        const int start = (int)rows.size();
        for (int i = 0; i < cfg.n_cond_latents; ++i) rows.push_back(RowDesc{0, i, 0, s.speaker});
        for (int i = 0; i < (int)s.text_ids.size(); ++i) {
            const int id = s.text_ids[i];
            if (id < 0 || id >= cfg.n_text_tokens) throw std::runtime_error("text token id out of range");
            rows.push_back(RowDesc{1, id, i, 0});
        }
        rows.push_back(RowDesc{2, cfg.start_audio_token, 0, 0});
        if (si < audio.size())
            for (int k = 0; k < (int)audio[si].size(); ++k) {
                const int id = audio[si][k];
                if (id < 0 || id >= V) throw std::runtime_error("audio token id out of range");
                rows.push_back(RowDesc{2, id, k + 1, 0});
            }
        const int n = (int)rows.size() - start;
        for (int i = 0; i < n; ++i) { row_slot.push_back(s.slot); row_pos.push_back(i); }
        as.push_back(AttnSeq{start, n, start, n});
        last_rows.push_back(start + n - 1);
        max_nq = std::max(max_nq, n);
    }
    const int M = (int)rows.size();
    if (M > prefill_rows_cap) throw std::runtime_error("prefill batch exceeds row budget");
    d_rows.upload(rows.data(), M, st); d_row_slot.upload(row_slot.data(), M, st); d_row_pos.upload(row_pos.data(), M, st);
    d_attnseq.upload(as.data(), as.size(), st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    return M;
}

void Engine::prefill(const std::vector<Sequence*>& seqs) {
    std::vector<int> last_rows; int max_nq = 0;
    const int M = build_prefill(seqs, {}, last_rows, max_nq);
    launch_build_rows(d_rows.p, M, tables(), wX.p, st);
    layers_forward(M, true, (int)seqs.size(), max_nq);
    std::vector<int> slots;
    for (auto* s : seqs) slots.push_back(s->slot);
    d_rowidx.upload(last_rows.data(), last_rows.size(), st);
    d_active.upload(slots.data(), slots.size(), st);
    head_and_sample((int)seqs.size(), d_rowidx.p, d_active.p, nullptr, 0, true);
    CUDA_CHECK(cudaStreamSynchronize(st));
    st_prefill_rows += M;
    const double t = now_s();
    for (auto* s : seqs) s->t_first = t;
}

// Fast-mode decode layers for rows [r0, r0 + Mi) of the step on stream `s`.  Every work buffer is row-major and the
// KV cache is per slot, so disjoint row ranges are independent: decode_step runs several of these as concurrent
// branches (micro-batches), which lets one branch's HBM-bound attention overlap another's latency-bound GEMM chain.
void Engine::decode_layers_rows(int r0, int Mi, cudaStream_t s, bool pdl_first, double ctx_sum) {
    float* X = wX.p + (size_t)r0 * H;
    __nv_bfloat16* Xn = wXn16.p + (size_t)r0 * H;
    float* QKV = wQKV.p + (size_t)r0 * 3 * H;
    __nv_bfloat16* ATT = wATT16.p + (size_t)r0 * H;
    __nv_bfloat16* FFb = wFF16.p + (size_t)r0 * FF;
    float* PART = wPART.p + (size_t)r0 * 8 * H;          // [splits <= 8][Mi][H] inside this branch's own region
    const int* act = d_active.p + r0;
    const bool pdl = use_pdl;
    if (f16) launch_layernorm<__half>(X, layers[0]->ln1w.p, layers[0]->ln1b.p, reinterpret_cast<__half*>(Xn), Mi, H, cfg.ln_eps, s, pdl && pdl_first);
    else launch_layernorm<__nv_bfloat16>(X, layers[0]->ln1w.p, layers[0]->ln1b.p, Xn, Mi, H, cfg.ln_eps, s, pdl && pdl_first);
    for (int l = 0; l < L; ++l) {
        Layer& ly = *layers[l];
        launch_gemm_bf16_tc(Xn, ly.qkv.w16.p, ly.qkv.b.p, nullptr, QKV, Mi, ly.qkv.N, ly.qkv.K, gflag, s, pdl);
        if (kv_fp8 && f16)
            launch_attn_decode<__nv_fp8_e4m3, __half>(QKV, act, Mi, d_ctx_len.p, d_block_tables.p, max_pages, k8p(l), v8p(l),
                                                      reinterpret_cast<__half*>(ATT), NH, s, ctx_sum, pdl);
        else if (kv_fp8)
            launch_attn_decode<__nv_fp8_e4m3, __nv_bfloat16>(QKV, act, Mi, d_ctx_len.p, d_block_tables.p, max_pages, k8p(l), v8p(l),
                                                             ATT, NH, s, ctx_sum, pdl);
        else if (f16)
            launch_attn_decode<__half, __half>(QKV, act, Mi, d_ctx_len.p, d_block_tables.p, max_pages, reinterpret_cast<__half*>(k16[l]->p),
                                               reinterpret_cast<__half*>(v16[l]->p), reinterpret_cast<__half*>(ATT), NH, s, ctx_sum, pdl);
        else
            launch_attn_decode<__nv_bfloat16, __nv_bfloat16>(QKV, act, Mi, d_ctx_len.p, d_block_tables.p, max_pages, k16[l]->p, v16[l]->p,
                                                             ATT, NH, s, ctx_sum, pdl);
        launch_gemm_bf16_tc_splitk(ATT, ly.o.w16.p, PART, Mi, H, H, 4, s, pdl, gflag);
        reduce_ln16(X, PART, 4, ly.o.b.p, ly.ln2w.p, ly.ln2b.p, Xn, Mi, s, pdl);
        launch_gemm_bf16_tc(Xn, ly.fc.w16.p, ly.fc.b.p, nullptr, FFb, Mi, ly.fc.N, ly.fc.K, GEMM_GELU | GEMM_OUT_BF16 | gflag, s, pdl);
        launch_gemm_bf16_tc_splitk(FFb, ly.proj.w16.p, PART, Mi, H, FF, 8, s, pdl, gflag);
        const bool last = (l + 1 == L);
        reduce_ln16(X, PART, 8, ly.proj.b.p, last ? nullptr : layers[l + 1]->ln1w.p, last ? nullptr : layers[l + 1]->ln1b.p,
                    last ? nullptr : Xn, Mi, s, pdl);
    }
}

void Engine::drop_graphs() {
    for (auto& kv : decode_graphs) cudaGraphExecDestroy(kv.second);
    decode_graphs.clear();
    for (auto& kv : prof_graphs) {
        cudaGraphExecDestroy(kv.second.first);
        for (auto& r : kv.second.second->recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
        delete kv.second.second;
    }
    prof_graphs.clear();
    last_prof = nullptr;
}

void Engine::decode_step(const std::vector<int>& active) {
    const int M = (int)active.size();
    d_active.upload(active.data(), M, st);
    const bool fast = bf16 && use_splitk && M <= NSLOT && (H / 64) % 4 == 0 && (FF / 64) % 8 == 0;
    const int nmb = (fast && n_micro > 1 && M >= micro_min_rows) ? std::min(n_micro, (int)kMaxMicro) : 1;
    auto enqueue = [&] {
        launch_build_decode_rows(d_active.p, M, d_last_tok.p, d_n_gen.p, tables(), wX.p, st, use_pdl);
        if (nmb > 1) {
            // fork: every branch starts after the row build; join: head + sampler run once over all rows
            CUDA_CHECK(cudaEventRecord(ev_fork, st));
            for (int i = 1; i < nmb; ++i) CUDA_CHECK(cudaStreamWaitEvent(st_mb[i], ev_fork, 0));
            for (int i = 0, r0 = 0; i < nmb; ++i) {
                const int Mi = M / nmb + (i < M % nmb ? 1 : 0);
                decode_layers_rows(r0, Mi, st_mb[i], i == 0, decode_ctx_sum * (double)Mi / (double)M);
                r0 += Mi;
            }
            for (int i = 1; i < nmb; ++i) {
                CUDA_CHECK(cudaEventRecord(ev_join[i], st_mb[i]));
                CUDA_CHECK(cudaStreamWaitEvent(st, ev_join[i], 0));
            }
            head_and_sample(M, nullptr, d_active.p, nullptr, 1, true, false);
        } else {
            if (fast) decode_layers_rows(0, M, st, true, decode_ctx_sum);
            else layers_forward(M, false, 0, 0);
            head_and_sample(M, nullptr, d_active.p, nullptr, 1, true);
        }
    };
    // The decode step is ~250 small launches whose arguments depend only on M (slot lists, positions and
    // lengths live in device memory), so it is captured once per batch size into a CUDA graph and replayed.
    // Kernel-family profiling and teacher forcing use the eager path.
    const bool graphable = use_graphs && !use_forced && eager_steps_done >= 2;
    if (!graphable) {
        enqueue();
        ++eager_steps_done;
    } else if (g_prof.enabled) {
        // kernel-family profiling: the same step captured with an event-record node on either side of every kernel
        // (full dependencies instead of PDL edges), replayed, and read back after the step's synchronize
        auto it = prof_graphs.find(M);
        if (it == prof_graphs.end()) {
            cudaGraph_t g = nullptr; cudaGraphExec_t ge = nullptr;
            auto* recs = new KernelProfiler::GraphRecs();
            recs->ctx_sum = decode_ctx_sum;
            const unsigned long long lc = g_launch_count;
            const bool pdl_was = g_use_pdl;
            g_use_pdl = false; g_prof.cap = recs;
            CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            try { enqueue(); }
            catch (...) { g_prof.cap = nullptr; g_use_pdl = pdl_was; cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); delete recs; throw; }
            g_prof.cap = nullptr; g_use_pdl = pdl_was;
            CUDA_CHECK(cudaStreamEndCapture(st, &g));
            CUDA_CHECK(cudaGraphInstantiate(&ge, g, 0));
            cudaGraphDestroy(g);
            graph_kernels[M] = g_launch_count - lc;
            g_launch_count = lc;
            it = prof_graphs.emplace(M, std::make_pair(ge, recs)).first;
        }
        CUDA_CHECK(cudaGraphLaunch(it->second.first, st));
        g_launch_count += graph_kernels[M];
        last_prof = it->second.second;
    } else {
        auto it = decode_graphs.find(M);
        if (it == decode_graphs.end()) {
            cudaGraph_t g = nullptr; cudaGraphExec_t ge = nullptr;
            const unsigned long long lc = g_launch_count;
            CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            try { enqueue(); }
            catch (...) { cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); throw; }
            CUDA_CHECK(cudaStreamEndCapture(st, &g));
            CUDA_CHECK(cudaGraphInstantiate(&ge, g, 0));
            cudaGraphDestroy(g);
            graph_kernels[M] = g_launch_count - lc;
            g_launch_count = lc;                       // capture enqueued nothing on the device
            it = decode_graphs.emplace(M, ge).first;
        }
        CUDA_CHECK(cudaGraphLaunch(it->second, st));
        g_launch_count += graph_kernels[M];            // kernels executed by the replay
    }
    ++st_decode_steps;
}

// ================================================================================================
// vocoder driver  (HifiDecoder.forward, hifigan_decoder.py:776-802 + HifiganGenerator.forward :228-260)
// ================================================================================================
// A batch is `nb` WINDOWS: item i = z-frames [z0, z0 + nz) of a chunk whose latents start at `lat` (device).  A window that
// starts at z-frame 0 / ends at the chunk's last z-frame sees the reference's zero padding there; inner window edges see
// zero padding too, so the caller discards `voc_hz` z-frames of output next to them (receptive field).  Windows of one
// batch may have different lengths: buffers are strided by the longest (Lz), kernels skip what lies beyond an item's end.
// All vocoder work is issued on st_voc.  wav_dev_out: [nb][Lz * hop].
// A speaking rate other than 1 adds one level in front (Xtts.inference: F.interpolate(scale_factor = 1 / speed)): T latents
// become T0 = floor(T * ls) frames, ls = 1 / (double)speed computed from the float32 speed.
int Engine::z_frames(int T, float speed) const {
    if (speed != 1.f) T = (int)std::floor((double)T * (1.0 / (double)speed));
    const double s1 = (double)cfg.code_stride / (double)cfg.output_hop_length;
    const double s2 = (double)cfg.output_sample_rate / (double)cfg.input_sample_rate;
    const int T1 = (int)std::floor((double)T * s1);
    return cfg.output_sample_rate != cfg.input_sample_rate ? (int)std::floor((double)T1 * s2) : T1;
}

// z-frames that can be interpolated from the first n latent frames of a chunk that is still growing, i.e. without touching
// either interpolation's end clamp: z[j] reads y[a0], y[a0 + 1] with a0 = floor((j + .5) / s2 - .5) and y[a] reads
// lat[b0], lat[b0 + 1] with b0 = floor((a + .5) / s1 - .5); one frame of slack on both levels (float rounding).  With a
// speaking rate the latents go through one more level first (same rule, same slack), and the two levels run on its output.
int Engine::z_avail(int n, float speed) const {
    const double s1 = (double)cfg.code_stride / (double)cfg.output_hop_length;
    const bool resample = cfg.output_sample_rate != cfg.input_sample_rate;
    const double s2 = resample ? (double)cfg.output_sample_rate / (double)cfg.input_sample_rate : 1.0;
    int n0 = n;                                                             // frames the y level may read
    if (speed != 1.f) {
        const double ls = 1.0 / (double)speed;
        const int A0 = (int)std::floor(((double)n - 1.5) * ls - 0.5) - 1;   // largest scaled index whose sources are < n - 1
        if (A0 < 1) return 0;
        n0 = A0 + 1;
    }
    const int A = (int)std::floor(((double)n0 - 1.5) * s1 - 0.5) - 1;       // largest y index whose sources are < n0 - 1
    if (A < 1) return 0;
    const int J = (int)std::floor(((double)A - 0.5) * s2 - 0.5) - 1;        // z indices < J read y indices <= A
    return std::max(0, std::min(J, z_frames(n, speed)));
}

int Engine::samples_for(int T, float speed) const { return z_frames(T, speed) * voc_hop; }

// Whether T latents at `speed` go through the speed stage: not at speed 1 (skipped, as Coqui does), and not when
// floor(T * ls) == T either (short chunks at speeds just below 1), where F.interpolate copies its input.  Once true for a
// chunk still growing, it stays true for its final length (T * (ls - 1) >= 1 only grows with T).
bool Engine::speed_stage(int T, float speed) const {
    return speed != 1.f && (int)std::floor((double)T * (1.0 / (double)speed)) != T;
}

// the interpolation launch item of a vocoder window (clamp lengths of every level, the speed stage's T0 / r0)
InterpItem Engine::interp_item(const VocItem& v) const {
    const double s1 = (double)cfg.code_stride / (double)cfg.output_hop_length;
    const bool resample = cfg.output_sample_rate != cfg.input_sample_rate;
    InterpItem ii{v.lat, v.T, 0, v.z0, v.nz};
    int Ty = v.T;                                   // frames the chunk-level interpolations run on
    if (speed_stage(v.T, v.speed)) {
        const double ls = 1.0 / (double)v.speed;
        ii.T0 = Ty = (int)std::floor((double)v.T * ls);
        ii.r0 = (float)(1.0 / ls);
    }
    ii.T1 = resample ? (int)std::floor((double)Ty * s1) : Ty;
    return ii;
}

// The windows that produce z-frames [zk0, Tz) of a finished chunk, none longer than the workspace's voc_max_Tz: each keeps
// [zk0_i, zk1_i) and carries voc_hz frames of margin on its inner edges.  One window unless a speaking rate < 1 stretched
// the chunk past voc_max_Tz; every window but the last is exactly voc_max_Tz long.
std::vector<Engine::VocSpan> Engine::split_windows(int zk0, int Tz) const {
    std::vector<VocSpan> out;
    for (int k0 = zk0;;) {
        const int w0 = std::max(0, k0 - voc_hz);
        if (Tz - w0 <= voc_max_Tz) { out.push_back(VocSpan{w0, Tz, k0, Tz}); break; }
        const int k1 = w0 + voc_max_Tz - voc_hz;
        out.push_back(VocSpan{w0, k1 + voc_hz, k0, k1});
        k0 = k1;
    }
    return out;
}

bool Engine::voc_fits(int nb, int Lz) const {
    if (nb < 1 || nb > kVocMaxItems || Lz < 1 || Lz > voc_max_Tz) return false;
    if ((size_t)nb * Lz > voc_cap_z) return false;
    if (tc_vocoder_ready && use_tc_vocoder) {
        if ((size_t)nb * cfg.voc_in_dim * atoms_lpad(Lz) > vz16_halves) return false;
        size_t mx = (size_t)cfg.voc_init_ch * atoms_lpad(Lz); int len = Lz;
        for (int i = 0; i < cfg.voc_n_up; ++i) { len *= cfg.voc_up_rates[i]; mx = std::max(mx, (size_t)stage_ch[i] * atoms_lpad(len)); }
        if ((size_t)nb * mx > va16_halves) return false;
    }
    return true;
}

void Engine::run_vocoder(const VocItem* it, int nb, float* wav_dev_out, const char* stage, float* stage_out, int64_t stage_cap) {
    if (nb < 1 || nb > kVocMaxItems) throw std::runtime_error("vocoder: batch out of range");
    int Lz = 0, spk[kVocMaxItems];
    for (int i = 0; i < nb; ++i) {
        if (it[i].nz <= 0 || it[i].T <= 0 || it[i].T > voc_max_T) throw std::runtime_error("vocoder: window out of range");
        const int sp = it[i].speaker;
        if (sp < 0 || sp >= S || !spk_valid[sp]) throw std::runtime_error("vocoder: speaker slot not set");
        spk[i] = sp;
        Lz = std::max(Lz, it[i].nz);
    }
    if (!voc_fits(nb, Lz)) throw std::runtime_error("vocoder: batch exceeds the workspace");
    launch_gather_rows(spk_cbias.p, spk, nb, cbias_stride, vcb.p, st_voc);
    if (tc_vocoder_ready && use_tc_vocoder) run_vocoder_tc(it, nb, Lz, wav_dev_out, stage, stage_out, stage_cap);
    else run_vocoder_f32(it, nb, Lz, wav_dev_out, stage, stage_out, stage_cap);
}

// fp32 CUDA-core path (parity mode).  Its kernels take equal-length batches: the items (sorted by length by the caller or
// not) are processed in runs of equal window length, each run one batch through the whole generator.
void Engine::run_vocoder_f32(const VocItem* it, int nb, int Lz, float* wav_dev_out, const char* stage, float* stage_out,
                             int64_t stage_cap) {
    const auto& c = cfg;
    cudaStream_t sv = st_voc;
    const double s1 = (double)c.code_stride / (double)c.output_hop_length;
    const double s2 = (double)c.output_sample_rate / (double)c.input_sample_rate;
    const bool resample = c.output_sample_rate != c.input_sample_rate;
    const int nk = c.voc_n_rb;
    const size_t wav_stride = (size_t)Lz * voc_hop;
    for (int i0 = 0; i0 < nb;) {
        int i1 = i0 + 1;
        while (i1 < nb && it[i1].nz == it[i0].nz) ++i1;
        const int rn = i1 - i0, Tz = it[i0].nz;
        const float* cb = vcb.p + (size_t)i0 * cbias_stride;
        const bool first = (i0 == 0);
        auto dump = [&](const char* name, const float* p, size_t n) {           // first batch item only
            if (first && stage && stage_out && std::strcmp(stage, name) == 0) {
                const size_t m = std::min<size_t>(n, (size_t)stage_cap);
                CUDA_CHECK(cudaMemcpyAsync(stage_out, p, m * sizeof(float), cudaMemcpyDeviceToHost, sv));
            }
        };
        InterpItem ii[kVocMaxItems];
        for (int k = 0; k < rn; ++k) ii[k] = interp_item(it[i0 + k]);
        launch_interp(ii, rn, vz.p, nullptr, 0, c.voc_in_dim, Tz, s1, resample ? s2 : 1.0, sv);
        dump("z", vz.p, (size_t)c.voc_in_dim * Tz);
        launch_conv1d(vz.p, conv_pre.wt.p, conv_pre.b.p, cb + cbias_off[0], nullptr, vpre.p, conv_pre.Cin, conv_pre.Cout, Tz,
                      conv_pre.K, 1, 1.0f, 1.0f, CONV_STORE, rn, cbias_stride, sv);
        dump("pre", vpre.p, (size_t)c.voc_init_ch * Tz);
        const float* cur = vpre.p;
        float in_scale = 1.0f;
        int len = Tz;
        float* X = vb[0].p; float* TMP = vb[1].p; float* R1 = vb[2].p; float* R2 = vb[3].p; float* ZS = vb[4].p;
        auto conv = [&](const ConvW& w, const float* x, const float* resid, float* out, int dil, int mode) {
            launch_conv1d(x, w.wt.p, w.b.p, nullptr, resid, out, w.Cin, w.Cout, len, w.K, dil, 1.0f, 0.1f, mode, rn, cbias_stride, sv);
        };
        for (int i = 0; i < c.voc_n_up; ++i) {
            const ConvW& u = *ups[i];
            launch_conv_transpose1d(cur, u.wt.p, u.b.p, cb + cbias_off[i + 1], X, nullptr, 0, 0.f, u.Cin, u.Cout, len, u.K,
                                    c.voc_up_rates[i], in_scale, 0.1f, rn, cbias_stride, sv);
            len *= c.voc_up_rates[i];
            const int C = u.Cout;
            { char nm[16]; snprintf(nm, sizeof(nm), "up%d", i); dump(nm, X, (size_t)C * len); }
            for (int j = 0; j < nk; ++j) {
                const RB& rb = *rbs[i * nk + j];
                const float* r_in = X;
                for (int t = 0; t < 3; ++t) {
                    conv(*rb.c1[t], r_in, nullptr, TMP, c.voc_rb_dilations[t], CONV_STORE);
                    if (t < 2) {
                        float* r_out = (t == 0) ? R1 : R2;
                        conv(*rb.c2[t], TMP, r_in, r_out, 1, CONV_STORE);
                        r_in = r_out;
                    } else {
                        conv(*rb.c2[t], TMP, r_in, ZS, 1, j == 0 ? CONV_STORE : CONV_ACCUM);
                    }
                }
            }
            { char nm[16]; snprintf(nm, sizeof(nm), "mrf%d", i); dump(nm, ZS, (size_t)C * len); }   // un-normalised sum
            // next stage reads the MRF sum scaled by 1/nk; its ConvT writes X (dead by now), and ZS is only
            // overwritten after that ConvT has consumed it (stream order)
            cur = ZS;
            in_scale = 1.0f / (float)nk;
        }
        launch_conv_post(cur, conv_post_w.p, wav_dev_out + (size_t)i0 * wav_stride, post_cin, len, 7, in_scale, 0.01f, rn, sv,
                         nullptr, (int)wav_stride);
        i0 = i1;
    }
}

// Tensor-core vocoder: every Conv1d operand is kept as activated fp16 atoms written by its producer's epilogue
// (ConvT / previous conv), so the conv kernels are pure bulk-copy + wgmma; fp32 is kept for the residual stream
// (x, r1, r2), the MRF sum and the final waveform.  (speaker biases were gathered into vcb by run_vocoder)
void Engine::run_vocoder_tc(const VocItem* it, int nb, int Lz, float* wav_dev_out, const char* stage, float* stage_out,
                            int64_t stage_cap) {
    const auto& c = cfg;
    cudaStream_t sv = st_voc;
    const double s1 = (double)c.code_stride / (double)c.output_hop_length;
    const double s2 = (double)c.output_sample_rate / (double)c.input_sample_rate;
    const bool resample = c.output_sample_rate != c.input_sample_rate;
    const float* cb = vcb.p;
    auto dump = [&](const char* name, const float* p, size_t n) {
        if (stage && stage_out && std::strcmp(stage, name) == 0) {
            const size_t m = std::min<size_t>(n, (size_t)stage_cap);
            CUDA_CHECK(cudaMemcpyAsync(stage_out, p, m * sizeof(float), cudaMemcpyDeviceToHost, sv));
        }
    };
    InterpItem ii[kVocMaxItems];
    int lens[kVocMaxItems];                  // per-item signal length at the current stage
    for (int k = 0; k < nb; ++k) {
        ii[k] = interp_item(it[k]);
        lens[k] = it[k].nz;
    }
    auto conv_tc = [&](const ConvW& w, const __half* a16, const float* cbias, const float* resid, float* out32, __half* out16,
                       int L, int lpad, int dil, int mode, float scale16) {
        launch_conv1d_tc(a16, w.blob.p, w.plan, w.b.p, cbias, resid, out32, out16, w.Cin, w.Cout, L, lpad, w.K, dil, 0.1f, scale16,
                         mode, nb, cbias_stride, sv, lens);
    };
    int lpad = atoms_lpad(Lz);
    __half* XA = va16[0].p; __half* TA = va16[1].p; __half* RA[2] = {va16[2].p, va16[3].p}; __half* PA = va16[4].p;
    launch_atoms_zero_pads(vz16.p, nb * c.voc_in_dim / 8, lpad, Lz, sv, nb, lens);
    launch_atoms_zero_pads(PA, nb * c.voc_init_ch / 8, lpad, Lz, sv, nb, lens);
    launch_interp(ii, nb, stage ? vz.p : nullptr, vz16.p, lpad, c.voc_in_dim, Lz, s1, resample ? s2 : 1.0, sv);
    if (stage) dump("z", vz.p, (size_t)c.voc_in_dim * Lz);
    // conv_pre: fp32 copy only for the stage tap; its activated fp16 atoms feed the first transposed conv
    conv_tc(conv_pre, vz16.p, cb + cbias_off[0], nullptr, stage ? vpre.p : nullptr, PA, Lz, lpad, 1, CONV_STORE, 1.0f);
    if (stage) dump("pre", vpre.p, (size_t)c.voc_init_ch * Lz);
    int len = Lz;
    const int nk = c.voc_n_rb;
    float* X = vb[0].p; float* R[2] = {vb[2].p, vb[3].p}; float* ZS = vb[4].p;
    for (int i = 0; i < c.voc_n_up; ++i) {
        const ConvW& u = *ups[i];
        const int C = u.Cout;
        const int up = c.voc_up_rates[i];
        const int lout = len * up;
        const int lpad_in = lpad;
        lpad = atoms_lpad(lout);
        int lens_out[kVocMaxItems];
        for (int k = 0; k < nb; ++k) lens_out[k] = lens[k] * up;
        for (__half* b : {XA, TA, RA[0], RA[1]}) launch_atoms_zero_pads(b, nb * C / 8, lpad, lout, sv, nb, lens_out);
        launch_convT_tc(PA, u.blob.p, u.plan, u.b.p, cb + cbias_off[i + 1], X, XA, u.Cin, C, len, lpad_in, lpad, up, 0.1f, nb,
                        cbias_stride, sv, lens);
        len = lout;
        for (int k = 0; k < nb; ++k) lens[k] = lens_out[k];
        { char nm[16]; snprintf(nm, sizeof(nm), "up%d", i); dump(nm, X, (size_t)C * len); }
        const bool more = (i + 1 < c.voc_n_up);
        if (more) launch_atoms_zero_pads(PA, nb * C / 8, lpad, len, sv, nb, lens);     // PA is re-shaped for the next stage's input
        for (int j = 0; j < nk; ++j) {
            const RB& rb = *rbs[i * nk + j];
            const bool emit = more && (j == nk - 1);
            const int mode = j == 0 ? CONV_STORE : CONV_ACCUM;
            if (use_resblock_tc && resblock_tc_tile_rows(C, rb.c1[0]->K, c.voc_rb_dilations, len) > 0) {
                // the whole resblock on chip: same bits as the six launches below
                const __half* wb[6]; const float* bs[6];
                for (int t = 0; t < 3; ++t) {
                    wb[2 * t] = rb.c1[t]->blob.p; wb[2 * t + 1] = rb.c2[t]->blob.p;
                    bs[2 * t] = rb.c1[t]->b.p; bs[2 * t + 1] = rb.c2[t]->b.p;
                }
                launch_resblock_tc(XA, X, wb, bs, ZS, emit ? PA : nullptr, C, len, lpad, rb.c1[0]->K, c.voc_rb_dilations, mode,
                                   1.0f / (float)nk, nb, lens, sv);
                continue;
            }
            const __half* in16 = XA;
            const float* resid = X;
            for (int t = 0; t < 3; ++t) {
                conv_tc(*rb.c1[t], in16, nullptr, nullptr, nullptr, TA, len, lpad, c.voc_rb_dilations[t], CONV_STORE, 1.0f);
                if (t < 2) {
                    conv_tc(*rb.c2[t], TA, nullptr, resid, R[t], RA[t], len, lpad, 1, CONV_STORE, 1.0f);
                    in16 = RA[t]; resid = R[t];
                } else {
                    // MRF sum; the last resblock also emits lrelu(sum / nk) as the next transposed conv's operand
                    conv_tc(*rb.c2[t], TA, nullptr, resid, ZS, emit ? PA : nullptr, len, lpad, 1, mode, 1.0f / (float)nk);
                }
            }
        }
        { char nm[16]; snprintf(nm, sizeof(nm), "mrf%d", i); dump(nm, ZS, (size_t)C * len); }
    }
    launch_conv_post(ZS, conv_post_w.p, wav_dev_out, post_cin, len, 7, 1.0f / (float)nk, 0.01f, nb, sv, lens);
}

// ================================================================================================
// scheduler
// ================================================================================================
float* Engine::pinned_get(size_t n, size_t* cap) {
    std::lock_guard<std::mutex> lk(pin_mu);
    size_t best = pinned_pool.size();                  // best fit: token-sized requests must not eat waveform-sized buffers
    for (size_t i = 0; i < pinned_pool.size(); ++i)
        if (pinned_pool[i].second >= n && (best == pinned_pool.size() || pinned_pool[i].second < pinned_pool[best].second)) best = i;
    if (best != pinned_pool.size() && pinned_pool[best].second <= 4 * n + 4096) {
        float* p = pinned_pool[best].first; *cap = pinned_pool[best].second;
        pinned_pool.erase(pinned_pool.begin() + best);
        return p;
    }
    float* p = nullptr;
    CUDA_CHECK(cudaMallocHost(&p, n * sizeof(float)));
    *cap = n;
    return p;
}
float* Engine::dev_get(size_t n, size_t* cap) {
    std::lock_guard<std::mutex> lk(pin_mu);
    size_t best = dev_pool.size();
    for (size_t i = 0; i < dev_pool.size(); ++i)
        if (dev_pool[i].second >= n && (best == dev_pool.size() || dev_pool[i].second < dev_pool[best].second)) best = i;
    if (best != dev_pool.size()) {
        float* p = dev_pool[best].first; *cap = dev_pool[best].second;
        dev_pool.erase(dev_pool.begin() + best);
        return p;
    }
    float* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, n * sizeof(float)));
    *cap = n;
    return p;
}
void Engine::dev_put(float* p, size_t cap) { std::lock_guard<std::mutex> lk(pin_mu); dev_pool.emplace_back(p, cap); }

void Engine::pinned_put(float* p, size_t cap) { std::lock_guard<std::mutex> lk(pin_mu); pinned_pool.emplace_back(p, cap); }

void Engine::submit(uint64_t id, const int32_t* text, int n_text, int speaker, const xtts_sampling& sp, float speed,
                    const xtts_beam* beam) {
    if (!(speed >= 0.25f && speed <= 4.0f)) throw std::runtime_error("speed out of range (0.25..4)");   // NaN included
    if (beam) {
        if (beam->num_beams < 1 || beam->num_beams > kMaxBeams || beam->num_beams > B)
            throw std::runtime_error("num_beams out of range (1..8, <= max_batch)");
        if (beam->num_beams > 1 && sp.early_tokens != 0) throw std::runtime_error("a beam-search chunk cannot stream (early_tokens must be 0)");
        if (beam->num_beams > 1 && !std::isfinite(beam->length_penalty)) throw std::runtime_error("length_penalty must be finite");
        if (beam->num_beams > 1 && beam->do_sample && !(sp.temperature > 0.f))
            throw std::runtime_error("beam sampling needs a temperature > 0 (transformers rejects it too)");
        if (beam->num_beams > 1 && !beam_supported(V, max_pages, CAP))
            throw std::runtime_error("beam search: this engine's geometry exceeds the beam kernels' limits");
    }
    if (n_text <= 0 || n_text > cfg.max_text_tokens + 2) throw std::runtime_error("n_text out of range (1..max_text_tokens+2)");
    if (speaker < 0 || speaker >= S) throw std::runtime_error("speaker slot out of range");
    // ids are checked here so that a bad id fails this call alone, not the batched step it would have joined
    for (int i = 0; i < n_text; ++i)
        if (text[i] < 0 || text[i] >= cfg.n_text_tokens) throw std::runtime_error("text token id out of range");
    std::shared_ptr<Sequence> s(new Sequence());
    s->id = id; s->text_ids.assign(text, text + n_text); s->speaker = speaker; s->sp = sp; s->speed = speed; s->t_submit = now_s();
    if (beam && beam->num_beams > 1) s->beam = *beam;
    require_finalized();
    if (!spk_valid[speaker]) throw std::runtime_error("speaker slot not set");
    {
        std::lock_guard<std::mutex> lk(q_mu);
        pending.push_back(s);
        ++inflight;
    }
    cv_work.notify_all();
}

// xtts_cancel: the reference aborts the vLLM request when its generator is dropped.  Handled by the scheduler thread at
// its next iteration: a queued chunk is dropped, a decoding one stops and gives its slot and KV pages back.
void Engine::cancel(uint64_t id) {
    {
        std::lock_guard<std::mutex> lk(q_mu);
        cancel_req.push_back(id);
    }
    cv_work.notify_all();
}

void Engine::free_seq_buffers(Sequence& s) {
    if (s.tok_host) { cudaFreeHost(s.tok_host); s.tok_host = nullptr; }
    if (s.wav_host) { cudaFreeHost(s.wav_host); s.wav_host = nullptr; }
    if (s.wav_dev) { cudaFree(s.wav_dev); s.wav_dev = nullptr; }
    if (s.lat_dev) { cudaFree(s.lat_dev); s.lat_dev = nullptr; }
}

void Engine::recycle_seq_buffers(Sequence& s) {
    if (s.tok_host) { pinned_put(reinterpret_cast<float*>(s.tok_host), s.tok_cap); s.tok_host = nullptr; }
    if (s.wav_host) { pinned_put(s.wav_host, s.wav_cap); s.wav_host = nullptr; }
    if (s.wav_dev) { dev_put(s.wav_dev, s.wav_dev_cap); s.wav_dev = nullptr; }
    if (s.lat_dev) { dev_put(s.lat_dev, s.lat_dev_cap); s.lat_dev = nullptr; }
}

// hands a piece to the completion queue (xtts_poll / xtts_fetch)
void Engine::deliver(std::shared_ptr<Piece> p, bool ends_sequence) {
    {
        std::lock_guard<std::mutex> lk(q_mu);
        done_q.push_back(p);
        done_map[p->s->id].push_back(p);
        if (ends_sequence) --inflight;
    }
    cv_done.notify_all();
}

// a chunk that never reached a slot (queued, or its admission failed) ends with `code`
void Engine::fail_unadmitted(std::shared_ptr<Sequence> s, int code, const char* what) {
    if (code != XTTS_ERR_CANCELLED) set_error(what);
    release_slot(*s);
    std::shared_ptr<Piece> p(new Piece());
    p->s = s; p->status = code; p->final = true; p->t_done = s->t_done = now_s();
    deliver(p, true);
}

// The decode of `s` is over (stop token / max_tokens: fail_status 0; cancelled or failed: < 0).  Its KV pages go back now;
// the slot — whose latent ring and token row the remaining vocoder work reads — when the final job has completed.
void Engine::on_finished(std::shared_ptr<Sequence> s, int n_tokens, int fail_status) {
    release_pages(*s);
    // a beam group: the hypothesis is in the primary slot now (beam_gather_kernel); the other slots go back
    for (size_t b = 1; b < s->beam_slots.size(); ++b) free_slots.push_back(s->beam_slots[b]);
    if (s->beam_slots.size() > 1) s->beam_slots.resize(1);
    s->n_tokens = std::max(0, std::min(n_tokens, CAP));
    st_tokens += s->n_tokens;
    VocJob j;
    j.s = s; j.final = true; j.fail_status = fail_status; j.T_clamp = std::max(1, s->n_tokens); j.tok_upto = s->n_tokens;
    if (fail_status == 0 && s->sp.vocode && s->n_tokens > 0) {
        const int Tz = z_frames(s->n_tokens, s->speed);
        j.zk0 = std::min(s->voc_z_done, Tz); j.zk1 = Tz;
        j.zw0 = std::max(0, j.zk0 - voc_hz); j.zw1 = Tz;
        if (j.zk0 < Tz) {
            // a slow speaking rate can stretch the rest of the chunk past one window: internal windows, then the final one
            const std::vector<VocSpan> w = split_windows(j.zk0, Tz);
            for (size_t i = 0; i + 1 < w.size(); ++i) {
                VocJob k;
                k.s = s; k.T_clamp = j.T_clamp; k.internal = true;
                k.zw0 = w[i].zw0; k.zw1 = w[i].zw1; k.zk0 = w[i].zk0; k.zk1 = w[i].zk1;
                voc_pending.push_back(std::move(k));
            }
            j.zw0 = w.back().zw0; j.zw1 = w.back().zw1; j.zk0 = w.back().zk0; j.zk1 = w.back().zk1;
        }
    }
    s->next_boundary = 0;
    voc_pending.push_back(std::move(j));
}

// A chunk that is still decoding: once the frames behind its next cut (plus the vocoder's receptive field) exist, the
// window up to the cut goes to the vocoder — audio is produced while the GPT is still busy with the rest of the chunk.
void Engine::maybe_cut_window(std::shared_ptr<Sequence>& s) {
    while (s->next_boundary > 0 && s->next_boundary < s->max_tok) {
        const int b = s->next_boundary;
        const int n_avail = s->steps + 1;                   // latent frames in the ring
        // a window has to use the speed stage exactly when the finished chunk will: not before it applies to n_avail
        if (s->speed != 1.f && !speed_stage(n_avail, s->speed)) return;
        const int zk1 = z_frames(b, s->speed), zw1 = zk1 + voc_hz;
        if (z_avail(n_avail, s->speed) < zw1) return;
        const int zk0 = s->voc_z_done;
        const int zw0 = std::max(0, zk0 - voc_hz);
        if (zw1 - zw0 > voc_max_Tz) { s->next_boundary = 0; return; }
        if (zk1 > zk0) {
            VocJob j;
            j.s = s; j.T_clamp = n_avail; j.zw0 = zw0; j.zw1 = zw1; j.zk0 = zk0; j.zk1 = zk1; j.tok_upto = b;
            voc_pending.push_back(std::move(j));
            s->voc_z_done = zk1;
        }
        s->next_boundary = s->seg_next > 0 ? b + s->seg_next : 0;
    }
}

// one vocoder launch sequence for `jobs` on st_voc: windows -> waveforms -> the kept samples into each chunk's own buffer,
// token ids (and, for final jobs, the latent snapshot) next to them; completion is observed through b.ev1
void Engine::dispatch_batch(std::vector<VocJob>& jobs, bool decode_active) {
    VocBatch b;
    CUDA_CHECK(cudaEventCreate(&b.ev0)); CUDA_CHECK(cudaEventCreate(&b.ev1));
    cudaStream_t sv = st_voc;
    try {
        CUDA_CHECK(cudaEventRecord(b.ev0, sv));
        std::vector<VocItem> items;
        std::vector<int> job_of;
        for (size_t k = 0; k < jobs.size(); ++k) {
            VocJob& j = jobs[k];
            Sequence& s = *j.s;
            if (!s.tok_host) s.tok_host = reinterpret_cast<int32_t*>(pinned_get((size_t)std::max(1, s.max_tok), &s.tok_cap));
            if (j.zk1 > j.zk0) {
                const size_t need = (size_t)std::max(1, samples_for(s.max_tok, s.speed));
                if (d2h_wav) { if (!s.wav_host) s.wav_host = pinned_get(need, &s.wav_cap); }
                else if (!s.wav_dev) s.wav_dev = dev_get(need, &s.wav_dev_cap);
                items.push_back(VocItem{d_latents.p + (size_t)s.slot * CAP * H, j.T_clamp, j.zw0, j.zw1 - j.zw0, s.speaker, s.speed});
                job_of.push_back((int)k);
            }
        }
        int Lz = 0;
        for (auto& it : items) Lz = std::max(Lz, it.nz);
        if (!items.empty()) {
            g_voc_sm_cap = (decode_active && voc_sms > 0) ? voc_sms : 0;
            run_vocoder(items.data(), (int)items.size(), vwav.p, nullptr, nullptr, 0);
            g_voc_sm_cap = 0;
        }
        const size_t wstride = (size_t)Lz * voc_hop;
        for (size_t i = 0; i < items.size(); ++i) {
            VocJob& j = jobs[job_of[i]];
            Sequence& s = *j.s;
            const size_t n = (size_t)(j.zk1 - j.zk0) * voc_hop, dst_off = (size_t)j.zk0 * voc_hop;
            const float* src = vwav.p + i * wstride + (size_t)(j.zk0 - j.zw0) * voc_hop;
            if (d2h_wav) CUDA_CHECK(cudaMemcpyAsync(s.wav_host + dst_off, src, n * sizeof(float), cudaMemcpyDeviceToHost, sv));
            else CUDA_CHECK(cudaMemcpyAsync(s.wav_dev + dst_off, src, n * sizeof(float), cudaMemcpyDeviceToDevice, sv));
            st_samples += n;
        }
        for (auto& j : jobs) {
            Sequence& s = *j.s;
            if (j.tok_upto > 0 && s.slot >= 0)
                CUDA_CHECK(cudaMemcpyAsync(s.tok_host, d_tokens.p + (size_t)s.slot * CAP, (size_t)j.tok_upto * sizeof(int32_t),
                                           cudaMemcpyDeviceToHost, sv));
            if (j.final && j.fail_status == 0 && s.n_tokens > 0 && s.slot >= 0) {
                s.lat_dev = dev_get((size_t)s.n_tokens * H, &s.lat_dev_cap);
                CUDA_CHECK(cudaMemcpyAsync(s.lat_dev, d_latents.p + (size_t)s.slot * CAP * H, (size_t)s.n_tokens * H * sizeof(float),
                                           cudaMemcpyDeviceToDevice, sv));
            }
        }
        CUDA_CHECK(cudaEventRecord(b.ev1, sv));
    } catch (...) {
        cudaEventDestroy(b.ev0); cudaEventDestroy(b.ev1);
        throw;
    }
    b.jobs = std::move(jobs);
    voc_inflight.push_back(std::move(b));
}

// Forms batches from the queued windows (oldest first): as many as the workspace holds, at most voc_max_items.  A full
// batch always goes; a partial one only while fewer than two batches are in flight, so that windows arriving while the
// vocoder is busy collect into larger launches instead of going out one by one.
void Engine::dispatch_ready(bool decode_active) {
    while (!voc_pending.empty()) {
        if (voc_inflight.size() >= 2 && (int)voc_pending.size() < voc_max_items) break;
        std::vector<VocJob> jobs;
        int nb = 0, Lz = 0;
        while (!voc_pending.empty()) {
            VocJob& j = voc_pending.front();
            const int w = j.zk1 > j.zk0 ? j.zw1 - j.zw0 : 0;
            if (w > 0) {
                if (nb + 1 > voc_max_items || !voc_fits(nb + 1, std::max(Lz, w))) break;
                ++nb; Lz = std::max(Lz, w);
            }
            jobs.push_back(std::move(j));
            voc_pending.pop_front();
        }
        if (jobs.empty()) throw std::runtime_error("vocoder: a window does not fit the workspace");
        // longest first: equal lengths end up adjacent (the fp32 path batches runs of equal length)
        std::stable_sort(jobs.begin(), jobs.end(), [](const VocJob& a, const VocJob& b) { return a.zw1 - a.zw0 > b.zw1 - b.zw0; });
        std::vector<VocJob> keep = jobs;                    // (dispatch_batch consumes `jobs`)
        try { dispatch_batch(jobs, decode_active); }
        catch (const std::exception& ex) {
            // the batch never reached the stream: its chunks fail, their slots are released
            set_error(ex.what());
            for (auto& j : keep) {
                if (!j.final) { j.s->next_boundary = 0; continue; }      // the final job of that chunk will follow and deliver
                std::shared_ptr<Piece> p(new Piece());
                p->s = j.s; p->status = XTTS_ERR_CUDA; p->final = true; p->t_done = j.s->t_done = now_s();
                release_slot(*j.s);
                deliver(p, true);
            }
        }
    }
}

void Engine::complete_batch(VocBatch& b) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, b.ev0, b.ev1) == cudaSuccess) st_voc_ms += ms;
    const double t = now_s();
    // dispatch_ready sorted the batch longest first: a chunk with several windows here gets them back in the order they
    // were cut (ascending z), its final result last; chunks keep their batch order
    const size_t n = b.jobs.size();
    std::vector<size_t> first(n), ord(n);
    for (size_t i = 0; i < n; ++i) {
        first[i] = i;
        for (size_t k = 0; k < i; ++k)
            if (b.jobs[k].s == b.jobs[i].s) { first[i] = first[k]; break; }
        ord[i] = i;
    }
    std::stable_sort(ord.begin(), ord.end(), [&](size_t x, size_t y) {
        const VocJob &a = b.jobs[x], &c = b.jobs[y];
        return std::make_tuple(first[x], a.final, a.zk0) < std::make_tuple(first[y], c.final, c.zk0);
    });
    for (size_t oi : ord) {
        VocJob& j = b.jobs[oi];
        Sequence& s = *j.s;
        const int samp_end = j.zk1 > j.zk0 ? j.zk1 * voc_hop : s.samp_delivered;
        if (!j.final) {
            if (!s.stream_pieces || j.internal) continue;   // accumulated silently: everything goes out with the final result
            std::shared_ptr<Piece> p(new Piece());
            p->s = j.s; p->status = 1; p->tok0 = s.tok_delivered; p->tok1 = j.tok_upto;
            p->samp0 = s.samp_delivered; p->nsamp = samp_end - s.samp_delivered; p->t_done = t;
            s.tok_delivered = j.tok_upto; s.samp_delivered = samp_end;
            deliver(p, false);
            continue;
        }
        std::shared_ptr<Piece> p(new Piece());
        p->s = j.s; p->final = true; p->status = j.fail_status; p->t_done = s.t_done = t;
        if (j.fail_status == 0) {
            const int total = s.sp.vocode ? samples_for(s.n_tokens, s.speed) : 0;
            p->tok0 = 0; p->tok1 = s.n_tokens;              // the final result lists every token; samples: what is left
            p->samp0 = s.samp_delivered; p->nsamp = std::max(0, total - s.samp_delivered);
        }
        release_slot(s);
        deliver(p, true);
    }
    cudaEventDestroy(b.ev0); cudaEventDestroy(b.ev1);
    b.ev0 = b.ev1 = nullptr;
}

// completed vocoder batches -> completion queue.  block: wait for the oldest batch (nothing else to do meanwhile)
void Engine::reap(bool block) {
    while (!voc_inflight.empty()) {
        VocBatch& b = voc_inflight.front();
        cudaError_t e = block ? cudaEventSynchronize(b.ev1) : cudaEventQuery(b.ev1);
        if (e == cudaErrorNotReady) { (void)cudaGetLastError(); return; }
        if (e != cudaSuccess) {
            // a failed batch fails its chunks (and, the context being what it is after a device fault, everything after it)
            set_error(std::string("vocoder batch failed: ") + cudaGetErrorString(e));
            for (auto& j : b.jobs) if (j.final && j.fail_status == 0) j.fail_status = XTTS_ERR_CUDA;
        }
        complete_batch(b);
        voc_inflight.pop_front();
        block = false;
    }
}

void Engine::process_cancels(const std::vector<uint64_t>& ids) {
    for (uint64_t id : ids) {
        bool found = false;
        for (auto it = waiting.begin(); it != waiting.end(); ++it)
            if ((*it)->id == id) {
                auto s = *it; waiting.erase(it);
                fail_unadmitted(s, XTTS_ERR_CANCELLED, "cancelled");
                found = true; break;
            }
        if (found) continue;
        for (auto it = running.begin(); it != running.end(); ++it)
            if ((*it)->id == id) {
                auto s = *it; running.erase(it);
                s->cancelled = true;
                on_finished(s, 0, XTTS_ERR_CANCELLED);      // queued behind its in-flight windows: the slot is freed after them
                break;
            }
        // (an id that is already finishing or finished: nothing to do, its result is on its way)
    }
}

void Engine::loop() {
    t_kctx = &kctx_;                                   // this thread issues this engine's work, and only this engine's
    cudaSetDevice(cfg.device);
    while (true) {
        for (int spin = 0; api_waiting.load() > 0 && spin < 20000; ++spin) std::this_thread::yield();   // API calls go first
        std::vector<uint64_t> cancels;
        {
            std::unique_lock<std::mutex> q(q_mu);
            cv_work.wait(q, [&] {
                return stop.load() || !pending.empty() || !cancel_req.empty() || (!waiting.empty() && !hold_admission.load()) ||
                       !running.empty() || !voc_pending.empty() || !voc_inflight.empty();
            });
            if (stop.load()) break;
            while (!pending.empty()) {
                // stable priority insert: lower `priority` (chunk index) first, FIFO among equals
                auto s = pending.front(); pending.pop_front();
                auto it = waiting.end();
                while (it != waiting.begin() && (*(it - 1))->sp.priority > s->sp.priority) --it;
                waiting.insert(it, s);
            }
            cancels.swap(cancel_req);
        }
        std::lock_guard<std::mutex> lk(mu);
        std::vector<std::shared_ptr<Sequence>> fresh_sp;      // admitted this iteration (outside the try: see the catch)
        bool gpt_work = false;
        try {
            process_cancels(cancels);
            // ---- admission (continuous batching): fill free slots, whole prompts, within the row budget
            std::vector<Sequence*> fresh;
            int rows = 0;
            while (!hold_admission.load() && !waiting.empty() && !free_slots.empty()) {
                auto s = waiting.front();
                const int p = cfg.n_cond_latents + (int)s->text_ids.size() + 1;
                if (!fresh.empty() && rows + p > prefill_rows_cap) break;
                // a beam group takes its num_beams slots at once (only beam 0's prompt is prefilled); one that does not
                // fit stops the wave, as the row budget does
                if ((int)free_slots.size() < s->beam.num_beams) break;
                waiting.pop_front();                          // (KV pages cannot run out: the pool holds max_pages per slot)
                if (!spk_valid[s->speaker]) { fail_unadmitted(s, XTTS_ERR_STATE, "speaker slot not set"); continue; }
                s->slot = free_slots.back(); free_slots.pop_back();
                if (s->beam.num_beams > 1) {
                    s->beam_slots.assign(1, s->slot);
                    for (int b = 1; b < s->beam.num_beams; ++b) { s->beam_slots.push_back(free_slots.back()); free_slots.pop_back(); }
                }
                rows += p;
                fresh.push_back(s.get()); fresh_sp.push_back(s);
            }
            const double t0 = now_s();
            if (!fresh.empty()) {
                gpt_work = true;
                init_slots(fresh, nullptr, 0);
                for (auto& s : fresh_sp) {
                    // vocoder windows: the first cut after early_tokens (streaming chunks) or voc_segment tokens, then every
                    // voc_segment; 0 = the chunk is vocoded whole when it ends
                    // (a beam chunk's hypothesis is known only when its group ends: no windows, no pieces)
                    const bool beams = s->beam.num_beams > 1;
                    s->stream_pieces = s->sp.early_tokens > 0 && s->sp.vocode && !beams;
                    s->seg_next = s->sp.vocode && !beams ? voc_segment : 0;
                    s->next_boundary = s->stream_pieces ? s->sp.early_tokens : s->seg_next;
                }
                prefill(fresh);
                std::vector<Sequence*> groups;
                std::vector<int> rows0;
                for (size_t i = 0; i < fresh.size(); ++i)
                    if (fresh[i]->beam.num_beams > 1) { groups.push_back(fresh[i]); rows0.push_back((int)i); }
                beam_step(groups, rows0, true);
                for (auto& s : fresh_sp) running.push_back(s);
                fresh_sp.clear();
                // a sequence may already be finished after its first token (max_tokens == 1 / instant stop)
                d_finished.download(h_finished, NSLOT, st);
                d_n_gen.download(h_finished + NSLOT, NSLOT, st);
                CUDA_CHECK(cudaStreamSynchronize(st));
            }
            if (!running.empty()) {
                std::vector<int> active;
                std::vector<Sequence*> groups;
                std::vector<int> rows0;
                double ctx_sum = 0;
                for (auto& s : running) {
                    if (h_finished[s->slot]) continue;
                    if (s->beam.num_beams > 1) { groups.push_back(s.get()); rows0.push_back((int)active.size()); }
                    const int nb = std::max(1, (int)s->beam_slots.size());
                    for (int b = 0; b < nb; ++b) { active.push_back(nb == 1 ? s->slot : s->beam_slots[b]); ctx_sum += s->n_prompt + s->steps + 1; }
                    ++s->steps;
                }
                if (!active.empty()) {
                    gpt_work = true;
                    decode_ctx_sum = ctx_sum;
                    decode_step(active);
                    beam_step(groups, rows0, false);     // eager on st, ahead of the read-back: no extra host sync
                    d_finished.download(h_finished, NSLOT, st);
                    d_n_gen.download(h_finished + NSLOT, NSLOT, st);
                    CUDA_CHECK(cudaStreamSynchronize(st));
                    if (last_prof) { g_prof.collect_graph(*last_prof, decode_ctx_sum); last_prof = nullptr; }
                }
            }
            if (gpt_work) st_gpt_ms += (now_s() - t0) * 1e3;
            // ---- vocoder work: final windows of the chunks that just ended, cuts of the ones still decoding
            std::vector<std::shared_ptr<Sequence>> keep;
            for (auto& s : running) {
                if (h_finished[s->slot]) on_finished(s, h_finished[NSLOT + s->slot], 0);
                else { maybe_cut_window(s); keep.push_back(s); }
            }
            running.swap(keep);
        } catch (const std::exception& ex) {
            // a failure inside a batched step fails every sequence that was part of it — including the ones admitted
            // in this iteration whose prefill threw before they reached `running`
            set_error(ex.what());
            for (auto& s : fresh_sp) { release_pages(*s); on_finished(s, 0, XTTS_ERR_CUDA); }
            for (auto& s : running) on_finished(s, 0, XTTS_ERR_CUDA);
            running.clear();
        }
        try {
            dispatch_ready(!running.empty());
            // nothing for the GPT to do: wait for the oldest vocoder batch instead of spinning
            reap(!gpt_work && running.empty() && !voc_inflight.empty());
        } catch (const std::exception& ex) { set_error(ex.what()); }
    }
}

int Engine::poll(xtts_result* out, int timeout_ms) {
    std::unique_lock<std::mutex> lk(q_mu);
    if (!cv_done.wait_for(lk, std::chrono::milliseconds(std::max(0, timeout_ms)), [&] { return !done_q.empty(); })) return 0;
    auto p = done_q.front(); done_q.pop_front();
    const Sequence& s = *p->s;
    out->seq_id = s.id; out->status = p->status; out->n_tokens = p->tok1 - p->tok0; out->n_samples = p->nsamp;
    out->n_prompt_rows = s.n_prompt; out->t_submit = s.t_submit; out->t_first_token = s.t_first; out->t_done = p->t_done;
    return 1;
}

// hands out the OLDEST unfetched piece of `id` (partial pieces before the final result)
void Engine::fetch(uint64_t id, int32_t* tokens, float* wav, float* latents) {
    std::shared_ptr<Piece> p;
    {
        std::lock_guard<std::mutex> lk(q_mu);
        auto it = done_map.find(id);
        if (it == done_map.end() || it->second.empty()) throw std::runtime_error("fetch: unknown or unfinished sequence id");
        p = it->second.front();
        it->second.pop_front();
        if (it->second.empty()) done_map.erase(it);
        for (auto q = done_q.begin(); q != done_q.end(); ++q) if (*q == p) { done_q.erase(q); break; }
    }
    Sequence& s = *p->s;
    const int nt = p->tok1 - p->tok0;
    if (tokens && nt > 0 && s.tok_host) std::memcpy(tokens, s.tok_host + p->tok0, (size_t)nt * sizeof(int32_t));
    if (wav && p->nsamp > 0 && s.wav_host) std::memcpy(wav, s.wav_host + p->samp0, (size_t)p->nsamp * sizeof(float));
    const bool dev_wav = wav && p->nsamp > 0 && !s.wav_host && s.wav_dev;
    const bool dev_lat = latents && p->final && s.lat_dev && s.n_tokens > 0;
    if (dev_wav || dev_lat) {
        // device copies on a stream of their own: no need to wait behind the scheduler's iteration
        CUDA_CHECK(cudaSetDevice(cfg.device));
        cudaStream_t sc = nullptr;
        CUDA_CHECK(cudaStreamCreateWithFlags(&sc, cudaStreamNonBlocking));
        cudaError_t e = cudaSuccess;
        if (dev_wav) e = cudaMemcpyAsync(wav, s.wav_dev + p->samp0, (size_t)p->nsamp * sizeof(float), cudaMemcpyDeviceToHost, sc);
        if (e == cudaSuccess && dev_lat) e = cudaMemcpyAsync(latents, s.lat_dev, (size_t)s.n_tokens * H * sizeof(float), cudaMemcpyDeviceToHost, sc);
        if (e == cudaSuccess) e = cudaStreamSynchronize(sc);
        cudaStreamDestroy(sc);
        CUDA_CHECK(e);
    }
    if (p->final) recycle_seq_buffers(s);
}

void Engine::set_option(const std::string& k, int64_t v) {
    if (k == "hold_admission") {       // no GPU state involved: must not wait for a running step
        hold_admission.store(v != 0);
        { std::lock_guard<std::mutex> q(q_mu); }
        cv_work.notify_all();
        return;
    }
    ApiLock lk(this);
    if (k == "d2h_wav") d2h_wav = v != 0;
    else if (k == "tc_vocoder") use_tc_vocoder = v != 0;
    else if (k == "attn_ctas_per_sm" || k == "gemm_bn") {
        if (k == "gemm_bn") { if (v != 0 && v != 32 && v != 64 && v != 128) throw std::runtime_error("gemm_bn: 0, 32, 64 or 128"); g_gemm_decode_bn = (int)v; }
        else g_attn_ctas_per_sm = (int)v;                        // < 0: absolute grid size (tests)
        drop_graphs();
    }
    else if (k == "voc_segment") voc_segment = (int)std::max<int64_t>(0, v);
    else if (k == "voc_sms") voc_sms = (int)std::max<int64_t>(0, v);
    else if (k == "tc_epilogue") g_conv_tc_epilogue = v ? 1 : 0;
    else if (k == "tc_resblock") use_resblock_tc = v != 0;
    else if (k == "pvoc_block_frames") {
        if (v < 1 || v > (1 << 20)) throw std::runtime_error("pvoc_block_frames: 1 .. 2^20 output frames");
        pvoc_block_frames = (int)v;
    }
    else if (k == "resample_block_samples") {
        if (v < 1 || v > (1 << 26)) throw std::runtime_error("resample_block_samples: 1 .. 2^26 output samples");
        resample_block_samples = (int)v;
    }
    else if (k == "flac_batch_frames") {
        if (v < 1 || v > (1 << 20)) throw std::runtime_error("flac_batch_frames: 1 .. 2^20 frames");
        flac_batch_frames = (int)v;
    }
    else if (k == "voc_batch") voc_max_items = (int)std::max<int64_t>(1, std::min<int64_t>(v, kVocMaxItems));
    else if (k == "gemm_wide") {                                  // 0 off, else the wide kernel's ring depth
        if (v != 0 && (v < 2 || v > 4)) throw std::runtime_error("gemm_wide: 0 (off) or a ring depth of 2, 3 or 4");
        g_gemm_wide = (int)v;
    }
    else if (k == "kv_fp8") {
        if (v != 0 && v != 1) throw std::runtime_error("kv_fp8: 0 (16-bit cache) or 1 (fp8 e4m3 cache)");
        if (!bf16) throw std::runtime_error("kv_fp8: the fp8 KV cache needs precision bf16 or fp16");
        if ((v != 0) == kv_fp8) return;
        bool queued;
        { std::lock_guard<std::mutex> q(q_mu); queued = !pending.empty(); }
        if (queued || !running.empty() || !waiting.empty() || !voc_pending.empty() || !voc_inflight.empty() ||
            (int)free_pages.size() != NSLOT * max_pages)
            throw StateError("kv_fp8: the KV format can only change on an idle engine");
        CUDA_CHECK(cudaSetDevice(cfg.device));
        CUDA_CHECK(cudaStreamSynchronize(st));
        drop_graphs();                                  // captured decode steps hold the old pools and kernels
        kv_fp8 = v != 0;
        alloc_kv();
    }
    else if (k == "cuda_graphs") use_graphs = v != 0;
    else if (k == "pdl") { use_pdl = v != 0; drop_graphs(); }
    else if (k == "splitk") { use_splitk = v != 0; drop_graphs(); }
    else if (k == "decode_chain") {                               // still accepted so that callers passing 0 keep working
        if (v != 0) throw std::runtime_error("decode_chain: the fused decode chain kernel was removed; only 0 is accepted");
    }
    else if (k == "microbatches" || k == "microbatch_min_rows") {
        if (k == "microbatches") n_micro = std::max<int>(1, std::min<int64_t>(v, kMaxMicro)); else micro_min_rows = (int)std::max<int64_t>(2, v);
        drop_graphs();
    }
    else if (k == "profile") {
        CUDA_CHECK(cudaSetDevice(cfg.device)); CUDA_CHECK(cudaStreamSynchronize(st)); CUDA_CHECK(cudaStreamSynchronize(st_voc));
        g_prof.reset(); g_prof.enabled = v != 0;
    }
    else if (k == "reset_stats") {
        st_decode_steps = st_prefill_rows = st_tokens = st_samples = 0; st_gpt_ms = st_voc_ms = st_cond_ms = 0;
        launch_base = g_launch_count;
    } else throw std::runtime_error("unknown option: " + k);
}

void Engine::get_stats(xtts_stats* s) {
    ApiLock lk(this);
    s->kernel_launches = g_launch_count - launch_base; s->decode_steps = st_decode_steps; s->prefill_rows = st_prefill_rows;
    s->tokens_generated = st_tokens; s->samples_generated = st_samples; s->gpt_ms = st_gpt_ms; s->vocoder_ms = st_voc_ms;
    s->cond_ms = st_cond_ms; s->hbm_bytes_weights = weight_bytes;
}

void Engine::kernel_profile(xtts_kernel_profile* out) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    CUDA_CHECK(cudaStreamSynchronize(st));
    CUDA_CHECK(cudaStreamSynchronize(st_voc));
    g_prof.collect();
    std::memset(out, 0, sizeof(*out));
    out->n = KF_COUNT;
    for (int i = 0; i < KF_COUNT && i < 16; ++i) {
        std::snprintf(out->name[i], sizeof(out->name[i]), "%s", kernel_family_name(i));
        out->ms[i] = g_prof.ms[i]; out->flops[i] = g_prof.flops[i]; out->bytes[i] = g_prof.bytes[i];
        out->launches[i] = g_prof.launches[i];
    }
}

// Stopwatch on the engine stream.  The decode branches fork from and join back into `st` inside a step; the vocoder stream
// is joined into `st` explicitly before the stop event, so that event completes after all device work submitted so far.
void Engine::device_timer(int op, double* ms) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    if (!ev_t0) { CUDA_CHECK(cudaEventCreate(&ev_t0)); CUDA_CHECK(cudaEventCreate(&ev_t1)); }
    if (op == 0) {
        CUDA_CHECK(cudaEventRecord(ev_t0, st));
        timer_armed = true;
    } else if (op == 1) {
        if (!timer_armed) throw std::runtime_error("device_timer: stop without start");
        CUDA_CHECK(cudaEventRecord(ev_vjoin, st_voc));             // the vocoder runs on its own stream: join it
        CUDA_CHECK(cudaStreamWaitEvent(st, ev_vjoin, 0));
        CUDA_CHECK(cudaEventRecord(ev_t1, st));
        CUDA_CHECK(cudaEventSynchronize(ev_t1));
        float t = 0.f;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev_t0, ev_t1));
        if (ms) *ms = (double)t;
    } else throw std::runtime_error("device_timer: op must be 0 (start) or 1 (stop)");
}

// debug timeline: op 1 arms the trace points of the decode / vocoder kernels (common.cuh), op 0 disarms and copies the
// records out: [n][2] u64 = (globaltimer ns, id << 32 | grid << 40 | last-CTA flag << 8 | phase).  Returns the record count.
int Engine::trace(int op, uint64_t* out, int cap) {
    ApiLock lk(this);
    CUDA_CHECK(cudaSetDevice(cfg.device));
    CUDA_CHECK(cudaStreamSynchronize(st)); CUDA_CHECK(cudaStreamSynchronize(st_voc));
    if (op == 1) {
        const unsigned n = 1u << 20;
        if (!d_trace.p) { d_trace.alloc((size_t)2 * n); d_trace_n.alloc(1); }
        d_trace_n.zero(st);
        CUDA_CHECK(cudaStreamSynchronize(st));
        TraceBuf tb{d_trace.p, d_trace_n.p, n};
        trace_set_gemm(tb); trace_set_gpt(tb); trace_set_conv(tb);
        CUDA_CHECK(cudaDeviceSynchronize());
        return 0;
    }
    TraceBuf off{nullptr, nullptr, 0};
    trace_set_gemm(off); trace_set_gpt(off); trace_set_conv(off);
    CUDA_CHECK(cudaDeviceSynchronize());
    if (!d_trace.p) return 0;
    unsigned n = 0;
    d_trace_n.download(&n, 1, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    n = std::min<unsigned>(n, 1u << 20);
    const int m = std::min<int>((int)n, cap);
    if (out && m > 0) { d_trace.download(reinterpret_cast<unsigned long long*>(out), (size_t)2 * m, st); CUDA_CHECK(cudaStreamSynchronize(st)); }
    return m;
}

void Engine::sync_idle() {
    std::unique_lock<std::mutex> lk(q_mu);
    cv_done.wait(lk, [&] { return inflight == 0; });
}

// ================================================================================================
// synchronous single-stage entry points
// ================================================================================================
void Engine::vocode_sync(const float* latents, int T, int speaker, float* wav, int* n_out, const char* stage,
                         float* stage_out, int64_t stage_cap) {
    ApiLock lk(this);
    require_finalized();
    CUDA_CHECK(cudaSetDevice(cfg.device));
    if (T <= 0 || T > voc_max_T) throw std::runtime_error("vocoder: latent count out of range");
    DBuf<float> lat; lat.alloc((size_t)T * cfg.voc_in_dim);
    lat.upload(latents, (size_t)T * cfg.voc_in_dim, st_voc);
    const int Tz = z_frames(T), ns = Tz * voc_hop;
    VocItem it{lat.p, T, 0, Tz, speaker};
    run_vocoder(&it, 1, vwav.p, stage, stage_out, stage_cap);
    if (wav) vwav.download(wav, ns, st_voc);
    CUDA_CHECK(cudaStreamSynchronize(st_voc));
    if (n_out) *n_out = ns;
}

// z-frames [z0, z0 + nz) of the chunk `latents` [T] as a window of its own (what the scheduler does while a chunk decodes):
// wav [nz * hop].  Samples further than the vocoder's receptive field from an inner window edge equal the whole chunk's.
void Engine::vocode_window_sync(const float* latents, int T, int speaker, int z0, int nz, float* wav) {
    ApiLock lk(this);
    require_finalized();
    CUDA_CHECK(cudaSetDevice(cfg.device));
    if (T <= 0 || T > voc_max_T) throw std::runtime_error("vocoder: latent count out of range");
    if (z0 < 0 || nz <= 0 || z0 + nz > z_frames(T)) throw std::runtime_error("vocoder: window outside the chunk");
    DBuf<float> lat; lat.alloc((size_t)T * cfg.voc_in_dim);
    lat.upload(latents, (size_t)T * cfg.voc_in_dim, st_voc);
    VocItem it{lat.p, T, z0, nz, speaker};
    run_vocoder(&it, 1, vwav.p, nullptr, nullptr, 0);
    if (wav) vwav.download(wav, (size_t)nz * voc_hop, st_voc);
    CUDA_CHECK(cudaStreamSynchronize(st_voc));
}

// The vocoder at a speaking rate: z-frames [z0, z0 + nz) as one window (nz >= 0), or the whole chunk (nz < 0) — in the
// windows the scheduler would cut for it (split_windows) when it is longer than one, their kept samples stitched.
void Engine::vocode_speed_sync(const float* latents, int T, int speaker, float speed, int z0, int nz, float* wav, int* n_out) {
    ApiLock lk(this);
    require_finalized();
    CUDA_CHECK(cudaSetDevice(cfg.device));
    if (!(speed >= 0.25f && speed <= 4.0f)) throw std::runtime_error("speed out of range (0.25..4)");
    if (T <= 0 || T > voc_max_T) throw std::runtime_error("vocoder: latent count out of range");
    if (speaker < 0 || speaker >= S || !spk_valid[speaker]) throw std::runtime_error("vocoder: speaker slot not set");
    const int Tz = z_frames(T, speed);
    std::vector<VocSpan> spans;
    if (nz >= 0) {
        if (z0 < 0 || nz == 0 || z0 + nz > Tz) throw std::runtime_error("vocoder: window outside the chunk");
        spans.push_back(VocSpan{z0, z0 + nz, z0, z0 + nz});
    } else if (Tz > 0) {
        spans = split_windows(0, Tz);
    }
    const int zbase = nz >= 0 ? z0 : 0;
    if (!spans.empty()) {
        DBuf<float> lat; lat.alloc((size_t)T * cfg.voc_in_dim);
        lat.upload(latents, (size_t)T * cfg.voc_in_dim, st_voc);
        for (const VocSpan& w : spans) {
            VocItem it{lat.p, T, w.zw0, w.zw1 - w.zw0, speaker, speed};
            run_vocoder(&it, 1, vwav.p, nullptr, nullptr, 0);
            if (wav)
                CUDA_CHECK(cudaMemcpyAsync(wav + (size_t)(w.zk0 - zbase) * voc_hop, vwav.p + (size_t)(w.zk0 - w.zw0) * voc_hop,
                                           (size_t)(w.zk1 - w.zk0) * voc_hop * sizeof(float), cudaMemcpyDeviceToHost, st_voc));
        }
        CUDA_CHECK(cudaStreamSynchronize(st_voc));
    }
    if (n_out) *n_out = (nz >= 0 ? nz : Tz) * voc_hop;
}

void Engine::gpt_prefill_sync(const int32_t* text, int n_text, int speaker, const int32_t* audio, int n_audio,
                              float* hidden_out, float* logits_out, float* latents_out) {
    ApiLock lk(this);
    require_finalized();
    require_idle();
    CUDA_CHECK(cudaSetDevice(cfg.device));
    Sequence s; s.text_ids.assign(text, text + n_text); s.speaker = speaker; s.slot = B;
    s.sp.max_tokens = CAP; s.sp.stop_token = cfg.stop_audio_token; s.sp.repetition_penalty = 1.f; s.sp.temperature = 0.f;
    { std::vector<Sequence*> one{&s}; init_slots(one, nullptr, 0); }
    const int n = std::max(1, n_audio);
    std::vector<std::vector<int32_t>> aud(1);
    if (n_audio > 1) aud[0].assign(audio, audio + n_audio - 1);       // rows fed by t_1..t_{n-1}
    std::vector<int> last_rows; int max_nq = 0;
    std::vector<Sequence*> seqs{&s};
    const int M = build_prefill(seqs, aud, last_rows, max_nq);
    launch_build_rows(d_rows.p, M, tables(), wX.p, st);
    layers_forward(M, true, 1, max_nq);
    if (hidden_out) {
        // ln_f of every row
        launch_layernorm<float>(wX.p, lnfw.p, lnfb.p, wQKV.p, M, H, cfg.ln_eps, st);
        CUDA_CHECK(cudaMemcpyAsync(hidden_out, wQKV.p, (size_t)M * H * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    std::vector<int> ridx(n), slots(n, B), lpos(n);
    for (int i = 0; i < n; ++i) { ridx[i] = M - n + i; lpos[i] = i; }
    d_rowidx.upload(ridx.data(), n, st); d_active.upload(slots.data(), 1, st);
    DBuf<int> dslots; dslots.alloc(n); dslots.upload(slots.data(), n, st);
    d_lat_pos.upload(lpos.data(), n, st);
    head_and_sample(n, d_rowidx.p, dslots.p, d_lat_pos.p, 0, false);
    if (logits_out)
        CUDA_CHECK(cudaMemcpy2DAsync(logits_out, (size_t)V * sizeof(float), wLOG.p, (size_t)Vpad * sizeof(float),
                                     (size_t)V * sizeof(float), n, cudaMemcpyDeviceToHost, st));
    if (latents_out) d_latents.download(latents_out, (size_t)n * H, st, (size_t)B * CAP * H);
    CUDA_CHECK(cudaStreamSynchronize(st));
    release_slot(s);
}

void Engine::gpt_teacher_forced_sync(const int32_t* text, int n_text, int speaker, const int32_t* forced, int n,
                                     const xtts_sampling& sp, float* logits_out, float* latents_out, int32_t* sampled_out) {
    ApiLock lk(this);
    require_finalized();
    require_idle();
    if (n < 1 || n > CAP) throw std::runtime_error("teacher_forced: n out of range");
    CUDA_CHECK(cudaSetDevice(cfg.device));
    Sequence s; s.text_ids.assign(text, text + n_text); s.speaker = speaker; s.slot = B; s.sp = sp;
    s.sp.max_tokens = n;
    use_forced = forced != nullptr;
    try {
        std::vector<Sequence*> seqs{&s};
        init_slots(seqs, forced, n);
        prefill(seqs);                                   // samples token 1 (forced -> t_1)
        if (logits_out)
            CUDA_CHECK(cudaMemcpyAsync(logits_out, wLOG.p, (size_t)V * sizeof(float), cudaMemcpyDeviceToHost, st));
        std::vector<int> active{B};
        for (int k = 1; k < n; ++k) {
            decode_step(active);
            if (logits_out)
                CUDA_CHECK(cudaMemcpyAsync(logits_out + (size_t)k * V, wLOG.p, (size_t)V * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
        if (latents_out) d_latents.download(latents_out, (size_t)n * H, st, (size_t)B * CAP * H);
        if (sampled_out) d_sampled.download(sampled_out, n, st, (size_t)B * CAP);
        CUDA_CHECK(cudaStreamSynchronize(st));
    } catch (...) {
        use_forced = false; release_slot(s);
        throw;
    }
    use_forced = false;
    release_slot(s);
}

// The kernel isolation harness (harness.cu) behind the xtts_debug_* entry points: one call at a time on an idle engine
void Engine::run_idle(const std::function<void(const HarnessCtx&)>& f) {
    ApiLock lk(this);
    require_idle();
    CUDA_CHECK(cudaSetDevice(cfg.device));
    f(HarnessCtx{st, cfg.ln_eps, use_pdl, conditioner.get()});
}

}  // namespace xtts

// ================================================================================================
// C ABI
// ================================================================================================
using xtts::Engine;
using xtts::HarnessCtx;
struct xtts_engine { Engine* impl; };

#define XTTS_TRY(body)                                                  \
    try { Engine::Bind bind_ctx_(e->impl); body; return XTTS_OK; }      \
    catch (const xtts::CudaError& ex) { xtts::set_error(ex.what()); return XTTS_ERR_CUDA; } \
    catch (const xtts::StateError& ex) { xtts::set_error(ex.what()); return XTTS_ERR_STATE; } \
    catch (const std::exception& ex) { xtts::set_error(ex.what()); return XTTS_ERR_INVALID; } \
    catch (...) { xtts::set_error("unknown error"); return XTTS_ERR_INVALID; }

extern "C" {

const char* xtts_last_error(void) {
    if (!xtts::t_last_error.empty()) return xtts::t_last_error.c_str();
    std::lock_guard<std::mutex> lk(xtts::g_err_mu);
    xtts::t_last_error = xtts::g_last_error;
    return xtts::t_last_error.c_str();
}
const char* xtts_version(void) { return "libxtts_b200 0.1 (sm_90a)"; }

#define XTTS_TRY_UNBOUND(body)                                          \
    try { body; return XTTS_OK; }                                       \
    catch (const xtts::CudaError& ex) { xtts::set_error(ex.what()); return XTTS_ERR_CUDA; } \
    catch (const std::exception& ex) { xtts::set_error(ex.what()); return XTTS_ERR_INVALID; } \
    catch (...) { xtts::set_error("unknown error"); return XTTS_ERR_INVALID; }

int xtts_create(const xtts_config* cfg, xtts_engine** out) {
    if (!cfg || !out) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    XTTS_TRY_UNBOUND({ Engine* eng = new Engine(*cfg); *out = new xtts_engine{eng}; })
}
int xtts_destroy(xtts_engine* e) {
    if (!e) return XTTS_OK;
    XTTS_TRY_UNBOUND({ delete e->impl; delete e; })
}
int xtts_load_weight(xtts_engine* e, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
    XTTS_TRY(e->impl->load_weight(name, data, shape, ndim))
}
int xtts_finalize_weights(xtts_engine* e) { XTTS_TRY(e->impl->finalize_weights()) }
int xtts_set_speaker(xtts_engine* e, int32_t slot, const float* cond, const float* g) { XTTS_TRY(e->impl->set_speaker(slot, cond, g)) }
int xtts_get_speaker(xtts_engine* e, int32_t slot, float* cond, float* g) { XTTS_TRY(e->impl->get_speaker(slot, cond, g)) }
int xtts_condition(xtts_engine* e, int32_t slot, const float* wav22k, int64_t n22, const float* wav16k, int64_t n16,
                   int32_t gpt_cond_len_s, int32_t gpt_cond_chunk_len_s) {
    XTTS_TRY(e->impl->condition(slot, wav22k, n22, wav16k, n16, gpt_cond_len_s, gpt_cond_chunk_len_s))
}
int xtts_enhance(xtts_engine* e, const float* wav, int64_t n, const xtts_enhance_config* cfg, float* out, int64_t cap,
                 int64_t* n_out) {
    if (!cfg || !n_out) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    *n_out = xtts::Enhancer::out_len(n, *cfg);
    XTTS_TRY(*n_out = e->impl->enhance(wav, n, *cfg, out, cap))
}
int xtts_change_speed(xtts_engine* e, const float* wav, int64_t n, double rate, float* out, int64_t cap, int64_t* n_out) {
    if (!n_out) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    *n_out = xtts::PhaseVocoder::out_len(n, rate);
    XTTS_TRY(*n_out = e->impl->change_speed(wav, n, rate, out, cap))
}
int xtts_resample(xtts_engine* e, const float* wav, int64_t n, int32_t orig_sr, int32_t new_sr, float* out, int64_t cap,
                  int64_t* n_out) {
    if (!n_out) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    *n_out = xtts::Resampler::out_len(n, orig_sr, new_sr);
    XTTS_TRY(*n_out = e->impl->resample(wav, n, orig_sr, new_sr, out, cap))
}
int xtts_encode_flac(xtts_engine* e, const int16_t* pcm, int64_t n, int32_t sample_rate, const uint8_t* md5,
                     uint8_t* out, int64_t cap, int64_t* n_out) {
    if (!n_out) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    *n_out = 0;
    XTTS_TRY(e->impl->encode_flac(pcm, n, sample_rate, md5, out, cap, n_out))
}
int xtts_decode_flac(xtts_engine* e, const uint8_t* data, int64_t n_bytes, int32_t* out, int64_t cap,
                     xtts_flac_info* info) {
    if (!info) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    std::memset(info, 0, sizeof(*info));
    XTTS_TRY(e->impl->decode_flac(data, n_bytes, out, cap, info))
}
int xtts_submit(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                const xtts_sampling* sp) {
    return xtts_submit_speed(e, seq_id, text_ids, n_text, speaker_slot, sp, 1.0f);
}
int xtts_submit_speed(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                      const xtts_sampling* sp, float speed) {
    XTTS_TRY(e->impl->submit(seq_id, text_ids, n_text, speaker_slot, *sp, speed))
}
int xtts_submit_beams(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                      const xtts_sampling* sp, float speed, const xtts_beam* beam) {
    if (!sp || !beam) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    XTTS_TRY(e->impl->submit(seq_id, text_ids, n_text, speaker_slot, *sp, speed, beam))
}
int xtts_debug_beam_step(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t layers, int32_t V, const xtts_sampling* sp,
                         const xtts_beam* beam, int32_t first, int32_t advance, const float* logits, int32_t* n_gen,
                         int32_t* ctx_len, int32_t* last_tok, uint32_t* seen, int32_t max_pages, int32_t* block_tables,
                         int32_t n_pages, int32_t* pool, int32_t cap, int32_t* hist, xtts_beam_state* state, void* kpool,
                         void* vpool, float* scores) {
    if (!sp || !beam || !logits || !n_gen || !ctx_len || !last_tok || !seen || !block_tables || !pool || !hist || !state ||
        !kpool || !vpool || !scores) { xtts::set_error("null argument"); return XTTS_ERR_INVALID; }
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_beam_step(c, kv_type, heads, layers, V, *sp, *beam, first, advance, logits, n_gen, ctx_len, last_tok, seen,
                              max_pages, block_tables, n_pages, pool, cap, hist, state, kpool, vpool, scores);
    }))
}
int xtts_cancel(xtts_engine* e, uint64_t seq_id) { XTTS_TRY(e->impl->cancel(seq_id)) }
int xtts_poll(xtts_engine* e, xtts_result* out, int32_t timeout_ms) {
    try { return e->impl->poll(out, timeout_ms); }       // (no device work: nothing to bind)
    catch (const std::exception& ex) { xtts::set_error(ex.what()); return XTTS_ERR_INVALID; }
}
int xtts_fetch(xtts_engine* e, uint64_t seq_id, int32_t* tokens, float* wav, float* latents) {
    XTTS_TRY(e->impl->fetch(seq_id, tokens, wav, latents))
}
int xtts_set_option(xtts_engine* e, const char* key, int64_t value) { XTTS_TRY(e->impl->set_option(key, value)) }
int xtts_get_stats(xtts_engine* e, xtts_stats* out) { XTTS_TRY(e->impl->get_stats(out)) }
int xtts_sync(xtts_engine* e) { XTTS_TRY(e->impl->sync_idle()) }
int xtts_get_kernel_profile(xtts_engine* e, xtts_kernel_profile* out) { XTTS_TRY(e->impl->kernel_profile(out)) }
int xtts_device_timer(xtts_engine* e, int32_t op, double* ms) { XTTS_TRY(e->impl->device_timer(op, ms)) }
int xtts_debug_trace(xtts_engine* e, int32_t op, uint64_t* out, int32_t cap) {
    try { Engine::Bind b(e->impl); return e->impl->trace(op, out, cap); }
    catch (const std::exception& ex) { xtts::set_error(ex.what()); return XTTS_ERR_INVALID; }
}
int xtts_vocode(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, float* wav, int32_t* n_out,
                const char* stage, float* stage_out, int64_t stage_cap) {
    XTTS_TRY(e->impl->vocode_sync(latents, T, speaker_slot, wav, n_out, stage, stage_out, stage_cap))
}
int xtts_vocode_window(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, int32_t z0, int32_t nz, float* wav) {
    XTTS_TRY(e->impl->vocode_window_sync(latents, T, speaker_slot, z0, nz, wav))
}
int xtts_vocode_speed(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, float speed, int32_t z0, int32_t nz,
                      float* wav, int32_t* n_out) {
    XTTS_TRY(e->impl->vocode_speed_sync(latents, T, speaker_slot, speed, z0, nz, wav, n_out))
}
int xtts_gpt_prefill(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                     const int32_t* audio_tokens, int32_t n_audio, float* hidden_out, float* logits_out, float* latents_out) {
    XTTS_TRY(e->impl->gpt_prefill_sync(text_ids, n_text, speaker_slot, audio_tokens, n_audio, hidden_out, logits_out, latents_out))
}
int xtts_gpt_teacher_forced(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                            const int32_t* forced_tokens, int32_t n, const xtts_sampling* sp, float* logits_out,
                            float* latents_out, int32_t* sampled_out) {
    XTTS_TRY(e->impl->gpt_teacher_forced_sync(text_ids, n_text, speaker_slot, forced_tokens, n, *sp, logits_out, latents_out, sampled_out))
}
int xtts_debug_gemm(xtts_engine* e, int32_t mode, const float* A, const float* W, const float* bias, const float* resid,
                    float* out, int32_t M, int32_t N, int32_t K, int32_t flags, int32_t iters, float* ms_per_iter) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_gemm(c, mode, A, W, bias, resid, out, M, N, K, flags, iters, ms_per_iter);
    }))
}
int xtts_debug_ln_gemm(xtts_engine* e, int32_t mode, int32_t launch, int32_t M, int32_t N, int32_t K, const float* X,
                       const float* ln_w, const float* ln_b, const float* W, const float* bias, const float* resid, int32_t flags,
                       float* Y, float* out) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_ln_gemm(c, mode, launch, M, N, K, X, ln_w, ln_b, W, bias, resid, flags, Y, out);
    }))
}
int xtts_debug_norms(xtts_engine* e, int32_t out_type, int32_t M, int32_t H, const float* X, int32_t x_rows,
                     const int32_t* row_index, const float* w1, const float* b1, const float* w2, const float* b2, float* Y,
                     float* latents, int32_t n_slots, int32_t lat_rows, const int32_t* slots, const int32_t* lat_pos,
                     const int32_t* n_gen) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_norms(c, out_type, M, H, X, x_rows, row_index, w1, b1, w2, b2, Y, latents, n_slots, lat_rows, slots,
                          lat_pos, n_gen);
    }))
}
int xtts_debug_kv_write(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t M, const float* qkv, const int32_t* row_slot,
                        const int32_t* row_pos, int32_t n_slots, const int32_t* ctx_len, const int32_t* block_tables,
                        int32_t max_pages, int32_t n_pages, void* kpool, void* vpool) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_kv_write(c, kv_type, heads, M, qkv, row_slot, row_pos, n_slots, ctx_len, block_tables, max_pages, n_pages,
                             kpool, vpool);
    }))
}
int xtts_debug_build_rows(xtts_engine* e, int32_t H, int32_t n_cond, const float* text_emb, int32_t n_text, const float* text_pos,
                          int32_t n_text_pos, const float* wte, int32_t n_audio, const float* wpe, int32_t n_wpe,
                          const float* spk_cond, int32_t n_spk, const int32_t* rows, int32_t n_rows, float* X) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_build_rows(c, H, n_cond, text_emb, n_text, text_pos, n_text_pos, wte, n_audio, wpe, n_wpe, spk_cond, n_spk,
                               rows, n_rows, X);
    }))
}
int xtts_debug_build_decode_rows(xtts_engine* e, int32_t H, const float* wte, int32_t n_audio, const float* wpe, int32_t n_wpe,
                                 int32_t M, const int32_t* active, int32_t n_slots, const int32_t* last_tok, const int32_t* n_gen,
                                 float* X) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_build_decode_rows(c, H, wte, n_audio, wpe, n_wpe, M, active, n_slots, last_tok, n_gen, X);
    }))
}
int xtts_debug_sample_slots(xtts_engine* e, int32_t V, int32_t M, const int32_t* active, int32_t n_slots, const float* logits,
                            int32_t ld, const xtts_sampling* sp, int32_t cap, int32_t advance_ctx, const int32_t* forced,
                            int32_t* n_gen, int32_t* ctx_len, int32_t* finished, int32_t* last_tok, uint8_t* seen,
                            int32_t* tokens, int32_t* sampled) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_sample_slots(c, V, M, active, n_slots, logits, ld, sp, cap, advance_ctx, forced, n_gen, ctx_len, finished,
                                 last_tok, seen, tokens, sampled);
    }))
}
int xtts_debug_attn_decode(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t M, const int32_t* active, int32_t n_slots,
                           const int32_t* ctx_len, const int32_t* block_tables, int32_t max_pages, int32_t n_pages,
                           void* kpool, void* vpool, const float* qkv, float* out) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_attn_decode(c, kv_type, heads, M, active, n_slots, ctx_len, block_tables, max_pages, n_pages, kpool, vpool,
                                qkv, out);
    }))
}
int xtts_debug_attn_prefill(xtts_engine* e, int32_t out_type, int32_t heads, const int32_t* seqs, int32_t nseq, int32_t causal,
                            float scale, const float* q, int64_t q_len, int32_t q_row_stride, int32_t q_head_stride,
                            const float* kv, int64_t kv_len, int32_t kv_row_stride, int32_t kv_head_stride, int64_t k_off,
                            int64_t v_off, float* out, int32_t out_rows) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_attn_prefill(c, out_type, heads, seqs, nseq, causal, scale, q, q_len, q_row_stride, q_head_stride, kv,
                                 kv_len, kv_row_stride, kv_head_stride, k_off, v_off, out, out_rows);
    }))
}
int xtts_debug_splitk_ln(xtts_engine* e, int32_t mode, int32_t M, int32_t N, int32_t K, int32_t splits, const float* A,
                         const float* W, const float* bias, float* X, const float* ln_w, const float* ln_b, float* Y) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_splitk_ln(c, mode, M, N, K, splits, A, W, bias, X, ln_w, ln_b, Y);
    }))
}
int xtts_debug_conv_tc(xtts_engine* e, int32_t up, int32_t Cin, int32_t Cout, int32_t K, int32_t dil, int32_t batch, int32_t L,
                       const int32_t* item_len, const float* w, const float* bias, const float* cbias, int32_t cbias_stride,
                       const float* x, const float* resid, int32_t mode, float slope_out, float scale16, int32_t max_ctas,
                       float* out32, float* out16) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_conv_tc(c, up, Cin, Cout, K, dil, batch, L, item_len, w, bias, cbias, cbias_stride, x, resid, mode,
                            slope_out, scale16, max_ctas, out32, out16);
    }))
}
int xtts_debug_resblock_tc(xtts_engine* e, int32_t C, int32_t K, const int32_t* dil, int32_t batch, int32_t L,
                           const int32_t* item_len, const float* w, const float* bias, const float* x, int32_t mode,
                           float scale16, int32_t max_ctas, int32_t fused, float* zs, float* pa) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::debug_resblock_tc(c, C, K, dil, batch, L, item_len, w, bias, x, mode, scale16, max_ctas, fused, zs, pa);
    }))
}
int xtts_debug_cond(xtts_engine* e, int32_t op, const int32_t* dims, int32_t n_dims, const float* scal, int32_t n_scal,
                    const float* const* in, const int64_t* in_len, int32_t n_in, float* out, int64_t out_len) {
    XTTS_TRY(e->impl->run_idle([&](const HarnessCtx& c) {
        xtts::cond_debug(c.cnd, op, dims, n_dims, scal, n_scal, in, in_len, n_in, out, out_len, c.st);
    }))
}

}  // extern "C"
