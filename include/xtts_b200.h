/* libxtts_b200 — C ABI of the H100-native (sm_90a) XTTSv2 hot path.
 *
 * The reference (astramind-ai/Auralis) has no FFI of its own: its hot path sits behind two Python
 * surfaces, the `BaseAsyncTTSEngine` plugin API (src/auralis/models/base.py:57-224) and the vLLM
 * engine calls made by `XTTSv2Engine` (src/auralis/models/xttsv2/XTTSv2.py).  Each entry point below
 * names the reference call it stands in for; `INTEGRATION.md` shows the ctypes binding a maintainer
 * adds on the reference side.
 *
 * Conventions: every function returns 0 on success and a negative code on failure;
 * `xtts_last_error()` gives the message.  All pointers are HOST pointers owned by the caller unless
 * stated otherwise; sizes are in elements.  No torch types, no callbacks.  One engine = one GPU.
 * Thread-safe per engine (internal mutex + one scheduler thread).
 */
#ifndef XTTS_B200_H
#define XTTS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XTTS_OK 0
#define XTTS_ERR_INVALID -1
#define XTTS_ERR_CUDA -2
#define XTTS_ERR_STATE -3
#define XTTS_ERR_TIMEOUT -4
#define XTTS_ERR_CANCELLED -5 /* the chunk was cancelled with xtts_cancel before it finished */

#define XTTS_PRECISION_FP32 0 /* parity mode: fp32 CUDA-core GEMMs, fp32 KV cache            */
#define XTTS_PRECISION_BF16 1 /* fast mode: bf16 wgmma GEMMs (fp32 accumulate), bf16 KV      */
#define XTTS_PRECISION_FP16 2 /* fast mode with IEEE fp16 operands and KV: the same kernels at the same rate, 11 significand
                                 bits instead of 8 — closer to the fp32 parity mode (the reference's GPU vocoder is fp16 too) */

typedef struct xtts_engine xtts_engine;

/* Model geometry = the integers of XTTSGPTConfig / XTTSConfig
 * (config/xttsv2_gpt_config.py:133-229, config/xttsv2_config.py:237-301, hifigan_decoder.py:698-723). */
typedef struct xtts_config {
    int32_t device;            /* CUDA device ordinal                                          */
    int32_t precision;         /* XTTS_PRECISION_*                                             */
    int32_t max_batch;         /* concurrent sequences (= vLLM max_num_seqs, XTTSv2.py:224)    */
    int32_t max_speakers;      /* speaker-conditioning cache slots                             */
    /* GPT */
    int32_t hidden, layers, heads, ff;
    int32_t n_text_tokens, n_audio_tokens, start_audio_token, stop_audio_token;
    int32_t max_audio_tokens, max_text_tokens, n_cond_latents;
    float ln_eps;
    /* vocoder */
    int32_t voc_in_dim, voc_init_ch, voc_n_up;
    int32_t voc_up_rates[4], voc_up_kernels[4];
    int32_t voc_n_rb;
    int32_t voc_rb_kernels[4], voc_rb_dilations[4];
    int32_t d_vector;
    int32_t code_stride, output_hop_length, input_sample_rate, output_sample_rate;
    /* conditioning */
    int32_t n_mels, cond_blocks, perceiver_depth, perceiver_heads, perceiver_dim_head, perceiver_ff_mult;
    int32_t spk_layers[4], spk_filters[4], spk_mels, spk_proj;
} xtts_config;

/* Per-chunk sampling parameters = ExtendedSamplingParams built at XTTSv2.py:726-739. */
typedef struct xtts_sampling {
    float temperature, top_p, repetition_penalty;
    int32_t top_k, max_tokens, stop_token;
    uint64_t seed;             /* Philox key; the reference is unseeded                        */
    int32_t seq_seed;          /* per-sequence stream id                                       */
    int32_t vocode;            /* 1: run the vocoder on completion; 0: tokens + latents only   */
    int32_t priority;          /* admission order: lower first (the engine passes the chunk index,
                                  so every request's first chunk is decoded before any second chunk) */
    int32_t early_tokens;      /* 0 (default): one result per chunk, as the reference (FINAL_ONLY, XTTSv2.py:738).
                                  n > 0: streaming — the chunk's audio is delivered while it is still decoding: the samples
                                  of the first n tokens as soon as n + ~7 tokens exist, then (engine option "voc_segment" = m > 0)
                                  of every further m tokens, each as a PARTIAL result (status 1); the final result carries all
                                  tokens and the remaining samples.  Each piece is vocoded as a window with the vocoder's
                                  receptive field as margin, so the pieces concatenate to exactly the waveform of the
                                  unsplit chunk.  SURVEY.md §8f-3.                                                        */
} xtts_sampling;

typedef struct xtts_result {
    uint64_t seq_id;
    int32_t status;            /* 0 ok (final result), <0 failed / cancelled, 1 = partial piece (see early_tokens).
                                  xtts_fetch(seq_id) hands out the pieces of an id oldest first: fetch each result
                                  before polling further                                          */
    int32_t n_tokens;          /* final: = TTSOutput.token_length (XTTSv2.py:813), stop token included;
                                  partial: the tokens whose audio this piece carries               */
    int32_t n_samples;         /* 24 kHz samples                                               */
    int32_t n_prompt_rows;
    double t_submit, t_first_token, t_done;   /* seconds, engine clock                         */
} xtts_result;

typedef struct xtts_stats {
    uint64_t kernel_launches, decode_steps, prefill_rows, tokens_generated, samples_generated;
    double gpt_ms, vocoder_ms, cond_ms;        /* device time by CUDA events                   */
    uint64_t hbm_bytes_weights;
} xtts_stats;

/* Per-kernel-family device time (CUDA events on the engine's stream) and algorithmic FLOPs / bytes, collected
 * while option "profile" is 1 — what bench.py's `roofline` object is computed from. */
typedef struct xtts_kernel_profile {
    int32_t n;
    char name[16][32];
    double ms[16], flops[16], bytes[16];
    uint64_t launches[16];
} xtts_kernel_profile;

const char* xtts_last_error(void);
const char* xtts_version(void);

/* XTTSv2Engine.__init__/from_pretrained (XTTSv2.py:53-150,235-310): allocates weights, KV pages,
 * workspaces on `cfg->device`.  Fails loudly (XTTS_ERR_CUDA) if there is no sm_90 GPU. */
int xtts_create(const xtts_config* cfg, xtts_engine** out);
int xtts_destroy(xtts_engine* e);

/* load_state_dict / XttsGPT.load_weights (XTTSv2.py:289-301, vllm_mm_gpt.py:714-733): tensors are passed
 * by their checkpoint names (checkpoint_converter.py:230-272), fp32, host memory. */
int xtts_load_weight(xtts_engine* e, const char* name, const float* data, const int64_t* shape, int32_t ndim);
/* folds weight-norm, transposes/convert weights, verifies nothing is missing */
int xtts_finalize_weights(xtts_engine* e);

/* Speaker cache = the (gpt_cond_latent [32,H], speaker_embedding [d_vector]) pair returned by
 * get_audio_conditioning (XTTSv2.py:579-615) and reused by prepare_for_streaming_generation (tts.py:91-105). */
int xtts_set_speaker(xtts_engine* e, int32_t slot, const float* cond_latents, const float* d_vector);
int xtts_get_speaker(xtts_engine* e, int32_t slot, float* cond_latents, float* d_vector);
/* get_conditioning_latents (XTTSv2.py:409-468): reference audio -> speaker slot, computed on the GPU.
 * wav22k mono @22.05 kHz (already truncated to max_ref_length), wav16k the same audio @16 kHz. */
int xtts_condition(xtts_engine* e, int32_t slot, const float* wav22k, int64_t n22, const float* wav16k, int64_t n16,
                   int32_t gpt_cond_len_s, int32_t gpt_cond_chunk_len_s);

/* TTSRequest.enhance_speech (requests.py:199-248, enhancer.py:12-153): the reference's AudioPreprocessingConfig.
 * Flags are 0 / non-zero; the stages run in this order: trim_silence (VAD), remove_noise (spectral gating),
 * enhance_speech (clarity shaping), normalize (BS.1770 loudness to target_lufs, tanh soft clip). */
typedef struct xtts_enhance_config {
    int32_t sample_rate;
    int32_t normalize, trim_silence, remove_noise, enhance_speech;
    int32_t vad_frame_length, noise_reduce_frames;
    float vad_threshold, noise_reduce_margin, enhance_amount, target_lufs;
} xtts_enhance_config;
/* EnhancedAudioProcessor.process on the GPU, then the 16-bit PCM write/read of the reference's temp file
 * (rint(x * 32767) / 32768).  wav: n mono samples at cfg->sample_rate.  Writes *n_out samples to out (n_out <= n:
 * gating and clarity drop the tail past a multiple of 512); cap < *n_out fails with *n_out set.  Returns
 * XTTS_ERR_INVALID for a bad config and where the reference's enhancer fails: non-finite input, n < vad_frame_length
 * (or n <= 1024) with trim_silence, fewer than 0.4 s of audio at the loudness stage, a non-finite result.
 * Runs on the conditioning stream; its time counts in xtts_stats.cond_ms. */
int xtts_enhance(xtts_engine* e, const float* wav, int64_t n, const xtts_enhance_config* cfg, float* out, int64_t cap,
                 int64_t* n_out);

/* TTSOutput.change_speed (output.py:40-92): librosa.stft (n_fft 2048, hop 512) -> librosa.phase_vocoder(rate) ->
 * librosa.istft -> librosa.util.normalize(norm=inf) on the GPU, with librosa 0.10's arithmetic under NumPy's NEP 50
 * promotion.  wav: n mono samples (any sample rate).  rate > 1 is faster; a double, so the frame count ceil(T / rate)
 * (T = 1 + n / 512) and the frame positions t * rate are numpy's.  Writes *n_out = 512 * (ceil(T / rate) - 1) samples
 * with max |out| == 1 (all-zero input stays zero); *n_out is always set, cap < *n_out fails.  Returns XTTS_ERR_INVALID
 * where the reference raises: rate not finite or <= 0, a non-finite sample, an empty result (ceil(T / rate) == 1), a
 * non-finite result.  Works in blocks of at most "pvoc_block_frames" output frames (bit-identical for every value).
 * Runs on the conditioning stream; its time counts in xtts_stats.cond_ms. */
int xtts_change_speed(xtts_engine* e, const float* wav, int64_t n, double rate, float* out, int64_t cap, int64_t* n_out);

/* torchaudio.functional.resample(wav, orig_sr, new_sr) with its defaults (sinc_interp_hann, lowpass_filter_width 6,
 * rolloff 0.99), the reference's resampler for speaker files, conditioning and TTSOutput.resample (common/utilities.py:94,
 * models/base.py:220, XTTSv2.py:322,362), on the GPU: wav n mono float32 samples at orig_sr Hz -> *n_out = ceil(M n / L)
 * samples at new_sr Hz (L, M = the rates over their gcd).  Coefficients are torchaudio's float32 kernel, built with its
 * operation order; only the taps whose scaled argument lies strictly inside the window (-6, 6) are evaluated (at most
 * 2 width + 2 per output, width = ceil(6 L / (0.99 min(L, M)))).  The taps torchaudio also evaluates have the clamped
 * argument +-6 and coefficients below 5e-24.  Each output is an fp32 FMA chain in a fixed tap order, so it does not
 * depend on the launch shape.  Input outside [0, n) reads as 0.  orig_sr == new_sr copies the samples; n == 0 gives 0.
 * Workspace: a band table of about M (2 width + 2) floats, cached for the last rate pair, and passes of at most
 * "resample_block_samples" outputs with the input they read (2 x that many + 2 width + L floats); bit-identical for
 * every value.  *n_out is always set (0 for an invalid rate or length); cap < *n_out fails.  XTTS_ERR_INVALID: a rate
 * outside 1 .. 1048575, n < 0, a NULL pointer with n > 0, cap < *n_out, a non-finite sample (checked on the device).
 * Runs on the conditioning stream; its time counts in xtts_stats.cond_ms. */
int xtts_resample(xtts_engine* e, const float* wav, int64_t n, int32_t orig_sr, int32_t new_sr, float* out, int64_t cap,
                  int64_t* n_out);

/* TTSOutput.to_bytes("flac") (output.py:119-187): a complete, lossless FLAC stream (RFC 9639) of n mono 16-bit samples
 * at sample_rate Hz, encoded on the GPU.  "fLaC", one STREAMINFO block (min/max block size 4096, the real min/max frame
 * sizes, total samples n, the 16-byte md5 the caller passes or zeros for NULL = "not computed"), then fixed blocks of
 * 4096 samples (the last holds the remainder), 16 bits, no wasted bits.  Each block keeps the smallest of these
 * subframes, exactly costed in bits (ties: the first): CONSTANT (all samples equal), VERBATIM, FIXED orders 0..4, LPC
 * orders 1..12 at 12-bit precision with shift 0..15 (Tukey(0.5)-windowed fp64 autocorrelation, Levinson-Durbin; an
 * order whose residual would reach |r| >= 2^31 is dropped).  An order o is tried only on blocks of more than o
 * samples; a 1-sample block is CONSTANT.  Residuals: partitioned Rice (method 00, parameters 0..14, no escape),
 * partition orders 0..6 where the block allows, each parameter by exact cost.  No subframe is larger than VERBATIM, so
 * the stream is at most 42 + ceil(n / 4096) * 8211 bytes.  *n_out is always set (the length needed when cap is too
 * small); cap < *n_out fails.  XTTS_ERR_INVALID: sample_rate outside 1 .. 1048575, n < 0, a NULL pcm with n > 0,
 * cap < *n_out.  n == 0 gives STREAMINFO and no frames.  Works in batches of at most "flac_batch_frames" frames (the
 * bytes are identical for every value).  Runs on the conditioning stream; its time counts in xtts_stats.cond_ms. */
int xtts_encode_flac(xtts_engine* e, const int16_t* pcm, int64_t n, int32_t sample_rate, const uint8_t* md5,
                     uint8_t* out, int64_t cap, int64_t* n_out);

/* FLAC input for speaker references (engine.load_audio) and TTSOutput.from_file (common/utilities.py:72-97,
 * output.py:274-285, where torchaudio.load decodes it through ffmpeg): a whole FLAC stream (RFC 9639) -> planar int32
 * samples out[channels][total_samples], each the signed integer the frames code, right-aligned (lossless).  Accepts
 * an ID3v2 tag before "fLaC", any metadata blocks after STREAMINFO, 1-8 channels, 4-32 bits per sample, fixed and
 * variable blocking, independent / left-side / side-right / mid-side channels, CONSTANT, VERBATIM, FIXED 0-4 and LPC
 * 1-32 subframes with wasted bits, RICE and RICE2 residuals with escapes and partition orders up to 15.  The stream
 * ends after the frames holding STREAMINFO's total (trailing bytes are ignored); a total of 0 means the frames run to
 * the end of the data, before a 128-byte ID3v1 "TAG" trailer if there is one, and the total is what they hold.
 * *info is filled whenever the metadata parses (total_samples: the decoded count); cap < channels * total_samples
 * fails with *info telling the caller what to allocate.  XTTS_ERR_INVALID, never a wrong sample, for: no "fLaC", a
 * first block that is not a 34-byte STREAMINFO, block type 127, truncation anywhere, a sync code / reserved value /
 * reserved bit / header field that disagrees with STREAMINFO, a CRC-8 or CRC-16 mismatch, frame or sample numbers
 * out of sequence, a fixed-blocksize stream whose block size changes before its last frame, non-zero padding, LPC
 * precision 1111 or a negative shift, a residual outside 32 bits, a sample outside its bit depth.  The MD5 is NOT
 * checked here (native.py checks it).  Frames are found by a scan of every byte position on the GPU and decoded in
 * batches of at most "flac_batch_frames" frames and flac_batch_frames * 4096 samples (identical samples for every
 * value).  Runs on the conditioning stream; its time counts in xtts_stats.cond_ms. */
typedef struct xtts_flac_info {
    int32_t sample_rate, channels, bits_per_sample, min_block, max_block;
    int64_t total_samples;          /* per channel, as decoded */
    uint8_t md5[16];                /* STREAMINFO's; all zero = not set */
} xtts_flac_info;
int xtts_decode_flac(xtts_engine* e, const uint8_t* data, int64_t n_bytes, int32_t* out, int64_t cap,
                     xtts_flac_info* info);

/* llm_engine.generate(...) per text chunk (XTTSv2.py:741-757): text_ids = [bos]+bpe+[eos] (XTTSv2.py:519-522).
 * Asynchronous: the scheduler thread admits, prefills, decodes (continuous batching), vocodes. */
int xtts_submit(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                const xtts_sampling* sp);
/* xtts_submit with a speaking rate (Coqui Xtts.inference(speed=...); xtts_submit = speed 1).  speed in [0.25, 4] (the range
 * of OpenAI's /v1/audio/speech; > 1 is faster), anything else — NaN included — fails this call with XTTS_ERR_INVALID before
 * anything is queued.  The GPT decode is untouched (same tokens, same latents); the T latents of the chunk are time-scaled
 * by one more linear interpolation to T0 = floor(T * ls) frames, ls = 1 / (double)speed, before the vocoder's own two
 * (F.interpolate(scale_factor = ls, mode "linear")), so the pitch stays.  n_samples = 256 * z_frames(T0); T0 == 0 (e.g. 3
 * tokens at speed 4) gives a final result with every token and 0 samples.  Speed 1 skips the stage: bit-identical to
 * xtts_submit (and so does T0 == T, where F.interpolate copies).  Streaming (early_tokens, "voc_segment") works at any
 * speed; a finished chunk longer than one vocoder window is vocoded in several, none of them a partial result. */
int xtts_submit_speed(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                      const xtts_sampling* sp, float speed);
/* Beam-search decoding of one chunk (Coqui Xtts.inference(num_beams, length_penalty, do_sample) -> transformers'
 * generate): transformers 5.5 _beam_search for one batch item, num_return_sequences 1, early_stopping unset.  Each step
 * takes log_softmax of the mel-head logits in fp32, applies the repetition penalty over the prompt ids and the beam's own
 * hypothesis (s < 0 ? s * p : s / p) and, with do_sample, temperature, top-k and top-p (min_tokens_to_keep 2), adds the
 * beam's running score and picks 2 num_beams candidates over num_beams x V: the top ones (ties: the lower
 * beam * V + token), or with do_sample draws without replacement by an Exp(1) race on the sampler's Philox stream
 * (key = seed, counter = ((beam * V + token) / 4, step, seq_seed, 0)).  Finished candidates (stop token, or max_tokens)
 * are scored score / gen_len ^ length_penalty into the best-num_beams finished set; the group stops by transformers'
 * default heuristic.  The result is the best finished hypothesis: its tokens (stop token included), and latents and
 * samples exactly as xtts_submit_speed would give for those token ids.  num_beams beams take num_beams batch slots and
 * KV pages for num_beams full-length chunks; they share the prompt's pages and fork each other's pages every step.
 * num_beams in 1 .. 8 and <= max_batch, early_tokens 0 when num_beams > 1 (no partial results: the hypothesis is known
 * only at the end), a finite length_penalty, temperature > 0 with do_sample (transformers rejects it too), and an engine
 * geometry the beam kernels take (<= 128 KV pages per chunk); otherwise XTTS_ERR_INVALID.  num_beams == 1 is xtts_submit_speed. */
typedef struct xtts_beam {
    int32_t num_beams;
    float length_penalty;
    int32_t do_sample;         /* 0: beam search, non-zero: beam sampling */
} xtts_beam;
int xtts_submit_beams(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                      const xtts_sampling* sp, float speed, const xtts_beam* beam);
/* One beam step on caller arrays, for the isolation tests: logprob, select, reorder and partial-page copy of the engine's
 * beam kernels, on one group of num_beams = nb (2..8) beams in slots 0..nb-1, without the final gather.  V <= 2048 tokens;
 * sp: repetition_penalty, temperature / top_k / top_p (do_sample), max_tokens, stop_token, seed, seq_seed.  first: the
 * group's first selection (row 0 of logits for every beam, running scores [0, -1e9, ...], only beam 0 owns pages);
 * advance: KV positions the step appended (0 after the prefill, 1 after a decode step).  In / out: n_gen, ctx_len [nb]
 * (equal across beams), seen [nb][ceil(V / 32)] bitmaps, block_tables [nb][max_pages] (max_pages <= 128), pool [nb *
 * max_pages] (the first state->n_free entries are free page ids, n_free >= nb), hist [cap][8][2] (parent, token) rows,
 * *state (the group state, transformers' beam-search tensors; sel_* / copy_* are this step's outputs), kpool / vpool
 * [layers][n_pages pages] in the layout of xtts_debug_attn_decode, kv_type 0 fp32, 1 bf16, 2 fp16, 3 fp8 (a copied token
 * takes its exponent bytes along).  Out: last_tok [nb],
 * scores [nb][V] (the processed, accumulated scores the selection ranked).  logits: [1][V] when first, else [nb][V]. */
typedef struct xtts_beam_state {
    float run_score[8], fin_score[8];
    int32_t fin_valid[8], fin_step[8], fin_beam[8], fin_tok[8];
    int32_t heur_unsat, done;
    int32_t sel_parent[8], sel_tok[8];
    int32_t n_copy, copy_src[8], copy_dst[8], copy_ntok[8];
    int32_t n_free, n_pages[8];
} xtts_beam_state;
int xtts_debug_beam_step(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t layers, int32_t V, const xtts_sampling* sp,
                         const xtts_beam* beam, int32_t first, int32_t advance, const float* logits, int32_t* n_gen,
                         int32_t* ctx_len, int32_t* last_tok, uint32_t* seen, int32_t max_pages, int32_t* block_tables,
                         int32_t n_pages, int32_t* pool, int32_t cap, int32_t* hist, xtts_beam_state* state, void* kpool,
                         void* vpool, float* scores);
/* Aborts a chunk (the reference aborts the vLLM request when its generator is dropped).  A queued chunk is dropped, a
 * decoding one stops at the scheduler's next iteration and returns its batch slot and KV pages; either way exactly one
 * final result with status XTTS_ERR_CANCELLED is delivered.  Unknown / already finished ids are ignored. */
int xtts_cancel(xtts_engine* e, uint64_t seq_id);
/* completion queue (replaces `async for output in generator` + get_model_logits + hifigan_decoder,
 * XTTSv2.py:785-814).  Returns 1 and fills *out when a chunk finished, 0 on timeout. */
int xtts_poll(xtts_engine* e, xtts_result* out, int32_t timeout_ms);
/* copies out and releases the OLDEST unfetched result of a chunk (its partial pieces, then the final one); any of tokens /
 * wav / latents may be NULL (a partial piece has no latents; a failed result has no data and is only released). */
int xtts_fetch(xtts_engine* e, uint64_t seq_id, int32_t* tokens, float* wav, float* latents);
/* engine knobs (key, value):
 *   "d2h_wav"             0 = leave waveforms in HBM (kernel-only timing), 1 = D2H into pinned memory (default)
 *   "cuda_graphs" / "pdl" / "splitk" / "tc_vocoder"   0/1, fast-mode execution features (all default 1)
 *   "hold_admission"      1 = queue submissions without admitting them, 0 = release (atomic batch submit)
 *   "decode_chain"        0 only (a no-op, kept so that callers passing it keep working); any other value is an error:
 *                         the fused persistent per-layer GEMM/LayerNorm chain kernel was removed
 *   "microbatches"        1..4 concurrent branches the decode step's rows are split into (default 2)
 *   "microbatch_min_rows" steps with fewer active rows stay single-branch (default 48)
 *   "gemm_wide"           4 (default), 3 or 2 = GEMMs with M >= 256 rows (prefill, conditioning) run on the persistent
 *                         wide-tile kernel (128x256 tiles) with that ring depth, 0 = the one-tile-per-CTA kernel
 *   "voc_segment"         m > 0: a chunk is vocoded in windows of m tokens WHILE it decodes (the vocoder runs on its own
 *                         stream beside the decode step), 0 = one window per chunk when it ends.  Same samples either way.
 *   "voc_sms"             SMs the vocoder's persistent conv kernels may occupy while a decode step is in flight (0 = all)
 *   "voc_batch"           windows per vocoder launch (1..32, default 32; ragged lengths are batched together)
 *   "pvoc_block_frames"   xtts_change_speed's block: at most this many output STFT frames (and this many + 2 input frames)
 *                         per pass, 1 .. 2^20, default 4096 (a spectral workspace of about 45 KB per frame, ~185 MB,
 *                         whatever the input length).  Bit-identical results for every value.
 *   "flac_batch_frames"   xtts_encode_flac's batch: at most this many 4096-sample frames on the device at once, 1 .. 2^20,
 *                         default 8192 (about 16 KB of device memory per frame, ~135 MB, whatever the input length).
 *                         Identical bytes for every value.  xtts_decode_flac's batch: at most this many frames and this
 *                         many x 4096 samples, all channels together (one larger frame is a batch alone); about 4 B
 *                         per sample (12 B at 32 bits) beside the compressed stream, which is whole on the device.
 *                         Identical samples for every value.
 *   "resample_block_samples"   xtts_resample's pass: at most this many output samples, and the input they read (at most
 *                         this many + 2 width + L samples) per pass, 1 .. 2^26, default 2^22 (about 32 MB of device memory
 *                         at the default, whatever the input length).  Bit-identical results for every value.
 *   "tc_epilogue"         epilogue of the fast-mode vocoder's tensor-core Conv1d: 1 (default) = staged through shared
 *                         memory (residual prefetched by a loader warp, outputs drained by bulk copies while the next
 *                         tile's MMAs run), 0 = straight from the accumulators.  Bit-identical results either way.
 *   "tc_resblock"         test / measurement switch, not a tuning knob (the path follows from the channel count): 1
 *                         (default) = the fast-mode vocoder's resblocks of 32 or 64 channels run as one fused kernel each
 *                         (resblock_tc) wherever it takes their geometry, 0 = as six tensor-core Conv1d launches, for
 *                         A/B timing and the bit-identity tests.  Bit-identical results.
 *   "kv_fp8"              1 = the KV cache in fp8 e4m3 with one power-of-two scale per (token, head) for K and for V
 *                         (layout at xtts_debug_attn_decode): half the KV bytes per slot and per decode step; 0 (default) =
 *                         the cache in the precision's 16-bit type.  bf16 / fp16 precision only (fp32: XTTS_ERR_INVALID),
 *                         on an idle engine only (a queued or running chunk: XTTS_ERR_STATE).  Switching reallocates the KV
 *                         pools in the chosen format and drops the captured decode graphs; 0 again gives the bits of an
 *                         engine that never switched.
 *   "attn_ctas_per_sm"    > 0 caps the decode-attention grid (each CTA walks several items); < 0: absolute grid size (tests)
 *   "profile"             1 = CUDA events around every launch (xtts_get_kernel_profile), "reset_stats" = zero the counters */
int xtts_set_option(xtts_engine* e, const char* key, int64_t value);
int xtts_get_stats(xtts_engine* e, xtts_stats* out);
int xtts_sync(xtts_engine* e);   /* waits until no submitted work is pending */
int xtts_get_kernel_profile(xtts_engine* e, xtts_kernel_profile* out);
/* device-side stopwatch for bench.py: op 0 records a CUDA event on the engine's stream (call with the engine idle);
 * op 1 records a second one behind all work submitted so far, waits for it and returns the elapsed milliseconds
 * between the two in *ms.  No reference counterpart (the reference times with time.time(), two_phase_scheduler.py:139). */
int xtts_device_timer(xtts_engine* e, int32_t op, double* ms);

/* ---- synchronous single-stage entry points (parity tests; they serialise with the scheduler) ---- */
/* HifiDecoder.forward (hifigan_decoder.py:776-802): latents [T,in_dim] -> wav [n_samples]. Returns n_samples
 * in *n_out; `stage` (may be NULL) names an intermediate to copy to stage_out ("z","pre","up0","mrf0",...). */
int xtts_vocode(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, float* wav, int32_t* n_out,
                const char* stage, float* stage_out, int64_t stage_cap);
/* The vocoder on z-frames [z0, z0 + nz) of the chunk `latents` [T, in_dim] as a window of its own: wav [nz * 256].
 * Samples further than the generator's receptive field (~14 z-frames) from an inner window edge equal the whole chunk's —
 * the property "voc_segment" / early_tokens rest on (tests/test_gpu_vocoder.py). */
int xtts_vocode_window(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, int32_t z0, int32_t nz, float* wav);
/* The vocoder at a speaking rate (speed in [0.25, 4], see xtts_submit_speed): z-frames [z0, z0 + nz) of the speed-scaled
 * chunk as a window of its own (wav [nz * 256]), or with nz < 0 the whole chunk (wav [256 * z_frames(T0)]).
 * A whole chunk longer than the vocoder workspace (slow rates: up to 4x the frames) is vocoded in the windows the scheduler
 * cuts for it, their kept samples stitched — the same samples a submitted chunk gets.  *n_out = samples written (0 when
 * T0 == 0).  At speed 1: nz < 0 is xtts_vocode, nz >= 0 is xtts_vocode_window, bit for bit. */
int xtts_vocode_speed(xtts_engine* e, const float* latents, int32_t T, int32_t speaker_slot, float speed, int32_t z0, int32_t nz,
                      float* wav, int32_t* n_out);
/* one prefill over [prompt ; forced audio tokens] (the reference's 2nd pass, XTTSv2.py:617-687):
 * outputs ln_f hidden of every row, raw logits + latents of the last n_audio rows */
int xtts_gpt_prefill(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                     const int32_t* audio_tokens, int32_t n_audio, float* hidden_out, float* logits_out,
                     float* latents_out);
/* prefill + step-by-step decode with forced tokens: raw logits [n,V], latents [n,H], sampled ids [n] */
int xtts_gpt_teacher_forced(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                            const int32_t* forced_tokens, int32_t n, const xtts_sampling* sp, float* logits_out,
                            float* latents_out, int32_t* sampled_out);
/* GEMM under test: mode 0 = fp32 CUDA-core, 1 = bf16 wgmma, 2 = fp16 wgmma.  A [M,K], W [N,K], bias [N] or NULL, resid [M,N] or NULL;
 * out [M,N] = epi(A . W^T + bias) under the engine's current GEMM options ("gemm_wide", "gemm_bn").  flags (XTTS_DEBUG_GEMM_*; 0 / 1 = without / with GELU, as before the flag word):
 *   GELU    gelu_new after the bias, before the residual
 *   OUT16   16-bit output in the operand type (modes 1 / 2, no resid), returned widened to fp32
 *   INPLACE out is preloaded with resid and passed as the residual too (the engine's o-proj / down-proj without split-K)
 *   PDL     launched with programmatic dependent launch behind the kernel that converts A (modes 1 / 2; the launch then never
 *           goes to the wide-tile kernel)
 * Rejected before any launch: unknown bits, OUT16 / PDL in mode 0, INPLACE without resid or with OUT16, K % 64 or N % 32 in
 * modes 1 / 2.  iters > 0: *ms_per_iter = mean time of that many further launches. */
#define XTTS_DEBUG_GEMM_GELU 1
#define XTTS_DEBUG_GEMM_OUT16 2
#define XTTS_DEBUG_GEMM_INPLACE 4
#define XTTS_DEBUG_GEMM_PDL 8
int xtts_debug_gemm(xtts_engine* e, int32_t mode, const float* A, const float* W, const float* bias, const float* resid,
                    float* out, int32_t M, int32_t N, int32_t K, int32_t flags, int32_t iters, float* ms_per_iter);
/* debug timeline: op 1 arms %globaltimer stamps in the decode / vocoder kernels (first and last CTA: entry, dependency
 * resolved, exit), op 0 disarms and copies up to `cap` records [n][2] u64 = (ns, id<<32 | grid<<40 | last<<8 | phase) into
 * `out`; returns the count (>= 0) or a negative error.  Nothing is serialised: shows the step as it really runs. */
int xtts_debug_trace(xtts_engine* e, int32_t op, uint64_t* out, int32_t cap);
/* Single-kernel entry points below: an idle engine, private device buffers, the engine's current kernel options
 * (xtts_set_option), no engine state touched. */
/* fused sampler (one launch): row r of logits [M][ld] samples for slot active[r] (M distinct slots < n_slots) over ids
 * 0 .. V-1 (1 <= V <= 2048, ld >= V) with the slot's parameters sp[slot] (temperature, top_p, repetition_penalty, top_k,
 * max_tokens, stop_token, seed, seq_seed; the other fields are ignored).  Per-slot state, in/out, as the kernel leaves
 * it for active and inactive slots alike: n_gen, ctx_len, finished, last_tok [n_slots]; seen [n_slots][V] (0/1, the
 * penalty set); tokens, sampled [n_slots][cap].  forced [n_slots][cap] or NULL: an entry >= 0 at [slot][n_gen] replaces
 * the drawn id in tokens / last_tok / seen.  advance_ctx 1 adds one to ctx_len of every active slot.  Rejected before
 * any launch: V, M, ld or cap out of range, duplicate or out-of-range active slots, a negative n_gen, NULL (except
 * forced), and with forced an n_gen >= cap or a forced id >= V. */
int xtts_debug_sample_slots(xtts_engine* e, int32_t V, int32_t M, const int32_t* active, int32_t n_slots, const float* logits,
                            int32_t ld, const xtts_sampling* sp, int32_t cap, int32_t advance_ctx, const int32_t* forced,
                            int32_t* n_gen, int32_t* ctx_len, int32_t* finished, int32_t* last_tok, uint8_t* seen,
                            int32_t* tokens, int32_t* sampled);
/* paged decode attention (one launch, appends each row's k / v): kv_type 0 fp32, 1 bf16, 2 fp16 (the output has the cache
 * type, returned as fp32), 3 fp8 cache with fp16 output, 4 fp8 cache with bf16 output.  active [M] (distinct slots <
 * n_slots), ctx_len [n_slots], block_tables [n_slots][max_pages]; kpool / vpool: n_pages pages of raw cache-typed elements in
 * the device layout (K [page][head][64/X][32 tok][X], X = 16 bytes per element group; V [page][head][32 tok][64]), updated
 * in place; qkv [M][3 * heads * 64]; out [M][heads * 64].
 * fp8 (kv_type 3 / 4): each (page, head) block is 2080 bytes, the e4m3 data in the layout above (X = 16) followed by 32 int8
 * exponents, one per token: value = e4m3 * 2^e.  Per (token, head), for K and V separately, e is the smallest integer with
 * max |x| * 2^-e <= 448, clamped to [-128, 127] (-128 for an all-zero row), and the byte is e4m3(x * 2^-e) rounded to
 * nearest even. */
int xtts_debug_attn_decode(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t M, const int32_t* active, int32_t n_slots,
                           const int32_t* ctx_len, const int32_t* block_tables, int32_t max_pages, int32_t n_pages,
                           void* kpool, void* vpool, const float* qkv, float* out);
/* prefill / encoder attention (head dim 64): out_type 0 fp32, 1 bf16, 2 fp16 (returned as fp32); seqs [nseq][4] =
 * (q_start, nq, kv_start, nk); q element (row r, head h, dim d) at q[r * q_row_stride + h * q_head_stride + d], k / v at
 * kv[k_off | v_off + r * kv_row_stride + h * kv_head_stride + d]; causal: key j visible to query i iff j <= i + nk - nq;
 * out [out_rows][heads * 64], rows outside every sequence are NaN */
int xtts_debug_attn_prefill(xtts_engine* e, int32_t out_type, int32_t heads, const int32_t* seqs, int32_t nseq, int32_t causal,
                            float scale, const float* q, int64_t q_len, int32_t q_row_stride, int32_t q_head_stride,
                            const float* kv, int64_t kv_len, int32_t kv_row_stride, int32_t kv_head_stride, int64_t k_off,
                            int64_t v_off, float* out, int32_t out_rows);
/* decode projection as in fast mode: mode 1 bf16 / 2 fp16 operands, partials = split-K GEMM of A [M,K] . W [N,K]^T in `splits`
 * K ranges, then X [M,N] += bias + sum of partials (in place) and Y = LayerNorm(X; ln_w, ln_b, the engine's eps) in the
 * 16-bit type (returned as fp32); ln_w = ln_b = NULL: X only (the last layer) */
int xtts_debug_splitk_ln(xtts_engine* e, int32_t mode, int32_t M, int32_t N, int32_t K, int32_t splits, const float* A,
                         const float* W, const float* bias, float* X, const float* ln_w, const float* ln_b, float* Y);
/* the decode step's LayerNorm -> GEMM pair as the fast-mode decode launches it (mode 1 bf16 / 2 fp16): Y [M,K] =
 * LayerNorm(X [M,K]; ln_w, ln_b, the engine's eps) in the 16-bit type (returned as fp32), then out [M,N] = epi(Y . W^T + bias)
 * + resid on the one-tile GEMM, flags XTTS_DEBUG_GEMM_GELU / OUT16 only (OUT16: 16-bit out, returned as fp32, no resid).
 * launch 0: plain launches; 1: both with PDL.  Rejected before any launch: another launch mode, N % 32, K % 64, K > 8192,
 * NULL except bias / resid. */
int xtts_debug_ln_gemm(xtts_engine* e, int32_t mode, int32_t launch, int32_t M, int32_t N, int32_t K, const float* X,
                       const float* ln_w, const float* ln_b, const float* W, const float* bias, const float* resid, int32_t flags,
                       float* Y, float* out);
/* LayerNorms in the output type out_type (0 fp32, 1 bf16, 2 fp16; returned as fp32), eps = the engine's, H <= 8192.
 * w2 == b2 == NULL: Y[i] = LN(X[i]; w1, b1) for i < M (row_index, latents NULL; x_rows >= M).
 * w2 != NULL, the GPT head: r = row_index ? row_index[i] : i (< x_rows), y = LN(LN(X[r]; w1, b1); w2, b2), Y[i] = y, and with
 * latents [n_slots][lat_rows][H] (in/out, may be NULL): latents[slots[i]][p] = LN(y; w2, b2), p = lat_pos ? lat_pos[i] :
 * n_gen[slots[i]], written only when 0 <= p < lat_rows.  Rejected before any launch: a row index outside X, a slot outside
 * n_slots, latents without slots / lat_rows / lat_pos or n_gen. */
int xtts_debug_norms(xtts_engine* e, int32_t out_type, int32_t M, int32_t H, const float* X, int32_t x_rows,
                     const int32_t* row_index, const float* w1, const float* b1, const float* w2, const float* b2, float* Y,
                     float* latents, int32_t n_slots, int32_t lat_rows, const int32_t* slots, const int32_t* lat_pos,
                     const int32_t* n_gen);
/* the prefill's paged-cache write: k / v of QKV row r (qkv [M][3 * heads * 64]) go to slot row_slot[r] at token position
 * p = row_pos ? row_pos[r] : ctx_len[row_slot[r]], page block_tables[slot][p / 32], rounded to kv_type (0 fp32, 1 bf16,
 * 2 fp16, 3 / 4 fp8 with its exponents).  kpool / vpool: raw pools in the layout of xtts_debug_attn_decode, updated in place.  Rejected before any
 * launch: a slot outside n_slots, a position outside the block table, a page id outside the pool. */
int xtts_debug_kv_write(xtts_engine* e, int32_t kv_type, int32_t heads, int32_t M, const float* qkv, const int32_t* row_slot,
                        const int32_t* row_pos, int32_t n_slots, const int32_t* ctx_len, const int32_t* block_tables,
                        int32_t max_pages, int32_t n_pages, void* kpool, void* vpool);
/* prompt row build over private fp32 tables [rows][H] (H % 4 == 0): rows [n_rows][4] = (kind, a, b, c) as the engine builds
 * them: kind 0 X = spk_cond[c][a] (spk_cond [n_spk][n_cond][H]); 1 X = text_emb[a] + text_pos[b]; 2 X = wte[a] + wpe[b].
 * Rejected before any launch: another kind, an index outside its table. */
int xtts_debug_build_rows(xtts_engine* e, int32_t H, int32_t n_cond, const float* text_emb, int32_t n_text, const float* text_pos,
                          int32_t n_text_pos, const float* wte, int32_t n_audio, const float* wpe, int32_t n_wpe,
                          const float* spk_cond, int32_t n_spk, const int32_t* rows, int32_t n_rows, float* X);
/* decode row build: X[i] = wte[last_tok[s]] + wpe[n_gen[s]], s = active[i] < n_slots.  Launched with PDL when option "pdl"
 * is on.  Rejected before any launch: a slot, token or position outside its table. */
int xtts_debug_build_decode_rows(xtts_engine* e, int32_t H, const float* wte, int32_t n_audio, const float* wpe, int32_t n_wpe,
                                 int32_t M, const int32_t* active, int32_t n_slots, const int32_t* last_tok, const int32_t* n_gen,
                                 float* X);
/* fast-mode vocoder convolution on the tensor cores (fp16 operands, fp32 accumulate), weights packed as the engine packs
 * them.  up 0: Conv1d(Cin -> Cout, odd K, dilation dil, "same" padding), w [Cout][Cin][K]; up u in {2, 4, 8}:
 * ConvTranspose1d(Cin -> Cout, kernel K = 2u, stride u, padding u/2), w [Cin][Cout][2u], dil 1, no resid, mode 0,
 * scale16 1.  x [batch][Cin][L]: the already-activated input, rounded to fp16; item_len [batch] (0 <= L_i <= L) or NULL
 * (all L).  Lout = L * u (up > 0) or L.  bias [Cout], cbias [batch][cbias_stride], resid [batch][Cout][Lout]: each
 * optional.  Per item i and output step t < Lout_i:
 *   y = conv(x_i) + bias + cbias_i + resid_i;  out32 = y (mode 0) or out32 + y (mode 1, needs out32);
 *   out16 = fp16(lrelu(out32 value * scale16, slope_out))   (with mode 1: the activated sum)
 * out32 [batch][Cout][Lout] fp32 and out16 [batch][Cout/8][lpad(Lout)][8] (the raw output atom image, uploaded as fp16 and
 * returned as fp32, lpad(n) = 64 + ceil((n + 1) / 512) * 512 + 64, signal at rows 64 .. 64 + Lout_i) are in/out, NULL = not
 * produced; rows the kernel does not write keep their contents.  max_ctas > 0 caps the persistent grid for this call
 * (0: one CTA per SM).  Rejected before any launch: a geometry without a tensor-core plan, an even Conv1d K,
 * (K-1)/2*dil > 64, batch outside 1..32, L_i > L. */
int xtts_debug_conv_tc(xtts_engine* e, int32_t up, int32_t Cin, int32_t Cout, int32_t K, int32_t dil, int32_t batch, int32_t L,
                       const int32_t* item_len, const float* w, const float* bias, const float* cbias, int32_t cbias_stride,
                       const float* x, const float* resid, int32_t mode, float slope_out, float scale16, int32_t max_ctas,
                       float* out32, float* out16);
/* one ResBlock1 of the fast-mode vocoder on caller data: for t = 0..2 x <- x + c2_t(lrelu(c1_t(
 * lrelu(x), dil[t]))) with c2_t of dilation 1, then zs = x (mode 0) or zs + x (mode 1), and (pa != NULL) pa = fp16(lrelu(
 * zs * scale16, 0.1)) as atoms.  fused 1: one resblock_tc launch; 0: the six tensor-core Conv1d launches it replaces.  Both
 * give the same bits.  w [6][C][C][K] and bias [6][C] in the order c1_0, c2_0, c1_1, c2_1, c1_2, c2_2; x [batch][C][L]
 * with L % 4 == 0 and item_len (NULL = all L) as in xtts_debug_conv_tc; zs [batch][C][L] and pa [batch][C/8][lpad(L)][8]
 * are in/out as there.  max_ctas > 0 caps the persistent grid.  Rejected before any launch: an even K, a dilation < 1,
 * fused with C other than 32 / 64 or a halo (K-1)/2*(dil[0]+dil[1]+dil[2]+3) that is not a multiple of 4 or too wide
 * for the fused tile, six launches with a C that has no tensor-core
 * plan, batch outside 1..32, L_i > L. */
int xtts_debug_resblock_tc(xtts_engine* e, int32_t C, int32_t K, const int32_t* dil, int32_t batch, int32_t L,
                           const int32_t* item_len, const float* w, const float* bias, const float* x, int32_t mode,
                           float scale16, int32_t max_ctas, int32_t fused, float* zs, float* pa);
/* one speaker-conditioning kernel (csrc/cond.cu) on caller data, launched with the grid, block size and shared memory
 * xtts_condition uses.  dims [n_dims] and scal [n_scal] are the op's parameters; in [n_in] its fp32 inputs of in_len[i]
 * floats each; out [out_len] is in/out: uploaded before the launch (the base of the in-place ops, and what an element the
 * kernel does not write comes back as) and downloaded after it.  The device copy of out has 256 sentinel words on each
 * side; a kernel that writes one of them is an error.  Rejected before any launch: an unknown op, a wrong n_dims / n_scal
 * / n_in, a dim out of range, any in_len or out_len other than the one the dims imply, a NULL pointer.  Layouts are
 * row-major; per op, "dims; scal; inputs -> out":
 *   FRAME_WINDOW   n, wlen, hop, off, pad, pad_mode (0 reflect, 1 zero), frames, threads (128 or 256); -; x [n], win [wlen]
 *                  -> F [frames][wlen], F[t][i] = win[i] * xp[t*hop + off + i], xp = x padded by `pad` on each side
 *                  (reflect; or zero with NaN / inf samples read as 0)
 *   POWER          frames, nb; -; D [frames][2*nb] (re | im) -> P [frames][nb] = re^2 + im^2
 *   MEL_LOG        n, C, mode; -; mode 0: stats [C], mode 1: none -> out [n] in place: mode 0 log(max(v, 1e-5)) / stats[i % C],
 *                  mode 1 log(v + 1e-6)
 *   PREEMPHASIS    n (>= 2); coef; x [n] -> y [n] = x[i] - coef * x[i-1], x[-1] = x[1]
 *   INSTNORM_T     T, C; eps; x [T][C] -> y [C][T], each channel normalised over time (biased variance)
 *   GROUPNORM      T, C, groups (C % groups == 0); eps; x [T][C], w [C], b [C] -> y [T][C]
 *   GEGLU          rows, F; -; h [rows][2F] -> y [rows][F] = h[:, :F] * gelu_erf(h[:, F:])
 *   RMSNORM_ACCUM  rows, C; scale; x [rows][C], gamma [C] -> acc [rows][C] in place:
 *                  acc += x / max(|x|, 1e-12) * sqrt(C) * gamma * scale
 *   CONV2D         Cin, Cout, Hin, Win, k (odd), stride, relu_before_bn, has_bias, has_bn; -; x [Cin][Hin][Win],
 *                  w [Cout][Cin][k][k], then bias [Cout] if has_bias, then bn_scale [Cout], bn_shift [Cout] if has_bn
 *                  -> y [Cout][Hout][Wout], padding k/2, Hout = (Hin - 1) / stride + 1 (Wout alike);
 *                  y = bn(relu?(conv + bias)).  Rejected too: a weight slice 4 * Cin * k * k floats above 48 KB
 *   CHANNEL_MEAN   C, HW; -; x [C][HW] -> m [C]
 *   SE_GATE        C, R; -; m [C], w1 [R][C], b1 [R], w2 [C][R], b2 [C] -> s [C] = sigmoid(w2 relu(w1 m + b1) + b2)
 *   SE_APPLY       C, HW; -; x [C][HW], gate [C], resid [C][HW] -> y [C][HW] = relu(x * gate + resid)
 *   TRANSPOSE      R, Cc; -; x [R][Cc] -> y [Cc][R]
 *   RELU_BN_ROWS   rows, C; -; scale [C], shift [C] -> x [rows][C] in place: relu(x) * scale + shift
 *   ASP            T, C; -; logits [T][C], x [C][T] -> [2][C]: mu = sum softmax_t * x, sqrt(max(sum softmax_t * x^2 - mu^2, 1e-5))
 *   L2NORM         n; -; none -> x [n] in place: x / max(|x|, 1e-12)
 *   GEMV           rows, cols, has_bias; -; W [rows][cols], g [cols], then b [rows] if has_bias -> y [rows] = W g + b
 *   MEL22          n (>= 2); -; wav [n] at 22.05 kHz -> [1 + n/256][n_mels]: the engine's Hann window, DFT basis, power,
 *                  slaney mel filterbank, log(max(., 1e-5)) / mel_stats (the GPT conditioning front-end)
 *   MEL16          n (>= 400); -; wav [n] at 16 kHz -> [spk_mels][1 + n/160]: pre-emphasis 0.97, the engine's Hamming window,
 *                  DFT basis, power, mel filterbank, log(. + 1e-6), InstanceNorm over time (the speaker encoder front-end)
 * MEL22 / MEL16 need a checkpoint with the conditioning weights. */
#define XTTS_COND_FRAME_WINDOW 0
#define XTTS_COND_POWER 1
#define XTTS_COND_MEL_LOG 2
#define XTTS_COND_PREEMPHASIS 3
#define XTTS_COND_INSTNORM_T 4
#define XTTS_COND_GROUPNORM 5
#define XTTS_COND_GEGLU 6
#define XTTS_COND_RMSNORM_ACCUM 7
#define XTTS_COND_CONV2D 8
#define XTTS_COND_CHANNEL_MEAN 9
#define XTTS_COND_SE_GATE 10
#define XTTS_COND_SE_APPLY 11
#define XTTS_COND_TRANSPOSE 12
#define XTTS_COND_RELU_BN_ROWS 13
#define XTTS_COND_ASP 14
#define XTTS_COND_L2NORM 15
#define XTTS_COND_GEMV 16
#define XTTS_COND_MEL22 17
#define XTTS_COND_MEL16 18
#define XTTS_COND_N_OPS 19
int xtts_debug_cond(xtts_engine* e, int32_t op, const int32_t* dims, int32_t n_dims, const float* scal, int32_t n_scal,
                    const float* const* in, const int64_t* in_len, int32_t n_in, float* out, int64_t out_len);

#ifdef __cplusplus
}
#endif
#endif
