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

/* llm_engine.generate(...) per text chunk (XTTSv2.py:741-757): text_ids = [bos]+bpe+[eos] (XTTSv2.py:519-522).
 * Asynchronous: the scheduler thread admits, prefills, decodes (continuous batching), vocodes. */
int xtts_submit(xtts_engine* e, uint64_t seq_id, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                const xtts_sampling* sp);
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
 *   "decode_chain"        1 = fused persistent per-layer GEMM/LayerNorm chain kernel in the decode step, 0 = one launch per
 *                         GEMM / LayerNorm with "microbatches" concurrent row branches (default: measured faster)
 *   "microbatches"        1..4 concurrent branches the decode step's rows are split into (default 2)
 *   "microbatch_min_rows" steps with fewer active rows stay single-branch (default 48)
 *   "gemm_wide"           4 (default), 3 or 2 = GEMMs with M >= 256 rows (prefill, conditioning) run on the persistent
 *                         wide-tile kernel (128x256 tiles) with that ring depth, 0 = the one-tile-per-CTA kernel
 *   "voc_segment"         m > 0: a chunk is vocoded in windows of m tokens WHILE it decodes (the vocoder runs on its own
 *                         stream beside the decode step), 0 = one window per chunk when it ends.  Same samples either way.
 *   "voc_sms"             SMs the vocoder's persistent conv kernels may occupy while a decode step is in flight (0 = all)
 *   "voc_batch"           windows per vocoder launch (1..32, default 32; ragged lengths are batched together)
 *   "attn_warps"          warps per (row, head) item of the 16-bit decode attention: 4 (default), 1 / 2 / 8 / 16 measured slower
 *   "attn_ctas_per_sm"    > 0 caps the decode-attention grid (each CTA walks several items); < 0: absolute grid size (tests)
 *   "attn_l2_pages"       n > 0: each warp of the decode attention asks L2 for n of its later pages per item
 *                         (cp.async.bulk.prefetch.L2); default 0 (measured slower: the kernel is throughput-, not latency-bound)
 *   "attn_bulk"           c > 0: decode attention in bulk-copy form (c persistent CTAs per SM stream cache pages with
 *                         cp.async.bulk into "attn_stages" x 8 KB of shared-memory sub-rings, "attn_l2_ahead" = L2 prefetch
 *                         one item ahead); bit-identical to the default register-load kernel, measured slower; default 0
 *   "gemm_deep_ring"      1 = unsplit decode GEMMs use a ring that fills the SM (one CTA per SM); default 0 (measured slower)
 *   "gemm_l2_prefetch"    1 = decode GEMMs prefetch the weight tiles of their later ring passes into L2 before the
 *                         dependency wait; default 0 (no measurable effect)
 *   "dep_flags" / "branch_stagger_us"   counter dependencies / delayed second branch in the decode step (default off)
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
/* one prefill over [prompt ; forced audio tokens] (the reference's 2nd pass, XTTSv2.py:617-687):
 * outputs ln_f hidden of every row, raw logits + latents of the last n_audio rows */
int xtts_gpt_prefill(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                     const int32_t* audio_tokens, int32_t n_audio, float* hidden_out, float* logits_out,
                     float* latents_out);
/* prefill + step-by-step decode with forced tokens: raw logits [n,V], latents [n,H], sampled ids [n] */
int xtts_gpt_teacher_forced(xtts_engine* e, const int32_t* text_ids, int32_t n_text, int32_t speaker_slot,
                            const int32_t* forced_tokens, int32_t n, const xtts_sampling* sp, float* logits_out,
                            float* latents_out, int32_t* sampled_out);
/* GEMM under test: mode 0 = fp32 CUDA-core, 1 = bf16 wgmma, 2 = fp16 wgmma.  A [M,K], W [N,K], bias [N] or NULL, resid [M,N] or NULL */
int xtts_debug_gemm(xtts_engine* e, int32_t mode, const float* A, const float* W, const float* bias, const float* resid,
                    float* out, int32_t M, int32_t N, int32_t K, int32_t gelu, int32_t iters, float* ms_per_iter);
/* debug timeline: op 1 arms %globaltimer stamps in the decode / vocoder kernels (first and last CTA: entry, dependency
 * resolved, exit), op 0 disarms and copies up to `cap` records [n][2] u64 = (ns, id<<32 | grid<<40 | last<<8 | phase) into
 * `out`; returns the count (>= 0) or a negative error.  Nothing is serialised: shows the step as it really runs. */
int xtts_debug_trace(xtts_engine* e, int32_t op, uint64_t* out, int32_t cap);
/* sampler under test: logits [B,V]; seen [B,V] (0/1) ; out tokens [B] */
int xtts_debug_sample(xtts_engine* e, const float* logits, const uint8_t* seen, int32_t B, int32_t V,
                      const xtts_sampling* sp, int32_t step, int32_t* out_tokens);

#ifdef __cplusplus
}
#endif
#endif
