// Host-side launchers of every sm_90a kernel in the library (one declaration per kernel family).
// Each launcher enqueues on `st` and returns; errors surface as xtts::CudaError.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "kv_fp8.cuh"

namespace xtts {

// ------------------------------------------------------------------------------------------
// GEMM:  out[M,N] = epi(A[M,K] . W[N,K]^T + bias[N])      (W is [out,in] = K contiguous)
//   flags: GEMM_GELU  -> gelu_new after bias
//          GEMM_RESID -> out = resid + (...)   (resid may alias out)
// ------------------------------------------------------------------------------------------
// GEMM_OUT_BF16: 16-bit output in the operand format;  GEMM_F16: the 16-bit operands (and that output) are IEEE fp16, not bf16
enum : int { GEMM_GELU = 1, GEMM_RESID = 2, GEMM_OUT_BF16 = 4, GEMM_F16 = 8 };

// fp32 CUDA-core path (parity mode; also the GPU-side reference for the tensor-core path)
void launch_gemm_f32(const float* A, const float* W, const float* bias, const float* resid, float* out,
                     int M, int N, int K, int flags, cudaStream_t st);

// bf16 wgmma/TMA path (fast mode).  A [M,K] bf16 row-major, W [N,K] bf16 row-major; fp32 accumulators in registers.
// out is fp32 unless GEMM_OUT_BF16.  K % 64 == 0, N % 32 == 0 required.
// `pdl`: launch with the programmatic-dependent-launch attribute (decode chain); every kernel that can be launched
// that way executes griddepcontrol.wait before touching its predecessor's outputs
void launch_gemm_bf16_tc(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, const float* resid,
                         void* out, int M, int N, int K, int flags, cudaStream_t st, bool pdl = false);
// large-shape path (gemm_wgmma_wide.cu): persistent CTAs, 128 x 256 tiles
bool gemm_wide_supported(int M, int N, int K);
void launch_gemm_bf16_wide(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, const float* resid,
                           void* out, int M, int N, int K, int flags, cudaStream_t st);
void launch_gemm_bf16_tc_splitk(const __nv_bfloat16* A, const __nv_bfloat16* W, float* partials, int M, int N, int K,
                                int splits, cudaStream_t st, bool pdl = false, int flags = 0);

bool gemm_tc_init(std::string* err);   // resolves cuTensorMapEncodeTiled; false -> err filled
// TMA descriptor of a row-major 16-bit matrix [rows, cols]: boxes of 64 columns (128 B, SWIZZLE_128B) x box_rows rows, the
// operand image the wgmma kernels read (gemm_wgmma.cu, gemm_wgmma_wide.cu); rows past the end are zero-filled
void tma_encode_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows);

void trace_set_gemm(TraceBuf b);     // per-translation-unit setters of the debug timeline buffer (common.cuh)
void trace_set_gpt(TraceBuf b);
void trace_set_conv(TraceBuf b);

void launch_f32_to_bf16(const float* in, __nv_bfloat16* out, size_t n, cudaStream_t st);
void launch_f32_to_f16(const float* in, __half* out, size_t n, cudaStream_t st);

// ------------------------------------------------------------------------------------------
// GPT glue kernels
// ------------------------------------------------------------------------------------------
struct RowDesc {          // one prompt / teacher-forced input row
    int kind;             // 0: cond row `a` of speaker slot `c`; 1: text id `a` at text position `b`;
                          // 2: audio token `a` at audio position `b`
    int a, b, c;
};

struct GptTables {        // embedding tables (device, fp32)
    const float* text_emb;  // [n_text, H]
    const float* text_pos;  // [n_text_pos, H]
    const float* wte;       // [n_audio, H]
    const float* wpe;       // [n_wpe, H]
    const float* spk_cond;  // [n_speaker_slots, n_cond, H]
    int H, n_cond;
};

void launch_build_rows(const RowDesc* rows, int n_rows, GptTables t, float* X, cudaStream_t st);
// decode input rows: X[i] = wte[last_tok[slot]] + wpe[n_gen[slot]],  slot = active[i]
void launch_build_decode_rows(const int* active, int M, const int* last_tok, const int* n_gen, GptTables t,
                              float* X, cudaStream_t st, bool pdl = false);

template <typename TOut>
void launch_layernorm(const float* X, const float* w, const float* b, TOut* Y, int M, int H, float eps,
                      cudaStream_t st, bool pdl = false);

// X[m] += bias + sum_z partials[z][m]  (deterministic split-K reduction fused with the residual add), then
// Y[m] = LN(X[m]) when Y != nullptr  (the following block's LayerNorm)
template <typename TOut>
void launch_residual_reduce_layernorm(float* X, const float* partials, int splits, const float* bias, const float* w,
                                      const float* b, TOut* Y, int M, int H, float eps, cudaStream_t st, bool pdl = false);

// y = LN_fn(LN_lnf(X[row_index[i]]));  Y[i] = y (GEMM operand);
// latents[slots[i]][lat_pos ? lat_pos[i] : n_gen[slots[i]]] = LN_fn(y)
template <typename TOut>
void launch_head_norms(const float* X, const int* row_index, const float* lnf_w, const float* lnf_b,
                       const float* fn_w, const float* fn_b, TOut* Y, float* latents, const int* slots,
                       const int* lat_pos, const int* n_gen, int lat_rows_per_slot, int M, int H, float eps,
                       cudaStream_t st, bool pdl = false);

// KV page layout (per layer):  K: [page][head][D/X][32 tok][X]   V: [page][head][32 tok][D]
//   X = 16 bytes / sizeof(TKV)  (so one lane = one token reads 16 B, coalesced across the warp)
//   TKV = __nv_fp8_e4m3: the same per token, each (page, head) block followed by 32 exponent bytes (kv_fp8.cuh)
template <typename TKV>
void launch_kv_write(const float* QKV, int M, const int* row_slot, const int* row_pos, const int* ctx_len,
                     const int* block_tables, int max_pages, TKV* kpool, TKV* vpool, int heads,
                     cudaStream_t st);

// decode attention over the paged cache, ctx = ctx_len[slot] + 1.  The kernel also appends the new token's K/V
// (read from the QKV row) to the cache — the reshape_and_cache step — so no separate kv_write launch is needed.
// TKV: float / bf16 / fp16 with TOut = TKV, or __nv_fp8_e4m3 with TOut bf16 / fp16.
template <typename TKV, typename TOut>
void launch_attn_decode(const float* QKV, const int* active, int M, const int* ctx_len,
                        const int* block_tables, int max_pages, TKV* kpool, TKV* vpool,
                        TOut* out, int heads, cudaStream_t st, double ctx_sum_hint = 0, bool pdl = false);

struct AttnSeq { int q_start, nq, kv_start, nk; };
struct AttnLayout {
    const float* q; const float* k; const float* v;   // base pointers
    int q_row_stride, kv_row_stride;                   // elements between consecutive rows
    int q_head_stride, kv_head_stride;                 // elements between heads inside a row
    int heads;
    float scale;
    int causal;                                        // key j visible to query i iff j <= i + (nk - nq)
};
// generic fp32 attention (GPT prefill, conditioning encoder, perceiver); head_dim 64
template <typename TOut>
void launch_attn_generic(AttnLayout L, const AttnSeq* seqs, int nseq, int max_nq, TOut* out, int out_row_stride,
                         cudaStream_t st);

struct SampleState {      // per-slot arrays (device)
    int* last_tok; int* n_gen; int* ctx_len; int* finished;
    int* tokens;          // [slot][max_tokens_cap] chosen tokens
    int* sampled;         // [slot][max_tokens_cap] what the sampler drew (== tokens unless forced)
    const int* forced;    // [slot][max_tokens_cap] or nullptr; entry < 0 = not forced
    unsigned* seen;       // [slot][seen_words] bitmap of ids in prompt ∪ generated
    const float* temperature; const float* top_p; const int* top_k; const float* penalty;
    const int* max_tokens; const int* stop_token; const unsigned long long* seed; const int* seq_seed;
    const int* beam;      // [slot] != 0: the slot is a beam of a beam-search group, chosen by the beam kernels (or nullptr)
    int tokens_cap, seen_words;
};
void launch_sample(const float* logits, int ld_logits, const int* active, int M, int V, SampleState s,
                   int advance_ctx, cudaStream_t st, bool pdl = false);

// ------------------------------------------------------------------------------------------
// beam search (beam.cu): transformers 5.5 `_beam_search` for one batch item per group, num_return_sequences 1,
// early_stopping unset.  A group of nb <= 8 beams lives in nb slots; beam j is slot[j] for the group's whole life.
// ------------------------------------------------------------------------------------------
constexpr int kMaxBeams = 8;
struct BeamDesc {         // one running group, uploaded every step
    int primary;          // slot of beam 0: indexes the group's persistent state
    int nb;
    int slot[kMaxBeams];
    int row[kMaxBeams];   // logits row of each beam this step (all = the prefill row on the first step)
    int first;            // first selection: B copies of the prefill logits, running scores [0, -1e9, ...]
    int advance;          // KV positions appended by the step just run (0 after the prefill, 1 after a decode step)
    int do_sample;
    float length_penalty;
};
struct BeamState {        // persistent per group, indexed by the primary slot
    float run_score[kMaxBeams];
    float fin_score[kMaxBeams];
    int fin_valid[kMaxBeams];                    // is_sent_finished
    int fin_step[kMaxBeams], fin_beam[kMaxBeams], fin_tok[kMaxBeams];
    int heur_unsat;                              // is_early_stop_heuristic_unsatisfied
    int done;
    int sel_parent[kMaxBeams], sel_tok[kMaxBeams];   // this step's running beams: parent beam, token
    int n_copy;                                  // partial pages to copy this step
    int copy_src[kMaxBeams], copy_dst[kMaxBeams], copy_ntok[kMaxBeams];
    int n_free;                                  // pages in the group's free list
    int n_pages[kMaxBeams];                      // table entries of each beam
};
struct BeamArgs {
    const BeamDesc* desc; int n_groups;
    BeamState* state;     // [NSLOT]
    int2* hist;           // [NSLOT][tokens_cap][kMaxBeams]: (parent beam, token) of each running beam, per step
    int* pool;            // [NSLOT][pool_cap] free pages of each group
    int pool_cap;
    float* scores;        // [NSLOT][ld] processed, accumulated scores of each beam slot
    int* block_tables; int max_pages;
    float* latents; int H;                       // latent ring [NSLOT][tokens_cap][H]
};
// logprob -> select -> reorder (block tables, slot state) -> partial-page copy -> gather of finished groups (`gather`)
// kpool / vpool: device arrays of the `layers` per-layer pool base pointers; elem = bytes per KV element (1: the fp8
// format, whose copied tokens take their exponent bytes along)
void launch_beam_step(const float* logits, int ld_logits, int V, SampleState s, BeamArgs a, void* const* kpool,
                      void* const* vpool, int layers, int heads, int elem, cudaStream_t st, bool gather = true);
// the geometry the beam kernels take: V <= 2048, <= 128 KV pages per sequence, the gather's token list in shared memory
bool beam_supported(int V, int max_pages, int tokens_cap);
// per device (the current one): the beam kernels' dynamic shared memory limits
void beam_init_device();

// ------------------------------------------------------------------------------------------
// Vocoder kernels (fp32, channel-major activations [C][L])
// ------------------------------------------------------------------------------------------
// every vocoder launcher takes `batch` items laid out back to back ([batch][C][L]); the tensor-core path also takes
// ragged batches: `item_len[i] <= L` valid time steps per item (host array; nullptr = all L), buffers strided by L
constexpr int kVocMaxItems = 32;
// One item of an interpolation launch: z-frames [z0, z0 + nz) of a chunk whose latents start at `lat` ([T][C] fp32, device).
// T / T1 are the clamp lengths of the two linear interpolations (HifiDecoder.forward): the chunk's real length once it is
// known, otherwise any length the window does not reach (a window of a still-growing chunk never touches the clamp).
// r0 > 0: the chunk has a speaking rate (Xtts.inference's speed): the latents are first time-scaled by one more linear
// interpolation to T0 = floor(T * ls) frames, ls = 1 / (double)speed, source index r0 * (j + .5) - .5 with r0 = (float)(1 / ls)
// (torch's rule for F.interpolate(scale_factor=ls)); T1 is then the clamp length of the next level on those T0 frames.
// r0 == 0: no such stage (speed 1), the two-level code.
struct InterpItem { const float* lat; int T, T1, z0, nz; int T0 = 0; float r0 = 0.f; };
// z32 (fp32 [batch][C][Lz]) and/or z16 (fp16 atoms [batch][C/8][lpad][8]) — either may be null; Lz = row stride >= max nz
void launch_interp(const InterpItem* items, int batch, float* z32, __half* z16, int lpad, int C, int Lz, double scale1,
                   double scale2, cudaStream_t st);

// the scale factors of the two interpolations (HifiDecoder.forward): code_stride / hop, then out_sr / in_sr (1: no resampling)
inline double interp_scale1(int code_stride, int hop) { return (double)code_stride / (double)hop; }
inline double interp_scale2(int in_sr, int out_sr) { return in_sr != out_sr ? (double)out_sr / (double)in_sr : 1.0; }

enum : int { CONV_STORE = 0, CONV_ACCUM = 1 };
// Conv1d weight [Cout][Cin][K] (transposed = false) or ConvTranspose1d weight [Cin][Cout][K] (true), torch's layouts ->
// w_t [Cin][K][Cout], the layout launch_conv1d and launch_conv_transpose1d read
void conv_weight_ckc(const float* w, int Cin, int Cout, int K, bool transposed, float* w_t);
// out[co][t] (=|+=) bias[co] + cbias[co] + resid[co][t] + sum_{ci,j} w[ci][j][co] * act(in_scale*x[ci][t+(j-(K-1)/2)*dil])
//   act = leaky_relu(slope) (slope==1 -> identity).  w is pre-transposed to [Cin][K][Cout].
void launch_conv1d(const float* x, const float* w_t, const float* bias, const float* cbias, const float* resid,
                   float* out, int Cin, int Cout, int L, int K, int dil, float in_scale, float slope, int mode,
                   int batch, int cbias_batch_stride, cudaStream_t st);
// ---- tensor-core vocoder path (fast mode).  Activations that feed a Conv1d live in HBM as fp16 "atoms":
//   [C/8 plane][kAtomPadL + L + tail][8 channels], zero pads — the wgmma no-swizzle K-major operand image.
constexpr int kAtomPadL = 64, kAtomPadR = 64;
int atoms_lpad(int L);                                   // padded rows per plane for a signal of L steps
// dynamic shared memory a tensor-core conv kernel may take: the opt-in limit minus the kernels' static shared memory
constexpr int kMaxDynTc = 227 * 1024 - 4096;
struct ConvTcPlan { int N, CK, n_tiles, nacc; bool ok; size_t tile_halves, blob_halves; };
ConvTcPlan conv1d_tc_plan(int Cin, int Cout, int K);
void conv1d_tc_pack(const float* w /*[Cout][Cin][K]*/, int Cin, int Cout, int K, const ConvTcPlan& pl, __half* blob);
// dynamic shared memory of a launch: `direct` epilogue; `staged` epilogue (0 = does not fit / transposed conv) with its
// slab ring at `epi_off`, slabs of `slab_cols` GEMM columns x tile rows, `slab_bytes` each; nf = fp32 buffers per slab
struct ConvTcSmem { size_t direct, staged, epi_off, slab_bytes; int slab_cols; };
ConvTcSmem conv1d_tc_smem(const ConvTcPlan& pl, int K, int dil, int up, int nf);
// y = bias + cbias + resid + conv(a16);  out32 (fp32 [C][L], store/accumulate) and/or out16 (lrelu(y, slope_out) atoms)
// out16 = lrelu(y * scale16, slope_out)
// (engine knobs of the launchers — attention grid cap, decode GEMM tile, vocoder SM cap — live in
//  the calling engine's KernelCtx, common.cuh)
void launch_conv1d_tc(const __half* a16, const __half* wblob, const ConvTcPlan& pl, const float* bias, const float* cbias,
                      const float* resid, float* out32, __half* out16, int Cin, int Cout, int L, int lpad, int K, int dil,
                      float slope_out, float scale16, int mode, int batch, int cbias_batch_stride, cudaStream_t st,
                      const int* item_len = nullptr);
// One whole ResBlock1 (for t = 0..2: x += c2_t(lrelu(c1_t(lrelu(x), dil[t])), 1); then zs (=|+=) x) as one launch, bit-identical
// to its six launch_conv1d_tc calls.  xa: lrelu(x) atoms, x: fp32 [batch][C][L] (L % 4 == 0); wblob / bias: the six convs
// c1_0, c2_0, c1_1, c2_1, c1_2, c2_2 (conv1d_tc_pack blobs); pa (optional): lrelu(sum * scale16, 0.1) atoms.
// resblock_tc_tile_rows: output rows per CTA tile, 0 when the fused kernel does not take this geometry (C must be 32 or 64,
// the chain's halo (K-1)/2 * (dil[0] + dil[1] + dil[2] + 3) and the row stride L multiples of 4).
int resblock_tc_tile_rows(int C, int K, const int* dil, int L);
void launch_resblock_tc(const __half* xa, const float* x, const __half* const* wblob, const float* const* bias, float* zs,
                        __half* pa, int C, int L, int lpad, int K, const int* dil, int mode, float scale16, int batch,
                        const int* item_len, cudaStream_t st);
// ConvTranspose1d(kernel 2u, stride u, padding u/2) on the same kernel (u phases x 2 taps); plan = conv1d_tc_plan(Cin, u*Cr, 2)
void convT_tc_pack(const float* w /*[Cin][Cr][2u]*/, int Cin, int Cr, int u, const ConvTcPlan& pl, __half* blob);
void launch_convT_tc(const __half* a16, const __half* wblob, const ConvTcPlan& pl, const float* bias, const float* cbias,
                     float* out32, __half* out16, int Cin, int Cr, int Lin, int lpad_in, int lpad_out, int u, float slope_out,
                     int batch, int cbias_batch_stride, cudaStream_t st, const int* item_len = nullptr);
// planes_total = batch * planes per item; item_len (host, optional): per-item signal length
void launch_atoms_zero_pads(__half* buf, int planes_total, int lpad, int L, cudaStream_t st, int batch = 1,
                            const int* item_len = nullptr);
// transposed conv, stride u, kernel K = 2u, padding (K-u)/2;  w pre-transposed to [Cin][K][Cout]
void launch_conv_transpose1d(const float* x, const float* w_t, const float* bias, const float* cbias, float* out, int Cin,
                             int Cout, int Lin, int K, int u, float in_scale, float slope, int batch, int cbias_batch_stride,
                             cudaStream_t st);
// wav[t] = tanh(sum w[ci][j] * lrelu(in_scale*x[ci][t+j-3], slope));  x [batch][Cin][L], wav [batch][wav_stride (0 = L)];
// item_len as above
void launch_conv_post(const float* x, const float* w, float* wav, int Cin, int L, int K, float in_scale, float slope,
                      int batch, cudaStream_t st, const int* item_len = nullptr, int wav_stride = 0);

// ------------------------------------------------------------------------------------------
// slot bookkeeping
// ------------------------------------------------------------------------------------------
// Everything a freshly admitted sequence needs in its slot, written by ONE kernel from one staged upload (instead of a
// dozen small copies per sequence).
struct SlotInit {
    int slot, ctx_len, top_k, max_tokens, stop_token, seq_seed, start_token, n_pages;
    int beam;             // the slot is a beam of a beam-search group (SampleState::beam)
    float temperature, top_p, penalty;
    unsigned long long seed;
};
struct SlotArrays {       // per-slot device arrays (mutable view of SampleState + block tables)
    int* last_tok; int* n_gen; int* ctx_len; int* finished; unsigned* seen;
    float* temperature; float* top_p; int* top_k; float* penalty; int* max_tokens; int* stop_token;
    unsigned long long* seed; int* seq_seed; int* block_tables; int* beam;
    int seen_words, max_pages;
};
// pages: [n][max_pages] page ids of each sequence (first n_pages valid)
void launch_init_slots(const SlotInit* init, const int* pages, int n, SlotArrays a, cudaStream_t st);
// dst[i][0..width) = src[idx[i]][0..width)   (i < n <= kVocMaxItems): speaker-bias rows of a vocoder batch
void launch_gather_rows(const float* src, const int* idx_host, int n, int width, float* dst, cudaStream_t st);
// y[c] = W[c,:] . g + b[c]   (speaker conditioning 1x1 convs)
void launch_gemv(const float* W, const float* b, const float* g, float* y, int rows, int cols, cudaStream_t st);

}  // namespace xtts
