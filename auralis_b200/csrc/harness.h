// Kernel isolation harness behind the xtts_debug_* entry points (include/xtts_b200.h): each function runs one
// kernel's launcher (or one short chain of them) on private device buffers built from host arrays, validates its
// arguments before any launch, and copies every output back.  The engine calls them through Engine::run_idle, which
// holds its API lock, requires it to be idle and binds its launcher options (KernelCtx).
#pragma once
#include "../../include/xtts_b200.h"
#include "common.cuh"

namespace xtts {

class Conditioner;

// What the harness takes from the engine: its stream, LayerNorm epsilon, PDL option and conditioner (NULL when the
// checkpoint has no conditioning weights).
struct HarnessCtx { cudaStream_t st; float ln_eps; bool pdl; Conditioner* cnd; };

void debug_gemm(const HarnessCtx& c, int mode, const float* A, const float* W, const float* bias, const float* resid,
                float* out, int M, int N, int K, int dflags, int iters, float* ms);
void debug_ln_gemm(const HarnessCtx& c, int mode, int launch, int M, int N, int K, const float* X, const float* ln_w,
                   const float* ln_b, const float* W, const float* bias, const float* resid, int dflags, float* Y, float* out);
void debug_norms(const HarnessCtx& c, int out_type, int M, int H, const float* X, int x_rows, const int32_t* row_index,
                 const float* w1, const float* b1, const float* w2, const float* b2, float* Y, float* latents, int n_slots,
                 int lat_rows, const int32_t* slots, const int32_t* lat_pos, const int32_t* n_gen);
void debug_kv_write(const HarnessCtx& c, int kv_type, int heads, int M, const float* qkv, const int32_t* row_slot,
                    const int32_t* row_pos, int n_slots, const int32_t* ctx_len, const int32_t* block_tables, int max_pages,
                    int n_pages, void* kpool, void* vpool);
void debug_build_rows(const HarnessCtx& c, int H, int n_cond, const float* text_emb, int n_text, const float* text_pos,
                      int n_tpos, const float* wte, int n_audio, const float* wpe, int n_wpe, const float* spk, int n_spk,
                      const int32_t* rows, int n_rows, float* X);
void debug_build_decode_rows(const HarnessCtx& c, int H, const float* wte, int n_audio, const float* wpe, int n_wpe, int M,
                             const int32_t* active, int n_slots, const int32_t* last_tok, const int32_t* n_gen, float* X);
void debug_sample_slots(const HarnessCtx& c, int V, int M, const int32_t* active, int n_slots, const float* logits, int ld,
                        const xtts_sampling* sp, int cap, int advance_ctx, const int32_t* forced, int32_t* n_gen,
                        int32_t* ctx_len, int32_t* finished, int32_t* last_tok, uint8_t* seen, int32_t* tokens,
                        int32_t* sampled);
void debug_attn_decode(const HarnessCtx& c, int kv_type, int heads, int M, const int32_t* active, int n_slots,
                       const int32_t* ctx_len, const int32_t* block_tables, int max_pages, int n_pages, void* kpool,
                       void* vpool, const float* qkv, float* out);
void debug_attn_prefill(const HarnessCtx& c, int out_type, int heads, const int32_t* seqs, int nseq, int causal, float scale,
                        const float* q, int64_t q_len, int q_row_stride, int q_head_stride, const float* kv, int64_t kv_len,
                        int kv_row_stride, int kv_head_stride, int64_t k_off, int64_t v_off, float* out, int out_rows);
void debug_splitk_ln(const HarnessCtx& c, int mode, int M, int N, int K, int splits, const float* A, const float* W,
                     const float* bias, float* X, const float* ln_w, const float* ln_b, float* Y);
void debug_conv_tc(const HarnessCtx& c, int up, int Cin, int Cout, int K, int dil, int batch, int L, const int32_t* item_len,
                   const float* w, const float* bias, const float* cbias, int cbias_stride, const float* x, const float* resid,
                   int mode, float slope_out, float scale16, int max_ctas, float* out32, float* out16);
void debug_resblock_tc(const HarnessCtx& c, int C, int K, const int32_t* dil, int batch, int L, const int32_t* item_len,
                       const float* w, const float* bias, const float* x, int mode, float scale16, int max_ctas, int fused,
                       float* zs, float* pa);
void debug_vocoder(const HarnessCtx& c, int op, const int32_t* dims, int n_dims, const float* scal, int n_scal,
                   const float* const* in, const int64_t* in_len, int n_in, float* out, int64_t out_len);
void debug_beam_step(const HarnessCtx& c, int kv_type, int heads, int layers, int V, const xtts_sampling& sp,
                     const xtts_beam& bm, int first, int advance, const float* logits, int32_t* n_gen, int32_t* ctx_len,
                     int32_t* last_tok, uint32_t* seen, int max_pages, int32_t* block_tables, int n_pages, int32_t* pool,
                     int cap, int32_t* hist, xtts_beam_state* state, void* kpool, void* vpool, float* scores);

}  // namespace xtts
