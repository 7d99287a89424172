// GPT-2 acoustic-model kernels other than the GEMMs: embedding/prompt assembly, LayerNorm, the
// head norm chain, paged-KV write, prefill (generic) attention, paged decode attention and the fused
// penalty/temperature/top-k/top-p/sample kernel.
//
// Reference call sites these replace (SURVEY.md §2.4 / §8a):
//   K1,K2  vllm_mm_gpt.py:768-785,800-833 (wte+wpe gather, conditioning splice)      -> build_rows*
//   K3,K8  GPT2Block ln_1/ln_2, ln_f :762,848, final_norm :671, XTTSv2.py:687          -> layernorm, head_norms
//   K5     vLLM paged attention + reshape_and_cache (3rd party)                        -> kv_write, attn_*
//   K10    hijack.py:49-88 LogitsRepetitionPenalizer                                    -> sample (penalty)
//   K11    vLLM Sampler (SURVEY App. A.3)                                               -> sample
#include <algorithm>
#include <type_traits>
#include "kernels.h"

namespace xtts {
namespace {

// ------------------------------------------------------------------------------------------------
// prompt / input row assembly
// ------------------------------------------------------------------------------------------------
__global__ void build_rows_kernel(const RowDesc* __restrict__ rows, GptTables t, float* __restrict__ X) {
    const RowDesc d = rows[blockIdx.x];
    const int H = t.H;
    float4* x = reinterpret_cast<float4*>(X + (size_t)blockIdx.x * H);
    const float4* s1;
    const float4* s2 = nullptr;
    if (d.kind == 0) {
        s1 = reinterpret_cast<const float4*>(t.spk_cond + ((size_t)d.c * t.n_cond + d.a) * H);
    } else if (d.kind == 1) {
        s1 = reinterpret_cast<const float4*>(t.text_emb + (size_t)d.a * H);
        s2 = reinterpret_cast<const float4*>(t.text_pos + (size_t)d.b * H);
    } else {
        s1 = reinterpret_cast<const float4*>(t.wte + (size_t)d.a * H);
        s2 = reinterpret_cast<const float4*>(t.wpe + (size_t)d.b * H);
    }
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
        float4 v = s1[i];
        if (s2) { const float4 u = s2[i]; v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
        x[i] = v;
    }
}

__global__ void build_decode_rows_kernel(const int* __restrict__ active, const int* __restrict__ last_tok,
                                         const int* __restrict__ n_gen, GptTables t, float* __restrict__ X) {
    trace_pt(TR_ROWS, 0); pdl_trigger(); pdl_wait(); trace_pt(TR_ROWS, 1);
    const int slot = active[blockIdx.x];
    const int H = t.H;
    const float4* a = reinterpret_cast<const float4*>(t.wte + (size_t)last_tok[slot] * H);
    const float4* b = reinterpret_cast<const float4*>(t.wpe + (size_t)n_gen[slot] * H);
    float4* x = reinterpret_cast<float4*>(X + (size_t)blockIdx.x * H);
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
        float4 v = a[i]; const float4 u = b[i];
        v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
        x[i] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// slot initialisation of an admission wave: one CTA per admitted sequence
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
init_slots_kernel(const SlotInit* __restrict__ init, const int* __restrict__ pages, SlotArrays a) {
    const SlotInit d = init[blockIdx.x];
    const int slot = d.slot;
    if (threadIdx.x == 0) {
        a.last_tok[slot] = d.start_token; a.n_gen[slot] = 0; a.ctx_len[slot] = d.ctx_len; a.finished[slot] = 0;
        a.temperature[slot] = d.temperature; a.top_p[slot] = d.top_p; a.top_k[slot] = d.top_k; a.penalty[slot] = d.penalty;
        a.max_tokens[slot] = d.max_tokens; a.stop_token[slot] = d.stop_token; a.seed[slot] = d.seed; a.seq_seed[slot] = d.seq_seed;
        a.beam[slot] = d.beam;
    }
    // penalty set seed: the prompt ids are [1]*(32+Lt)+[start]  (vllm_mm_gpt.py:325, App. B.7)
    for (int w = threadIdx.x; w < a.seen_words; w += blockDim.x) {
        unsigned v = 0u;
        if (w == 0) v |= 1u << 1;
        if (w == (d.start_token >> 5)) v |= 1u << (d.start_token & 31);
        a.seen[(size_t)slot * a.seen_words + w] = v;
    }
    const int* pg = pages + (size_t)blockIdx.x * a.max_pages;
    for (int i = threadIdx.x; i < a.max_pages; i += blockDim.x)
        a.block_tables[(size_t)slot * a.max_pages + i] = i < d.n_pages ? pg[i] : 0;
}

struct GatherIdx { int idx[kVocMaxItems]; };
__global__ void gather_rows_kernel(const float* __restrict__ src, const GatherIdx G, int width, float* __restrict__ dst) {
    const float* s = src + (size_t)G.idx[blockIdx.x] * width;
    float* d = dst + (size_t)blockIdx.x * width;
    for (int i = threadIdx.x; i < width; i += blockDim.x) d[i] = s[i];
}

// ------------------------------------------------------------------------------------------------
// LayerNorm (fp32 statistics, two-pass), one CTA per row
// ------------------------------------------------------------------------------------------------
template <typename TOut>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ X, const float* __restrict__ w, const float* __restrict__ b,
                 TOut* __restrict__ Y, int H, float eps) {
    __shared__ float red[32];
    trace_pt(TR_LN, 0); pdl_trigger(); pdl_wait(); trace_pt(TR_LN, 1);
    const float* x = X + (size_t)blockIdx.x * H;
    float s = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) s += x[i];
    const float mean = block_sum(s, red) / (float)H;
    float v = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { const float d = x[i] - mean; v = fmaf(d, d, v); }
    const float var = block_sum(v, red) / (float)H;
    const float rstd = 1.0f / sqrtf(var + eps);
    TOut* y = Y + (size_t)blockIdx.x * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) y[i] = from_f32<TOut>((x[i] - mean) * rstd * w[i] + b[i]);
}

__device__ __forceinline__ void smem_layernorm(float* buf, const float* __restrict__ w, const float* __restrict__ b,
                                               int H, float eps, float* red) {
    float s = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) s += buf[i];
    const float mean = block_sum(s, red) / (float)H;
    float v = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { const float d = buf[i] - mean; v = fmaf(d, d, v); }
    const float var = block_sum(v, red) / (float)H;
    const float rstd = 1.0f / sqrtf(var + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) buf[i] = (buf[i] - mean) * rstd * w[i] + b[i];
    __syncthreads();
}

template <typename TOut>
__global__ void __launch_bounds__(256)
residual_reduce_ln_kernel(float* __restrict__ X, const float* __restrict__ P, int splits, size_t split_stride,
                          const float* __restrict__ bias, const float* __restrict__ w, const float* __restrict__ b,
                          TOut* __restrict__ Y, int H, float eps) {
    extern __shared__ float buf[];
    __shared__ float red[32];
    trace_pt(TR_REDUCE_LN, 0); pdl_trigger(); pdl_wait(); trace_pt(TR_REDUCE_LN, 1);
    float* x = X + (size_t)blockIdx.x * H;
    const float* p = P + (size_t)blockIdx.x * H;
    // 16-byte lanes: with H = 1024 every thread owns one float4, so the residual, the bias and all split partials of the
    // row are requested in a single round of loads (one L2 latency instead of four)
    for (int c = threadIdx.x * 4; c < H; c += blockDim.x * 4) {
        float4 pv[8];
#pragma unroll
        for (int z = 0; z < 8; ++z)
            pv[z] = (z < splits) ? *reinterpret_cast<const float4*>(p + (size_t)z * split_stride + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 xv = *reinterpret_cast<const float4*>(x + c);
        const float4 bv = *reinterpret_cast<const float4*>(bias + c);
        float4 v = make_float4(xv.x + bv.x, xv.y + bv.y, xv.z + bv.z, xv.w + bv.w);
#pragma unroll
        for (int z = 0; z < 8; ++z) { v.x += pv[z].x; v.y += pv[z].y; v.z += pv[z].z; v.w += pv[z].w; }   // fixed order: deterministic
        *reinterpret_cast<float4*>(x + c) = v;
        *reinterpret_cast<float4*>(buf + c) = v;
    }
    __syncthreads();
    if (Y == nullptr) return;
    smem_layernorm(buf, w, b, H, eps, red);
    TOut* y = Y + (size_t)blockIdx.x * H;
    for (int c = threadIdx.x; c < H; c += blockDim.x) y[c] = from_f32<TOut>(buf[c]);
    trace_pt(TR_REDUCE_LN, 2);
}

template <typename TOut>
__global__ void __launch_bounds__(256)
head_norms_kernel(const float* __restrict__ X, const int* __restrict__ row_index, const float* __restrict__ lnf_w,
                  const float* __restrict__ lnf_b, const float* __restrict__ fn_w, const float* __restrict__ fn_b,
                  TOut* __restrict__ Y, float* __restrict__ latents, const int* __restrict__ slots,
                  const int* __restrict__ lat_pos, const int* __restrict__ n_gen, int lat_rows_per_slot, int H,
                  float eps) {
    extern __shared__ float buf[];
    __shared__ float red[32];
    trace_pt(TR_HEAD, 0); pdl_trigger(); pdl_wait(); trace_pt(TR_HEAD, 1);
    const int i = blockIdx.x;
    const int r = row_index ? row_index[i] : i;
    const float* x = X + (size_t)r * H;
    for (int c = threadIdx.x; c < H; c += blockDim.x) buf[c] = x[c];
    __syncthreads();
    smem_layernorm(buf, lnf_w, lnf_b, H, eps, red);      // ln_f            (vllm_mm_gpt.py:848)
    smem_layernorm(buf, fn_w, fn_b, H, eps, red);        // final_norm      (vllm_mm_gpt.py:671)
    TOut* y = Y + (size_t)i * H;
    for (int c = threadIdx.x; c < H; c += blockDim.x) y[c] = from_f32<TOut>(buf[c]);
    __syncthreads();
    if (latents) {
        smem_layernorm(buf, fn_w, fn_b, H, eps, red);    // engine final_norm (XTTSv2.py:687) — App. B.2
        const int slot = slots[i];
        const int pos = lat_pos ? lat_pos[i] : n_gen[slot];
        if (pos >= 0 && pos < lat_rows_per_slot) {
            float* l = latents + ((size_t)slot * lat_rows_per_slot + pos) * H;
            for (int c = threadIdx.x; c < H; c += blockDim.x) l[c] = buf[c];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// paged KV cache write.  grid (rows, heads), 128 threads: 0..63 -> K[d], 64..127 -> V[d]
// ------------------------------------------------------------------------------------------------
template <typename TKV>
__global__ void kv_write_kernel(const float* __restrict__ QKV, const int* __restrict__ row_slot,
                                const int* __restrict__ row_pos, const int* __restrict__ ctx_len,
                                const int* __restrict__ block_tables, int max_pages, TKV* __restrict__ kpool,
                                TKV* __restrict__ vpool, int heads) {
    constexpr int X = 16 / sizeof(TKV);
    const int r = blockIdx.x, h = blockIdx.y;
    const int H = heads * kHeadDim;
    const int slot = row_slot[r];
    const int pos = row_pos ? row_pos[r] : ctx_len[slot];
    const int page = block_tables[(size_t)slot * max_pages + pos / kPageTokens];
    const int tk = pos % kPageTokens;
    const int d = threadIdx.x & 63;
    const size_t pbase = ((size_t)page * heads + h) * (kPageTokens * kHeadDim);
    if (threadIdx.x < 64) {
        const float k = QKV[(size_t)r * 3 * H + H + h * kHeadDim + d];
        kpool[pbase + ((size_t)(d / X) * kPageTokens + tk) * X + (d % X)] = from_f32<TKV>(k);
    } else {
        const float v = QKV[(size_t)r * 3 * H + 2 * H + h * kHeadDim + d];
        vpool[pbase + (size_t)tk * kHeadDim + d] = from_f32<TKV>(v);
    }
}

// the fp8 cache (kv_fp8.cuh): same grid and thread roles, each (row, head) quantised with its own K and V exponents
__global__ void __launch_bounds__(128)
kv_write_fp8_kernel(const float* __restrict__ QKV, const int* __restrict__ row_slot, const int* __restrict__ row_pos,
                    const int* __restrict__ ctx_len, const int* __restrict__ block_tables, int max_pages,
                    uint8_t* __restrict__ kpool, uint8_t* __restrict__ vpool, int heads) {
    __shared__ float red[4];
    const int r = blockIdx.x, h = blockIdx.y;
    const int H = heads * kHeadDim;
    const int slot = row_slot[r];
    const int pos = row_pos ? row_pos[r] : ctx_len[slot];
    const size_t b = kv8_block(block_tables[(size_t)slot * max_pages + pos / kPageTokens], heads, h);
    const int t = threadIdx.x;
    const float x = QKV[(size_t)r * 3 * H + (t < 64 ? H : 2 * H) + h * kHeadDim + (t & 63)];
    kv8_append(x, kpool + b, vpool + b, pos % kPageTokens, red);
}

// ------------------------------------------------------------------------------------------------
// decode attention over the paged cache: one CTA per (sequence, head); 4 warps split the pages;
// lane = token inside a page for QK^T (16-byte coalesced K reads), lane = 2 output dims for PV.
// HBM-bound: reads 2*ctx*64*sizeof(TKV) bytes per (seq, head).
// ------------------------------------------------------------------------------------------------
template <typename TKV> struct KVec;
template <> struct KVec<float> {
    static constexpr int X = 4;                       // elements per 16-byte atom
    static __device__ __forceinline__ void unpack(const uint4& raw, float* f) {
        f[0] = __uint_as_float(raw.x); f[1] = __uint_as_float(raw.y); f[2] = __uint_as_float(raw.z); f[3] = __uint_as_float(raw.w);
    }
};
template <> struct KVec<__nv_bfloat16> {
    static constexpr int X = 8;
    static __device__ __forceinline__ void unpack(const uint4& raw, float* f) {
        const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 t = __bfloat1622float2(b[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
    }
};
template <> struct KVec<__half> {
    static constexpr int X = 8;
    static __device__ __forceinline__ void unpack(const uint4& raw, float* f) {
        const __half2* b = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(b[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
    }
};
__device__ __forceinline__ uint4 ldg_stream(const void* p) {          // streaming 16-byte load: KV is read once per step
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// End of one fp8 decode-attention item, after each warp's pages: warp 0 adds the step's own token from shared memory, then
// the token groups of each warp (lanes with equal dim chunk) and the NW warps are folded into head h of output row i.  X:
// dims per lane, so 64 / X lanes cover a token row.  The same steps as the end of attn_decode_kernel, which keeps them
// inline: calling this from there changes its instruction schedule.
template <int X, int NW, typename TOut>
__device__ __forceinline__ void attn_decode_tail(const float* qs, const float* ks, const float* vs, float* pm, float* pl,
                                                 float (*pacc)[kHeadDim], float m, float l, float* acc, TOut* __restrict__ out,
                                                 int i, int h, int H) {
    constexpr int NCH = kHeadDim / X;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int tg = lane / NCH, dc = lane % NCH;
    if (w == 0) {
        // ---- the step's own token, from shared memory
        float s = qs[lane] * ks[lane] + qs[lane + 32] * ks[lane + 32];
        s = warp_sum(s);
        const float mnew = fmaxf(m, s);
        const float p = expf(s - mnew);
        const float corr = (m == -INFINITY) ? 0.f : expf(m - mnew);
        l = l * corr + p;
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] = acc[e] * corr + ((tg == 0) ? p * vs[dc * X + e] : 0.f);
        m = mnew;
    }
    // ---- fold the token groups of the warp (lanes with equal dc), then the 4 warps
#pragma unroll
    for (int o = NCH; o < 32; o <<= 1)
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
    if (lane == 0) { pm[w] = m; pl[w] = l; }
    if (lane < NCH) {
#pragma unroll
        for (int e = 0; e < X; ++e) pacc[w][dc * X + e] = acc[e];
    }
    __syncthreads();
    for (int t = tid; t < kHeadDim; t += 32 * NW) {
        float M = pm[0];
#pragma unroll
        for (int k = 1; k < NW; ++k) M = fmaxf(M, pm[k]);
        float L = 0.f, o = 0.f;
#pragma unroll
        for (int k = 0; k < NW; ++k) {
            const float e = (pm[k] == -INFINITY) ? 0.f : expf(pm[k] - M);
            L = fmaf(pl[k], e, L);
            o = fmaf(pacc[k][t], e, o);
        }
        out[(size_t)i * H + h * kHeadDim + t] = from_f32<TOut>(o / L);
    }
    __syncthreads();                                  // qs/ks/vs/pacc are reused by the next item
}

// One CTA per (sequence, head); the 4 warps take pages round-robin.  Per 32-token page a warp issues
//   QK^T : lane = token, 64/X independent 16-byte loads (K atoms of one token are 32*16 B apart, a warp-load is 512 B)
//   PV   : lane = (token group, 16-byte dim chunk), independent 16-byte loads, p broadcast by shuffle
// so ~16 wide loads are in flight per warp and page.  The step's own token is appended to the cache here (what
// reshape_and_cache does in vLLM) and attended to straight from shared memory, rounded to the cache type first so the
// result is identical to reading it back.
// HBM-bound: algorithmic bytes = 2 * ctx * 64 * sizeof(TKV) per (sequence, head).
template <typename TKV, typename TOut, int NW>
__global__ void __launch_bounds__(32 * NW)
attn_decode_kernel(const float* __restrict__ QKV, const int* __restrict__ active, const int* __restrict__ ctx_len,
                   const int* __restrict__ block_tables, int max_pages, TKV* __restrict__ kpool, TKV* __restrict__ vpool,
                   TOut* __restrict__ out, int heads, int n_items) {
    constexpr int X = KVec<TKV>::X;
    constexpr int NCH = kHeadDim / X;                 // 16-byte atoms per token row (8 bf16 / 16 fp32)
    constexpr int TPI = 32 / NCH;                     // tokens covered by one warp-wide V load (4 / 2)
    constexpr int VIT = kPageTokens / TPI;            // V loads per page (8 / 16)
    __shared__ __align__(16) float qs[kHeadDim], ks[kHeadDim], vs[kHeadDim];
    __shared__ float pm[NW], pl[NW];
    __shared__ float pacc[NW][kHeadDim];
    trace_pt(TR_ATTN, 0); pdl_trigger();
    // ncu: 24 resident warps per SM, long-scoreboard stalls dominate: the kernel is bound by the bytes its warps keep in
    // flight against ~1.6 us of HBM latency under load.
    pdl_wait();
    trace_pt(TR_ATTN, 1);
    const int H = heads * kHeadDim;
    // work items = (active row, head); the grid may be capped below M*heads (engine option "attn_ctas_per_sm") so that the
    // kernel leaves registers free for GEMM CTAs of a concurrent decode branch: then each CTA walks several items
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int i = item / heads, h = item - i * heads;
    const int slot = active[i];
    const int past = ctx_len[slot];                   // tokens already cached; the new one goes to position `past`
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int* bt = block_tables + (size_t)slot * max_pages;
    {
        const float* row = QKV + (size_t)i * 3 * H + h * kHeadDim;
        const int page = bt[past / kPageTokens], tk = past % kPageTokens;
        const size_t pbase = ((size_t)page * heads + h) * (kPageTokens * kHeadDim);
        for (int t = tid; t < 2 * kHeadDim; t += 32 * NW) {
            const int dd = t & 63;
            if (t < 64) {
                qs[dd] = row[dd] * 0.125f;                                           // 64^-0.5
                const TKV k = from_f32<TKV>(row[H + dd]);
                ks[dd] = to_f32<TKV>(k);
                kpool[pbase + ((size_t)(dd / X) * kPageTokens + tk) * X + (dd % X)] = k;
            } else {
                const TKV v = from_f32<TKV>(row[2 * H + dd]);
                vs[dd] = to_f32<TKV>(v);
                vpool[pbase + (size_t)tk * kHeadDim + dd] = v;
            }
        }
    }
    __syncthreads();
    const int tg = lane / NCH, dc = lane % NCH;       // PV role of this lane: token group, dim chunk
    float m = -INFINITY, l = 0.f;
    float acc[X];
#pragma unroll
    for (int e = 0; e < X; ++e) acc[e] = 0.f;
    const int npages = (past + kPageTokens - 1) / kPageTokens;
    for (int pg = w; pg < npages; pg += NW) {
        const int page = bt[pg];
        const size_t pbase = ((size_t)page * heads + h) * (kPageTokens * kHeadDim);
        const int nvalid = min(kPageTokens, past - pg * kPageTokens);
        // ---- issue every load of the page up front
        uint4 kraw[NCH], vraw[VIT];
        const TKV* kb = kpool + pbase + (size_t)lane * X;
#pragma unroll
        for (int c = 0; c < NCH; ++c) kraw[c] = ldg_stream(kb + (size_t)c * kPageTokens * X);
        const TKV* vb = vpool + pbase + (size_t)tg * kHeadDim + (size_t)dc * X;
#pragma unroll
        for (int it = 0; it < VIT; ++it) vraw[it] = ldg_stream(vb + (size_t)it * TPI * kHeadDim);
        // ---- scores
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            float kf[X];
            KVec<TKV>::unpack(kraw[c], kf);
#pragma unroll
            for (int e = 0; e < X; ++e) s = fmaf(kf[e], qs[c * X + e], s);
        }
        const bool valid = lane < nvalid;
        s = valid ? s : -INFINITY;
        const float mnew = fmaxf(m, warp_max(s));
        const float p = valid ? expf(s - mnew) : 0.f;
        const float corr = (m == -INFINITY) ? 0.f : expf(m - mnew);
        l = l * corr + warp_sum(p);
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] *= corr;
        // ---- PV
#pragma unroll
        for (int it = 0; it < VIT; ++it) {
            const int j = it * TPI + tg;
            const float pj = __shfl_sync(0xffffffffu, p, j);
            if (j < nvalid) {                           // stale page tails are never multiplied in
                float vf[X];
                KVec<TKV>::unpack(vraw[it], vf);
#pragma unroll
                for (int e = 0; e < X; ++e) acc[e] = fmaf(pj, vf[e], acc[e]);
            }
        }
        m = mnew;
    }
    if (w == 0) {
        // ---- the step's own token, from shared memory
        float s = qs[lane] * ks[lane] + qs[lane + 32] * ks[lane + 32];
        s = warp_sum(s);
        const float mnew = fmaxf(m, s);
        const float p = expf(s - mnew);
        const float corr = (m == -INFINITY) ? 0.f : expf(m - mnew);
        l = l * corr + p;
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] = acc[e] * corr + ((tg == 0) ? p * vs[dc * X + e] : 0.f);
        m = mnew;
    }
    // ---- fold the token groups of the warp (lanes with equal dc), then the 4 warps
#pragma unroll
    for (int o = NCH; o < 32; o <<= 1)
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
    if (lane == 0) { pm[w] = m; pl[w] = l; }
    if (lane < NCH) {
#pragma unroll
        for (int e = 0; e < X; ++e) pacc[w][dc * X + e] = acc[e];
    }
    __syncthreads();
    for (int t = tid; t < kHeadDim; t += 32 * NW) {
        float M = pm[0];
#pragma unroll
        for (int k = 1; k < NW; ++k) M = fmaxf(M, pm[k]);
        float L = 0.f, o = 0.f;
#pragma unroll
        for (int k = 0; k < NW; ++k) {
            const float e = (pm[k] == -INFINITY) ? 0.f : expf(pm[k] - M);
            L = fmaf(pl[k], e, L);
            o = fmaf(pacc[k][t], e, o);
        }
        out[(size_t)i * H + h * kHeadDim + t] = from_f32<TOut>(o / L);
    }
    __syncthreads();                                  // qs/ks/vs/pacc are reused by the next item
    }
    trace_pt(TR_ATTN, 2);
}

// The fp8 cache (kv_fp8.cuh).  A page is half the bytes of a 16-bit page, and the kernel is bound by the bytes each warp
// keeps in flight, so a warp takes two of its pages per iteration (pages pg and pg + NW: the same pages per warp as the
// 16-bit kernel): 8 K + 8 V 16-byte loads up front, as there, plus each lane's K and V exponent byte.  The exponents are
// applied to the score (2^ek) and to p_j before the PV broadcast (2^ev); l sums the unscaled p.  The step's own token is
// appended in the fp8 format and attended to as its dequantised values.
template <typename TOut>
__global__ void __launch_bounds__(128)
attn_decode_fp8_kernel(const float* __restrict__ QKV, const int* __restrict__ active, const int* __restrict__ ctx_len,
                       const int* __restrict__ block_tables, int max_pages, uint8_t* __restrict__ kpool,
                       uint8_t* __restrict__ vpool, TOut* __restrict__ out, int heads, int n_items) {
    constexpr int NW = 4;                             // kv8_append: one thread per K / V element of the new token
    constexpr int X = kKv8X;
    constexpr int NCH = kHeadDim / X;                 // 4 atoms per token row
    constexpr int TPI = 32 / NCH;                     // 8 tokens per warp-wide V load
    constexpr int VIT = kPageTokens / TPI;            // 4 V loads per page
    __shared__ __align__(16) float qs[kHeadDim], ks[kHeadDim], vs[kHeadDim];
    __shared__ float pm[NW], pl[NW], red[NW];
    __shared__ float pacc[NW][kHeadDim];
    trace_pt(TR_ATTN, 0); pdl_trigger();
    pdl_wait();
    trace_pt(TR_ATTN, 1);
    const int H = heads * kHeadDim;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int i = item / heads, h = item - i * heads;
    const int slot = active[i];
    const int past = ctx_len[slot];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int* bt = block_tables + (size_t)slot * max_pages;
    {
        const float* row = QKV + (size_t)i * 3 * H + h * kHeadDim;
        const size_t b = kv8_block(bt[past / kPageTokens], heads, h);
        const int dd = tid & 63;
        const float x = kv8_append(row[(tid < 64 ? H : 2 * H) + dd], kpool + b, vpool + b, past % kPageTokens, red);
        if (tid < 64) { qs[dd] = row[dd] * 0.125f; ks[dd] = x; } else vs[dd] = x;
    }
    __syncthreads();
    const int tg = lane / NCH, dc = lane % NCH;
    float m = -INFINITY, l = 0.f;
    float acc[X];
#pragma unroll
    for (int e = 0; e < X; ++e) acc[e] = 0.f;
    const int npages = (past + kPageTokens - 1) / kPageTokens;
    for (int pg = w; pg < npages; pg += 2 * NW) {
        // ---- issue every load of both pages up front
        uint4 kraw[2][NCH], vraw[2][VIT];
        int ek[2] = {0, 0}, ev[2] = {0, 0}, nvalid[2] = {0, 0};
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int p = pg + u * NW;
            if (p < npages) {
                const size_t b = kv8_block(bt[p], heads, h);
                nvalid[u] = min(kPageTokens, past - p * kPageTokens);
                const uint8_t* kb = kpool + b + (size_t)lane * X;
#pragma unroll
                for (int c = 0; c < NCH; ++c) kraw[u][c] = ldg_stream(kb + (size_t)c * kPageTokens * X);
                const uint8_t* vb = vpool + b + (size_t)tg * kHeadDim + (size_t)dc * X;
#pragma unroll
                for (int it = 0; it < VIT; ++it) vraw[u][it] = ldg_stream(vb + (size_t)it * TPI * kHeadDim);
                ek[u] = (int8_t)__ldg(kpool + b + kv8_e_off(lane));
                ev[u] = (int8_t)__ldg(vpool + b + kv8_e_off(lane));
            } else {
#pragma unroll
                for (int c = 0; c < NCH; ++c) kraw[u][c] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                for (int it = 0; it < VIT; ++it) vraw[u][it] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        // ---- scores of both pages, one softmax update
        float s[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            float d = 0.f;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                float kf[X];
                kv8_unpack16(kraw[u][c], kf);
#pragma unroll
                for (int e = 0; e < X; ++e) d = fmaf(kf[e], qs[c * X + e], d);
            }
            s[u] = lane < nvalid[u] ? d * kv8_pow2(ek[u]) : -INFINITY;
        }
        const float mnew = fmaxf(m, warp_max(fmaxf(s[0], s[1])));
        const float p0 = lane < nvalid[0] ? expf(s[0] - mnew) : 0.f;
        const float p1 = lane < nvalid[1] ? expf(s[1] - mnew) : 0.f;
        const float corr = (m == -INFINITY) ? 0.f : expf(m - mnew);
        l = l * corr + warp_sum(p0 + p1);
#pragma unroll
        for (int e = 0; e < X; ++e) acc[e] *= corr;
        // ---- PV: lane j's weight carries its token's V scale
        const float pv[2] = {p0 * kv8_pow2(ev[0]), p1 * kv8_pow2(ev[1])};
#pragma unroll
        for (int u = 0; u < 2; ++u) {
#pragma unroll
            for (int it = 0; it < VIT; ++it) {
                const int j = it * TPI + tg;
                const float pj = __shfl_sync(0xffffffffu, pv[u], j);
                if (j < nvalid[u]) {                    // stale page tails are never multiplied in
                    float vf[X];
                    kv8_unpack16(vraw[u][it], vf);
#pragma unroll
                    for (int e = 0; e < X; ++e) acc[e] = fmaf(pj, vf[e], acc[e]);
                }
            }
        }
        m = mnew;
    }
    attn_decode_tail<X, NW>(qs, ks, vs, pm, pl, pacc, m, l, acc, out, i, h, H);
    }
    trace_pt(TR_ATTN, 2);
}

// ------------------------------------------------------------------------------------------------
// generic fp32 attention for prefill-style work (GPT prompt, conditioning encoder, perceiver).
// CTA = 16 queries of one (sequence, head); K/V tiles of 32 keys staged in shared memory;
// each warp owns 4 queries; lane = key for QK^T, lane = dims {lane, lane+32} for PV.
// ------------------------------------------------------------------------------------------------
constexpr int AQ = 16;

template <typename TOut>
__global__ void __launch_bounds__(128)
attn_generic_kernel(AttnLayout L, const AttnSeq* __restrict__ seqs, TOut* __restrict__ out, int out_row_stride) {
    __shared__ __align__(16) float qT[kHeadDim][AQ];          // [d][query]
    __shared__ float Ks[32][kHeadDim + 1];
    __shared__ float Vs[32][kHeadDim];
    const AttnSeq sq = seqs[blockIdx.z];
    const int q0 = blockIdx.x * AQ;
    if (q0 >= sq.nq) return;
    const int h = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int shift = sq.nk - sq.nq;
    // stage queries (pre-scaled)
    for (int e = tid; e < AQ * kHeadDim; e += 128) {
        const int qi = e / kHeadDim, d = e % kHeadDim;
        const int gq = q0 + qi;
        float v = 0.f;
        if (gq < sq.nq) v = L.q[(size_t)(sq.q_start + gq) * L.q_row_stride + (size_t)h * L.q_head_stride + d] * L.scale;
        qT[d][qi] = v;
    }
    float m[4], l[4], a0[4], a1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { m[i] = -INFINITY; l[i] = 0.f; a0[i] = 0.f; a1[i] = 0.f; }
    const int q_last = min(q0 + AQ, sq.nq) - 1;
    const int kmax = L.causal ? min(sq.nk, q_last + shift + 1) : sq.nk;
    for (int k0 = 0; k0 < kmax; k0 += 32) {
        __syncthreads();
        for (int e = tid; e < 32 * kHeadDim; e += 128) {
            const int j = e / kHeadDim, d = e % kHeadDim;
            const int gk = k0 + j;
            float kv = 0.f, vv = 0.f;
            if (gk < sq.nk) {
                const size_t off = (size_t)(sq.kv_start + gk) * L.kv_row_stride + (size_t)h * L.kv_head_stride + d;
                kv = L.k[off];
                vv = L.v[off];
            }
            Ks[j][d] = kv;
            Vs[j][d] = vv;
        }
        __syncthreads();
        float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 16
        for (int d = 0; d < kHeadDim; ++d) {
            const float kd = Ks[lane][d];
            const float4 q4 = *reinterpret_cast<const float4*>(&qT[d][w * 4]);
            s[0] = fmaf(q4.x, kd, s[0]); s[1] = fmaf(q4.y, kd, s[1]);
            s[2] = fmaf(q4.z, kd, s[2]); s[3] = fmaf(q4.w, kd, s[3]);
        }
        const int gk = k0 + lane;
        float p[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int gq = q0 + w * 4 + i;
            const bool vis = (gk < sq.nk) && (!L.causal || gk <= gq + shift);
            const float si = vis ? s[i] : -INFINITY;
            const float mnew = fmaxf(m[i], warp_max(si));
            p[i] = (si == -INFINITY) ? 0.f : expf(si - mnew);
            const float corr = (m[i] == -INFINITY) ? 0.f : expf(m[i] - mnew);
            l[i] = l[i] * corr + warp_sum(p[i]);
            a0[i] *= corr; a1[i] *= corr;
            m[i] = mnew;
        }
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const float v0 = Vs[j][lane], v1 = Vs[j][lane + 32];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float pj = __shfl_sync(0xffffffffu, p[i], j);
                a0[i] = fmaf(pj, v0, a0[i]);
                a1[i] = fmaf(pj, v1, a1[i]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int gq = q0 + w * 4 + i;
        if (gq < sq.nq) {
            TOut* o = out + (size_t)(sq.q_start + gq) * out_row_stride + h * kHeadDim;
            const float inv = 1.0f / l[i];
            o[lane] = from_f32<TOut>(a0[i] * inv);
            o[lane + 32] = from_f32<TOut>(a1[i] * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// fused sampler: penalty -> (greedy | /T -> top-k -> top-p -> softmax -> argmax(p / Exp(1)))
// one CTA (256 threads) per sequence; V <= 2048.
// ------------------------------------------------------------------------------------------------
constexpr int SV = 2048;

struct KeyIdx { float v; int i; };
__device__ __forceinline__ bool key_less(const KeyIdx& a, const KeyIdx& b) {
    return (a.v < b.v) || (a.v == b.v && a.i < b.i);
}

__global__ void __launch_bounds__(256)
sample_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ active, int V, SampleState S,
              int advance_ctx) {
    __shared__ float zs[SV];         // logits after penalty (/T), original order
    __shared__ float sv[SV];         // sort values
    __shared__ short si[SV];         // sort indices
    __shared__ float red[32];
    __shared__ int redi[32];
    __shared__ float scan_part[256];
    trace_pt(TR_SAMPLE, 0); pdl_trigger(); pdl_wait(); trace_pt(TR_SAMPLE, 1);
    const int tid = threadIdx.x;
    const int slot = active[blockIdx.x];
    if (S.beam && S.beam[slot]) return;                 // a beam: the beam kernels choose its token (beam.cu)
    const int n = S.n_gen[slot];
    const float* z = logits + (size_t)blockIdx.x * ld;
    const float pen = S.penalty[slot];
    const unsigned* seen = S.seen + (size_t)slot * S.seen_words;
    const float T = S.temperature[slot];
    const bool greedy = T < 1e-5f;
    for (int v = tid; v < SV; v += 256) {
        float x = -INFINITY;
        if (v < V) {
            x = z[v];
            if (pen != 1.0f && ((seen[v >> 5] >> (v & 31)) & 1u)) x = (x > 0.f) ? x / pen : x * pen;
            if (!greedy) x = x / T;
        }
        zs[v] = x;
    }
    __syncthreads();
    int chosen = 0;
    const int tk_fast = S.top_k[slot];
    bool fast_done = false;
    if (!greedy && tk_fast > 0 && tk_fast <= 64 && tk_fast < V) {
        // ---- fast path (the usual top_k = 50): radix-select the k-th largest logit, compact the <= 128 survivors,
        //      sort just those, then top-p / softmax / Exp(1) race on the short list.  Same kept set and same
        //      arithmetic as the full-sort path below, which remains the fallback (top_k off, > 64, or > 128 ties).
        __shared__ unsigned hist[256];
        __shared__ unsigned sel_prefix, sel_k, ncand;
        __shared__ float cv[128];
        __shared__ short ci[128];
        __shared__ float cum[128];
        // order-preserving key; -0.0 maps to +0.0's key, since the full sort's float compare treats the two as equal
        auto fkey = [](float x) {
            unsigned b = __float_as_uint(x);
            if (b == 0x80000000u) b = 0u;
            return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
        };
        if (tid == 0) { sel_prefix = 0u; sel_k = (unsigned)tk_fast; ncand = 0u; }
        for (int pass = 3; pass >= 0; --pass) {
            hist[tid] = 0u;
            __syncthreads();
            const unsigned pfx = sel_prefix;
            const unsigned himask = (pass == 3) ? 0u : (0xFFFFFFFFu << ((pass + 1) * 8));
            for (int v = tid; v < V; v += 256) {
                const unsigned k = fkey(zs[v]);
                if ((k & himask) == pfx) atomicAdd(&hist[(k >> (pass * 8)) & 255u], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                unsigned need = sel_k, d = 255;
                for (;; --d) {                                   // from the top digit down: where does the k-th largest live?
                    if (hist[d] >= need) break;
                    need -= hist[d];
                    if (d == 0) break;
                }
                sel_k = need;
                sel_prefix = pfx | (d << (pass * 8));
            }
            __syncthreads();
        }
        const unsigned kth_key = sel_prefix;
        for (int v = tid; v < V; v += 256) {
            if (fkey(zs[v]) >= kth_key) {
                const unsigned pos = atomicAdd(&ncand, 1u);
                if (pos < 128u) { cv[pos] = zs[v]; ci[pos] = (short)v; }
            }
        }
        __syncthreads();
        const int nc = (int)ncand;
        if (nc <= 128) {
            if (tid < 128 && tid >= nc) { cv[tid] = -INFINITY; ci[tid] = (short)(SV + tid); }    // pads sort to the front
            __syncthreads();
            for (int k = 2; k <= 128; k <<= 1)
                for (int j = k >> 1; j > 0; j >>= 1) {
                    if (tid < 128) {
                        const int ixj = tid ^ j;
                        if (ixj > tid) {
                            KeyIdx a{cv[tid], ci[tid]}, b{cv[ixj], ci[ixj]};
                            const bool up = ((tid & k) == 0);
                            const bool sw = up ? key_less(b, a) : key_less(a, b);
                            if (sw) { cv[tid] = b.v; ci[tid] = (short)b.i; cv[ixj] = a.v; ci[ixj] = (short)a.i; }
                        }
                    }
                    __syncthreads();
                }
            const float mx = cv[127];
            const float tp = S.top_p[slot];
            if (tid == 0) {                                      // <= 128 entries: a serial ascending scan is the cheapest
                float run = 0.f;
                for (int i = 0; i < 128; ++i) { run += (cv[i] == -INFINITY) ? 0.f : expf(cv[i] - mx); cum[i] = run; }
            }
            __syncthreads();
            const float total_k = cum[127];
            if (tp < 1.0f && tid < 127) {
                if (cum[tid] * (1.0f / total_k) <= 1.0f - tp) cv[tid] = -INFINITY;
            }
            __syncthreads();
            if (tid == 0) {
                float run = 0.f;
                for (int i = 0; i < 128; ++i) run += (cv[i] == -INFINITY) ? 0.f : expf(cv[i] - mx);
                cum[0] = run;                                    // softmax denominator over the kept set
            }
            __syncthreads();
            const float total = cum[0];
            const unsigned long long seed = S.seed[slot];
            const uint32_t k0 = (uint32_t)(seed & 0xffffffffull), k1 = (uint32_t)(seed >> 32);
            float best = -1.f; int besti = 0x7fffffff;
            if (tid < 128 && cv[tid] != -INFINITY) {
                const int v = ci[tid];
                uint32_t r[4];
                philox4x32_10((uint32_t)(v >> 2), (uint32_t)n, (uint32_t)S.seq_seed[slot], 0u, k0, k1, r);
                const float p = expf(cv[tid] - mx) / total;
                const float uu = ((float)(r[v & 3] >> 9) + 0.5f) * (1.0f / 8388608.0f);
                best = p / (-logf(uu)); besti = v;
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
                if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
            }
            if ((tid & 31) == 0) { red[tid >> 5] = best; redi[tid >> 5] = besti; }
            __syncthreads();
            if (tid < 32) {
                best = (tid < 8) ? red[tid] : -2.f;
                besti = (tid < 8) ? redi[tid] : 0x7fffffff;
                for (int o = 16; o > 0; o >>= 1) {
                    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
                    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
                }
                chosen = besti;
            }
            fast_done = true;
        }
        __syncthreads();
    }
    if (!greedy && !fast_done) {
        // ---- ascending bitonic sort of (value, index); the SV-V pads (-inf, idx>=V) go to the front
        for (int v = tid; v < SV; v += 256) { sv[v] = zs[v]; si[v] = (short)v; }
        __syncthreads();
        for (int k = 2; k <= SV; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int t = tid; t < SV; t += 256) {
                    const int ixj = t ^ j;
                    if (ixj > t) {
                        KeyIdx a{sv[t], si[t]}, b{sv[ixj], si[ixj]};
                        const bool up = ((t & k) == 0);
                        const bool sw = up ? key_less(b, a) : key_less(a, b);
                        if (sw) { sv[t] = b.v; si[t] = (short)b.i; sv[ixj] = a.v; si[ixj] = (short)a.i; }
                    }
                }
                __syncthreads();
            }
        }
        // ---- top-k: keep >= k-th largest
        const int tk = S.top_k[slot];
        if (tk > 0 && tk < V) {
            const float kth = sv[SV - tk];
            __syncthreads();
            for (int v = tid; v < SV; v += 256) if (sv[v] < kth) sv[v] = -INFINITY;
            __syncthreads();
        }
        // ---- top-p on the ascending order: drop while cumulative softmax <= 1-p, always keep the last
        const float tp = S.top_p[slot];
        const float mx = sv[SV - 1];
        if (tp < 1.0f) {
            float e[8], loc = 0.f;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const float x = sv[tid * 8 + u];
                e[u] = (x == -INFINITY) ? 0.f : expf(x - mx);
                loc += e[u];
            }
            const float total = block_sum(loc, red);
            // inclusive scan of per-thread partial sums
            scan_part[tid] = loc;
            __syncthreads();
            for (int off = 1; off < 256; off <<= 1) {
                const float add = (tid >= off) ? scan_part[tid - off] : 0.f;
                __syncthreads();
                scan_part[tid] += add;
                __syncthreads();
            }
            float run = (tid == 0) ? 0.f : scan_part[tid - 1];
            const float thr = 1.0f - tp;
            const float inv = 1.0f / total;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                run += e[u];
                const int pos = tid * 8 + u;
                if (pos != SV - 1 && run * inv <= thr) sv[pos] = -INFINITY;
            }
            __syncthreads();
        }
        // ---- scatter the kept logits back to vocabulary order
        for (int v = tid; v < SV; v += 256) { const int id = si[v]; if (id < V) zs[id] = sv[v]; }
        __syncthreads();
        // ---- softmax over kept, then argmax(p / e), e ~ Exp(1) from Philox(counter=(v/4, step, seq_seed, 0))
        float loc = 0.f;
        for (int v = tid; v < V; v += 256) { const float x = zs[v]; loc += (x == -INFINITY) ? 0.f : expf(x - mx); }
        const float total = block_sum(loc, red);
        const unsigned long long seed = S.seed[slot];
        const uint32_t k0 = (uint32_t)(seed & 0xffffffffull), k1 = (uint32_t)(seed >> 32);
        const uint32_t sseed = (uint32_t)S.seq_seed[slot];
        float best = -1.f; int besti = 0x7fffffff;
        for (int blk = tid; blk * 4 < V; blk += 256) {
            uint32_t r[4];
            philox4x32_10((uint32_t)blk, (uint32_t)n, sseed, 0u, k0, k1, r);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int v = blk * 4 + u;
                if (v < V) {
                    const float x = zs[v];
                    const float p = (x == -INFINITY) ? 0.f : expf(x - mx) / total;
                    const float uu = ((float)(r[u] >> 9) + 0.5f) * (1.0f / 8388608.0f);
                    const float ee = -logf(uu);
                    const float ratio = p / ee;
                    if (ratio > best || (ratio == best && v < besti)) { best = ratio; besti = v; }
                }
            }
        }
        // block argmax (max ratio, lowest index on ties)
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
        }
        __syncthreads();
        if ((tid & 31) == 0) { red[tid >> 5] = best; redi[tid >> 5] = besti; }
        __syncthreads();
        if (tid < 32) {
            best = (tid < 8) ? red[tid] : -2.f;
            besti = (tid < 8) ? redi[tid] : 0x7fffffff;
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
                if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
            }
            chosen = besti;
        }
    } else if (greedy) {
        float best = -INFINITY; int besti = 0x7fffffff;
        for (int v = tid; v < V; v += 256) {
            const float x = zs[v];
            if (x > best || (x == best && v < besti)) { best = x; besti = v; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
        }
        if ((tid & 31) == 0) { red[tid >> 5] = best; redi[tid >> 5] = besti; }
        __syncthreads();
        if (tid < 32) {
            best = (tid < 8) ? red[tid] : -INFINITY;
            besti = (tid < 8) ? redi[tid] : 0x7fffffff;
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
                if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
            }
            chosen = besti;
        }
    }
    if (tid == 0) {
        if (chosen < 0 || chosen >= V) chosen = 0;          // all -inf/NaN guard
        int tok = chosen;
        if (S.forced) { const int f = S.forced[(size_t)slot * S.tokens_cap + n]; if (f >= 0) tok = f; }
        if (n < S.tokens_cap) {
            S.tokens[(size_t)slot * S.tokens_cap + n] = tok;
            S.sampled[(size_t)slot * S.tokens_cap + n] = chosen;
        }
        S.last_tok[slot] = tok;
        S.seen[(size_t)slot * S.seen_words + (tok >> 5)] |= (1u << (tok & 31));
        S.n_gen[slot] = n + 1;
        if (advance_ctx) S.ctx_len[slot] += 1;
        if (tok == S.stop_token[slot] || n + 1 >= S.max_tokens[slot]) S.finished[slot] = 1;
    }
}

}  // namespace

// ================================================================================================
// launchers
// ================================================================================================
XTTS_TRACE_SETTER(trace_set_gpt)

void launch_init_slots(const SlotInit* init, const int* pages, int n, SlotArrays a, cudaStream_t st) {
    if (n <= 0) return;
    ProfScope ps(KF_MISC, st, 0, (double)n * (sizeof(SlotInit) + 8.0 * a.max_pages + 4.0 * a.seen_words));
    init_slots_kernel<<<n, 128, 0, st>>>(init, pages, a);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_gather_rows(const float* src, const int* idx_host, int n, int width, float* dst, cudaStream_t st) {
    if (n <= 0) return;
    if (n > kVocMaxItems) throw CudaError("gather_rows: too many rows");
    GatherIdx G{};
    for (int i = 0; i < n; ++i) G.idx[i] = idx_host[i];
    ProfScope ps(KF_MISC, st, 0, 8.0 * n * width);
    gather_rows_kernel<<<n, 128, 0, st>>>(src, G, width, dst);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_build_rows(const RowDesc* rows, int n_rows, GptTables t, float* X, cudaStream_t st) {
    if (n_rows <= 0) return;
    ProfScope ps(KF_EMBED, st, 0, 12.0 * n_rows * t.H);
    build_rows_kernel<<<n_rows, 256, 0, st>>>(rows, t, X);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

void launch_build_decode_rows(const int* active, int M, const int* last_tok, const int* n_gen, GptTables t,
                              float* X, cudaStream_t st, bool pdl) {
    if (M <= 0) return;
    ProfScope ps(KF_EMBED, st, 0, 12.0 * M * t.H);
    launch_k(build_decode_rows_kernel, dim3(M), dim3(256), 0, st, pdl, active, last_tok, n_gen, t, X);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

template <typename TOut>
void launch_layernorm(const float* X, const float* w, const float* b, TOut* Y, int M, int H, float eps,
                      cudaStream_t st, bool pdl) {
    if (M <= 0) return;
    ProfScope ps(KF_NORM, st, 0, (4.0 + sizeof(TOut)) * M * H);
    launch_k(layernorm_kernel<TOut>, dim3(M), dim3(256), 0, st, pdl, X, w, b, Y, H, eps);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_layernorm<float>(const float*, const float*, const float*, float*, int, int, float, cudaStream_t, bool);
template void launch_layernorm<__nv_bfloat16>(const float*, const float*, const float*, __nv_bfloat16*, int, int, float, cudaStream_t, bool);
template void launch_layernorm<__half>(const float*, const float*, const float*, __half*, int, int, float, cudaStream_t, bool);

template <typename TOut>
void launch_residual_reduce_layernorm(float* X, const float* partials, int splits, const float* bias, const float* w,
                                      const float* b, TOut* Y, int M, int H, float eps, cudaStream_t st, bool pdl) {
    if (M <= 0) return;
    ProfScope ps(KF_NORM, st, 0, (8.0 + 4.0 * splits + sizeof(TOut)) * M * H);
    launch_k(residual_reduce_ln_kernel<TOut>, dim3(M), dim3(256), H * sizeof(float), st, pdl, X, partials, splits, (size_t)M * H, bias, w, b, Y, H, eps);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_residual_reduce_layernorm<float>(float*, const float*, int, const float*, const float*, const float*, float*, int, int, float, cudaStream_t, bool);
template void launch_residual_reduce_layernorm<__nv_bfloat16>(float*, const float*, int, const float*, const float*, const float*, __nv_bfloat16*, int, int, float, cudaStream_t, bool);
template void launch_residual_reduce_layernorm<__half>(float*, const float*, int, const float*, const float*, const float*, __half*, int, int, float, cudaStream_t, bool);

template <typename TOut>
void launch_head_norms(const float* X, const int* row_index, const float* lnf_w, const float* lnf_b,
                       const float* fn_w, const float* fn_b, TOut* Y, float* latents, const int* slots,
                       const int* lat_pos, const int* n_gen, int lat_rows_per_slot, int M, int H, float eps,
                       cudaStream_t st, bool pdl) {
    if (M <= 0) return;
    ProfScope ps(KF_NORM, st, 0, (8.0 + sizeof(TOut)) * M * H);
    launch_k(head_norms_kernel<TOut>, dim3(M), dim3(256), H * sizeof(float), st, pdl, X, row_index, lnf_w, lnf_b, fn_w, fn_b, Y,
             latents, slots, lat_pos, n_gen, lat_rows_per_slot, H, eps);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_head_norms<float>(const float*, const int*, const float*, const float*, const float*, const float*, float*, float*, const int*, const int*, const int*, int, int, int, float, cudaStream_t, bool);
template void launch_head_norms<__nv_bfloat16>(const float*, const int*, const float*, const float*, const float*, const float*, __nv_bfloat16*, float*, const int*, const int*, const int*, int, int, int, float, cudaStream_t, bool);
template void launch_head_norms<__half>(const float*, const int*, const float*, const float*, const float*, const float*, __half*, float*, const int*, const int*, const int*, int, int, int, float, cudaStream_t, bool);

template <typename TKV>
void launch_kv_write(const float* QKV, int M, const int* row_slot, const int* row_pos, const int* ctx_len,
                     const int* block_tables, int max_pages, TKV* kpool, TKV* vpool, int heads, cudaStream_t st) {
    if (M <= 0) return;
    if constexpr (std::is_same_v<TKV, __nv_fp8_e4m3>) {
        // fp32 QKV in, e4m3 bytes + one exponent byte per (row, head) for K and for V out
        ProfScope ps(KF_KV_WRITE, st, 0, (8.0 * kHeadDim + 2.0 * (kHeadDim + 1)) * M * heads);
        kv_write_fp8_kernel<<<dim3(M, heads), 128, 0, st>>>(QKV, row_slot, row_pos, ctx_len, block_tables, max_pages,
                                                            reinterpret_cast<uint8_t*>(kpool), reinterpret_cast<uint8_t*>(vpool), heads);
    } else {
        ProfScope ps(KF_KV_WRITE, st, 0, (8.0 + 2.0 * sizeof(TKV)) * M * heads * kHeadDim);
        kv_write_kernel<TKV><<<dim3(M, heads), 128, 0, st>>>(QKV, row_slot, row_pos, ctx_len, block_tables, max_pages,
                                                             kpool, vpool, heads);
    }
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_kv_write<float>(const float*, int, const int*, const int*, const int*, const int*, int, float*, float*, int, cudaStream_t);
template void launch_kv_write<__nv_bfloat16>(const float*, int, const int*, const int*, const int*, const int*, int, __nv_bfloat16*, __nv_bfloat16*, int, cudaStream_t);
template void launch_kv_write<__half>(const float*, int, const int*, const int*, const int*, const int*, int, __half*, __half*, int, cudaStream_t);
template void launch_kv_write<__nv_fp8_e4m3>(const float*, int, const int*, const int*, const int*, const int*, int, __nv_fp8_e4m3*, __nv_fp8_e4m3*, int, cudaStream_t);

template <typename TKV, typename TOut>
void launch_attn_decode(const float* QKV, const int* active, int M, const int* ctx_len, const int* block_tables,
                        int max_pages, TKV* kpool, TKV* vpool, TOut* out, int heads, cudaStream_t st,
                        double ctx_sum_hint, bool pdl) {
    if (M <= 0) return;
    constexpr bool fp8 = std::is_same_v<TKV, __nv_fp8_e4m3>;
    // algorithmic bytes: K and V of every cached token of every sequence, once (fp8: with the token's exponent byte)
    const double tok_bytes = fp8 ? kHeadDim + 1.0 : (double)kHeadDim * sizeof(TKV);
    ProfScope ps(KF_ATTN_DECODE, st, 4.0 * ctx_sum_hint * heads * kHeadDim, 2.0 * ctx_sum_hint * heads * tok_bytes);
    const int n_items = M * heads;
    int grid = n_items;
    if (g_attn_ctas_per_sm > 0) {
        grid = std::min(n_items, sm_count() * g_attn_ctas_per_sm);
    } else if (g_attn_ctas_per_sm < 0) {
        grid = std::min(n_items, -g_attn_ctas_per_sm);          // test hook: an absolute grid size
    }
    if constexpr (fp8)
        launch_k(attn_decode_fp8_kernel<TOut>, dim3(grid), dim3(128), 0, st, pdl, QKV, active, ctx_len, block_tables, max_pages,
                 reinterpret_cast<uint8_t*>(kpool), reinterpret_cast<uint8_t*>(vpool), out, heads, n_items);
    else
        launch_k(attn_decode_kernel<TKV, TOut, 4>, dim3(grid), dim3(128), 0, st, pdl, QKV, active, ctx_len, block_tables, max_pages,
                 kpool, vpool, out, heads, n_items);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_attn_decode<float, float>(const float*, const int*, int, const int*, const int*, int, float*, float*, float*, int, cudaStream_t, double, bool);
template void launch_attn_decode<__nv_bfloat16, __nv_bfloat16>(const float*, const int*, int, const int*, const int*, int, __nv_bfloat16*, __nv_bfloat16*, __nv_bfloat16*, int, cudaStream_t, double, bool);
template void launch_attn_decode<__half, __half>(const float*, const int*, int, const int*, const int*, int, __half*, __half*, __half*, int, cudaStream_t, double, bool);
template void launch_attn_decode<__nv_fp8_e4m3, __nv_bfloat16>(const float*, const int*, int, const int*, const int*, int, __nv_fp8_e4m3*, __nv_fp8_e4m3*, __nv_bfloat16*, int, cudaStream_t, double, bool);
template void launch_attn_decode<__nv_fp8_e4m3, __half>(const float*, const int*, int, const int*, const int*, int, __nv_fp8_e4m3*, __nv_fp8_e4m3*, __half*, int, cudaStream_t, double, bool);

template <typename TOut>
void launch_attn_generic(AttnLayout L, const AttnSeq* seqs, int nseq, int max_nq, TOut* out, int out_row_stride,
                         cudaStream_t st) {
    if (nseq <= 0 || max_nq <= 0) return;
    ProfScope ps(KF_ATTN_PREFILL, st);
    attn_generic_kernel<TOut><<<dim3(ceil_div(max_nq, AQ), L.heads, nseq), 128, 0, st>>>(L, seqs, out, out_row_stride);
    COUNT_LAUNCH(); KERNEL_CHECK();
}
template void launch_attn_generic<float>(AttnLayout, const AttnSeq*, int, int, float*, int, cudaStream_t);
template void launch_attn_generic<__nv_bfloat16>(AttnLayout, const AttnSeq*, int, int, __nv_bfloat16*, int, cudaStream_t);
template void launch_attn_generic<__half>(AttnLayout, const AttnSeq*, int, int, __half*, int, cudaStream_t);

void launch_sample(const float* logits, int ld_logits, const int* active, int M, int V, SampleState s,
                   int advance_ctx, cudaStream_t st, bool pdl) {
    if (M <= 0) return;
    if (V > SV) throw CudaError("sample: vocabulary larger than 2048 is not supported");
    ProfScope ps(KF_SAMPLE, st, 0, 4.0 * M * V);
    launch_k(sample_kernel, dim3(M), dim3(256), 0, st, pdl, logits, ld_logits, active, V, s, advance_ctx);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
