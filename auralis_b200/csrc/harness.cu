// Kernel isolation harness (harness.h): the bodies of the xtts_debug_* entry points.  Every argument check runs before the
// first launch; each entry point then issues the launcher calls the engine issues for that kernel, on the engine's stream.
#include "harness.h"
#include "kernels.h"

#include <algorithm>
#include <cstring>
#include <limits>
#include <type_traits>
#include <vector>

namespace xtts {
namespace {

// Calls f with a null T* for element type 0 (fp32), 1 (bf16) or 2 (fp16) and returns its result; any other type throws
// "<what> 0 (fp32), 1 (bf16) or 2 (fp16)".
template <typename F>
auto with_elem(int type, const char* what, F&& f) {
    switch (type) {
    case 0: return f(static_cast<float*>(nullptr));
    case 1: return f(static_cast<__nv_bfloat16*>(nullptr));
    case 2: return f(static_cast<__half*>(nullptr));
    }
    throw std::runtime_error(std::string(what) + " 0 (fp32), 1 (bf16) or 2 (fp16)");
}

// Calls f with a null cache-element pointer and a null attention-output pointer for the KV type of the debug entry points:
// 0..2 the cache in the output type (as with_elem), 3 / 4 the fp8 cache (kv_fp8.cuh) with fp16 / bf16 output.
template <typename F>
auto with_kv(int kv_type, const char* what, F&& f) {
    switch (kv_type) {
    case 3: return f(static_cast<__nv_fp8_e4m3*>(nullptr), static_cast<__half*>(nullptr));
    case 4: return f(static_cast<__nv_fp8_e4m3*>(nullptr), static_cast<__nv_bfloat16*>(nullptr));
    }
    if (kv_type < 0 || kv_type > 2)
        throw std::runtime_error(std::string(what) + " 0 (fp32), 1 (bf16), 2 (fp16), 3 (fp8, fp16 out) or 4 (fp8, bf16 out)");
    return with_elem(kv_type, what, [&](auto* tag) { return f(tag, tag); });
}

// element type -> the type code of download_f32
template <typename T> constexpr int type_code() { return std::is_same_v<T, float> ? 0 : std::is_same_v<T, __half> ? 2 : 1; }

// host h[0 .. n) in a new device buffer; an empty buffer (p == NULL) for a NULL h
template <typename T>
DBuf<T> to_dev(const T* h, size_t n, cudaStream_t st) {
    DBuf<T> d;
    if (h) { d.alloc(n); d.upload(h, n, st); }
    return d;
}

// n device values of element type `type` (0 fp32, 1 bf16, 2 fp16) -> fp32 on the host (exact); synchronises the stream
void download_f32(const void* d, int type, float* out, size_t n, cudaStream_t st) {
    if (type == 0) {
        CUDA_CHECK(cudaMemcpyAsync(out, d, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        return;
    }
    std::vector<uint16_t> h(n);
    CUDA_CHECK(cudaMemcpyAsync(h.data(), d, n * sizeof(uint16_t), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n; ++i) {
        if (type == 2) { __half_raw r; r.x = h[i]; out[i] = __half2float(__half(r)); }
        else { const uint32_t u = (uint32_t)h[i] << 16; std::memcpy(&out[i], &u, 4); }
    }
}

// fp32 -> the 16-bit operand type of `mode` (1 bf16, 2 IEEE fp16 bits in the same buffer type)
void to16(int mode, const float* in, __nv_bfloat16* out, size_t n, cudaStream_t st) {
    if (mode == 2) launch_f32_to_f16(in, reinterpret_cast<__half*>(out), n, st);
    else launch_f32_to_bf16(in, out, n, st);
}

// Per-slot sampling parameters on the device and a SampleState pointing at them; its slot-state fields are the caller's.
struct Sampling {
    DBuf<float> temperature, top_p, penalty;
    DBuf<int> top_k, max_tokens, stop_token, seq_seed;
    DBuf<unsigned long long> seed;
    SampleState S{};
};
// slot s < n takes sp[s], or sp[0] when `broadcast`
Sampling upload_sampling(const xtts_sampling* sp, int n, bool broadcast, cudaStream_t st) {
    std::vector<float> T(n), tp(n), pen(n);
    std::vector<int> tk(n), mt(n), stp(n), ss(n);
    std::vector<unsigned long long> seed(n);
    for (int s = 0; s < n; ++s) {
        const xtts_sampling& p = sp[broadcast ? 0 : s];
        T[s] = p.temperature; tp[s] = p.top_p; pen[s] = p.repetition_penalty; tk[s] = p.top_k;
        mt[s] = p.max_tokens; stp[s] = p.stop_token; ss[s] = p.seq_seed; seed[s] = p.seed;
    }
    Sampling r;
    r.temperature = to_dev(T.data(), n, st); r.top_p = to_dev(tp.data(), n, st); r.penalty = to_dev(pen.data(), n, st);
    r.top_k = to_dev(tk.data(), n, st); r.max_tokens = to_dev(mt.data(), n, st); r.stop_token = to_dev(stp.data(), n, st);
    r.seq_seed = to_dev(ss.data(), n, st); r.seed = to_dev(seed.data(), n, st);
    r.S.temperature = r.temperature.p; r.S.top_p = r.top_p.p; r.S.penalty = r.penalty.p; r.S.top_k = r.top_k.p;
    r.S.max_tokens = r.max_tokens.p; r.S.stop_token = r.stop_token.p; r.S.seq_seed = r.seq_seed.p; r.S.seed = r.seed.p;
    return r;
}

// active[0 .. M) are distinct slots below n_slots
void check_active(const int32_t* active, int M, int n_slots, const char* msg) {
    std::vector<char> used(n_slots, 0);
    for (int i = 0; i < M; ++i) {
        const int s = active[i];
        if (s < 0 || s >= n_slots || used[s]) throw std::runtime_error(msg);
        used[s] = 1;
    }
}

// ids[0 .. n) are pages of a pool of n_pages
void check_pages(const int32_t* ids, int n, int n_pages, const char* msg) {
    for (int i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= n_pages) throw std::runtime_error(msg);
}

// A device copy of a host array of raw fp32 (U = uint32_t) or fp16 (uint16_t) bits with kGuardWords sentinels on each side;
// fetch() brings the array back and throws if the kernel wrote a sentinel.
constexpr int kGuardWords = 256;
template <typename U>
struct Guarded {
    static constexpr U kBits = sizeof(U) == 4 ? (U)0x7fc5a5a5u : (U)0x7e5au;    // quiet-NaN payloads no kernel here produces
    std::vector<U> h;
    DBuf<U> d;
    Guarded(const U* src, size_t n, cudaStream_t st) : h(n + 2 * kGuardWords, kBits) {
        std::copy(src, src + n, h.begin() + kGuardWords);
        d.alloc(h.size());
        d.upload(h.data(), h.size(), st);
    }
    U* p() const { return d.p + kGuardWords; }
    void fetch(U* dst, cudaStream_t st, const std::string& what) {
        d.download(h.data(), h.size(), st);
        CUDA_CHECK(cudaStreamSynchronize(st));
        const size_t n = h.size() - 2 * kGuardWords;
        for (int i = 0; i < kGuardWords; ++i)
            if (h[i] != kBits || h[kGuardWords + n + i] != kBits) throw std::runtime_error("debug_vocoder: " + what + " wrote outside its output");
        std::memcpy(dst, h.data() + kGuardWords, n * sizeof(U));
    }
};

}  // namespace

// One GEMM launch on private buffers.  The weights are converted and synchronised first; the activation conversion is the
// kernel right before the GEMM, so a PDL launch overlaps it exactly as the decode chain overlaps a GEMM with its producer
// (weight tiles requested before griddepcontrol.wait, activation tiles and the residual after it).
void debug_gemm(const HarnessCtx& c, int mode, const float* A, const float* W, const float* bias, const float* resid,
                float* out, int M, int N, int K, int dflags, int iters, float* ms) {
    if (mode < 0 || mode > 2) throw std::runtime_error("debug_gemm: mode 0 (fp32), 1 (bf16) or 2 (fp16)");
    if (M < 1 || N < 1 || K < 1 || !A || !W || !out) throw std::runtime_error("debug_gemm: empty problem");
    if (dflags & ~(XTTS_DEBUG_GEMM_GELU | XTTS_DEBUG_GEMM_OUT16 | XTTS_DEBUG_GEMM_INPLACE | XTTS_DEBUG_GEMM_PDL))
        throw std::runtime_error("debug_gemm: unknown flag bits");
    const bool out16 = dflags & XTTS_DEBUG_GEMM_OUT16, inplace = dflags & XTTS_DEBUG_GEMM_INPLACE, pdl = dflags & XTTS_DEBUG_GEMM_PDL;
    if (mode == 0 && (out16 || pdl)) throw std::runtime_error("debug_gemm: 16-bit output and PDL need mode 1 or 2");
    if (inplace && (!resid || out16)) throw std::runtime_error("debug_gemm: an in-place residual needs resid and fp32 output");
    if (mode >= 1 && (K % 64 != 0 || N % 32 != 0)) throw std::runtime_error("debug_gemm: modes 1 / 2 need K % 64 == 0 and N % 32 == 0");
    const cudaStream_t st = c.st;
    DBuf<float> dA = to_dev(A, (size_t)M * K, st), dW = to_dev(W, (size_t)N * K, st), db = to_dev(bias, N, st);
    DBuf<float> dr = to_dev(inplace ? nullptr : resid, (size_t)M * N, st), dout;
    DBuf<__nv_bfloat16> dout16;
    if (out16) dout16.alloc((size_t)M * N); else dout.alloc((size_t)M * N);
    const int flags = ((dflags & XTTS_DEBUG_GEMM_GELU) ? GEMM_GELU : 0) | (resid ? GEMM_RESID : 0) | (out16 ? GEMM_OUT_BF16 : 0) |
                      (mode == 2 ? GEMM_F16 : 0);
    DBuf<__nv_bfloat16> hA, hW;                     // 16-bit operands (IEEE fp16 bits in mode 2)
    if (mode >= 1) {
        std::string err;
        if (!gemm_tc_init(&err)) throw std::runtime_error(err);
        hA.alloc((size_t)M * K); hW.alloc((size_t)N * K);
        to16(mode, dW.p, hW.p, (size_t)N * K, st);
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
    // in place: out holds the residual and is passed as both (the engine's o-proj / down-proj without split-K)
    const float* rp = inplace ? dout.p : dr.p;
    void* op = out16 ? (void*)dout16.p : (void*)dout.p;
    auto run = [&] {
        if (mode >= 1) launch_gemm_bf16_tc(hA.p, hW.p, db.p, rp, op, M, N, K, flags, st, pdl);
        else launch_gemm_f32(dA.p, dW.p, db.p, rp, dout.p, M, N, K, flags, st);
    };
    if (inplace) dout.upload(resid, (size_t)M * N, st);
    if (mode >= 1) to16(mode, dA.p, hA.p, (size_t)M * K, st);
    run();
    download_f32(op, out16 ? mode : 0, out, (size_t)M * N, st);
    if (iters > 0) {
        cudaEvent_t e0, e1;
        CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0, st));
        for (int i = 0; i < iters; ++i) run();
        CUDA_CHECK(cudaEventRecord(e1, st));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float t = 0; CUDA_CHECK(cudaEventElapsedTime(&t, e0, e1));
        if (ms) *ms = t / iters;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
}

// One launch of the fused sampler (launch_sample) on private per-slot arrays: row r of logits samples for slot active[r]
// with that slot's parameters, and every state array comes back as the kernel left it.  seen crosses as one byte per id
// and is packed into ceil(V / 32) bitmap words per slot, as the engine keeps it.
void debug_sample_slots(const HarnessCtx& c, int Vn, int M, const int32_t* active, int n_slots, const float* logits, int ld,
                        const xtts_sampling* sp, int cap, int advance_ctx, const int32_t* forced, int32_t* n_gen,
                        int32_t* ctx_len, int32_t* finished, int32_t* last_tok, uint8_t* seen, int32_t* tokens,
                        int32_t* sampled) {
    if (Vn < 1 || Vn > 2048) throw std::runtime_error("debug_sample_slots: V must be 1..2048");
    if (n_slots < 1 || M < 1 || M > n_slots) throw std::runtime_error("debug_sample_slots: M must be 1..n_slots");
    if (ld < Vn) throw std::runtime_error("debug_sample_slots: ld < V");
    if (cap < 1) throw std::runtime_error("debug_sample_slots: cap must be >= 1");
    if (!active || !logits || !sp || !n_gen || !ctx_len || !finished || !last_tok || !seen || !tokens || !sampled)
        throw std::runtime_error("debug_sample_slots: only forced may be NULL");
    check_active(active, M, n_slots, "debug_sample_slots: active slots must be distinct and < n_slots");
    for (int i = 0; i < M; ++i) {
        const int s = active[i];
        // the kernel reads forced[slot][n_gen] without a bound check and sets the forced id's seen bit
        if (n_gen[s] < 0) throw std::runtime_error("debug_sample_slots: n_gen must be >= 0");
        if (forced && n_gen[s] >= cap) throw std::runtime_error("debug_sample_slots: with forced, n_gen must be < cap");
        if (forced && forced[(size_t)s * cap + n_gen[s]] >= Vn) throw std::runtime_error("debug_sample_slots: forced id >= V");
    }
    const cudaStream_t st = c.st;
    const int sw = (Vn + 31) / 32;
    const size_t nt = (size_t)n_slots * cap;
    std::vector<unsigned> sb((size_t)n_slots * sw, 0u);
    for (int s = 0; s < n_slots; ++s)
        for (int v = 0; v < Vn; ++v)
            if (seen[(size_t)s * Vn + v]) sb[(size_t)s * sw + (v >> 5)] |= 1u << (v & 31);
    DBuf<float> dlg = to_dev(logits, (size_t)M * ld, st);
    DBuf<int> dact = to_dev(active, M, st), dng = to_dev(n_gen, n_slots, st), dctx = to_dev(ctx_len, n_slots, st),
              dfin = to_dev(finished, n_slots, st), dlast = to_dev(last_tok, n_slots, st), dtok = to_dev(tokens, nt, st),
              dsmp = to_dev(sampled, nt, st), dfor = to_dev(forced, nt, st);
    DBuf<unsigned> dseen = to_dev(sb.data(), sb.size(), st);
    Sampling smp = upload_sampling(sp, n_slots, false, st);
    SampleState& S = smp.S;
    S.last_tok = dlast.p; S.n_gen = dng.p; S.ctx_len = dctx.p; S.finished = dfin.p;
    S.tokens = dtok.p; S.sampled = dsmp.p; S.forced = dfor.p; S.seen = dseen.p;
    S.tokens_cap = cap; S.seen_words = sw;
    launch_sample(dlg.p, ld, dact.p, M, Vn, S, advance_ctx, st);
    dng.download(n_gen, n_slots, st); dctx.download(ctx_len, n_slots, st); dfin.download(finished, n_slots, st);
    dlast.download(last_tok, n_slots, st); dtok.download(tokens, nt, st); dsmp.download(sampled, nt, st);
    dseen.download(sb.data(), sb.size(), st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    for (int s = 0; s < n_slots; ++s) {
        for (int v = 0; v < Vn; ++v) seen[(size_t)s * Vn + v] = (uint8_t)((sb[(size_t)s * sw + (v >> 5)] >> (v & 31)) & 1u);
        if (Vn % 32 && (sb[(size_t)s * sw + sw - 1] >> (Vn % 32)))
            throw std::runtime_error("debug_sample_slots: the kernel set a seen bit at an id >= V");
    }
}

// One launch of the paged decode attention (launch_attn_decode) on private buffers, under the engine's current attention
// options.  The pools are raw cache-typed arrays in the device layout (kernels.h); they come back with the appended tokens.
void debug_attn_decode(const HarnessCtx& c, int kv_type, int heads, int M, const int32_t* active, int n_slots,
                       const int32_t* ctx_len, const int32_t* block_tables, int mp, int n_pages, void* kpool, void* vpool,
                       const float* qkv, float* out) {
    with_kv(kv_type, "debug_attn_decode: kv_type", [&](auto* tag, auto* otag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        using TO = std::remove_pointer_t<decltype(otag)>;
        if (heads < 1 || M < 1 || n_slots < 1 || mp < 1 || n_pages < 1) throw std::runtime_error("debug_attn_decode: empty problem");
        // the kernels' contract: distinct active slots, the new token's page inside the block table, page ids inside the pool
        check_active(active, M, n_slots, "debug_attn_decode: active slots must be distinct and < n_slots");
        for (int i = 0; i < M; ++i) {
            const int s = active[i];
            if (ctx_len[s] < 0 || ctx_len[s] / kPageTokens >= mp) throw std::runtime_error("debug_attn_decode: ctx_len outside the block table");
            check_pages(block_tables + (size_t)s * mp, ctx_len[s] / kPageTokens + 1, n_pages, "debug_attn_decode: page id outside the pool");
        }
        const cudaStream_t st = c.st;
        const size_t pool = (size_t)n_pages * heads * kv_block_bytes(sizeof(T)), Hq = (size_t)heads * kHeadDim;
        DBuf<int> dact = to_dev(active, M, st), dctx = to_dev(ctx_len, n_slots, st), dbt = to_dev(block_tables, (size_t)n_slots * mp, st);
        DBuf<float> dqkv = to_dev(qkv, (size_t)M * 3 * Hq, st);
        DBuf<uint8_t> dk = to_dev(static_cast<const uint8_t*>(kpool), pool, st), dv = to_dev(static_cast<const uint8_t*>(vpool), pool, st);
        DBuf<TO> dout;
        dout.alloc((size_t)M * Hq);
        double ctx_sum = 0;
        for (int i = 0; i < M; ++i) ctx_sum += ctx_len[active[i]];
        launch_attn_decode<T, TO>(dqkv.p, dact.p, M, dctx.p, dbt.p, mp, reinterpret_cast<T*>(dk.p), reinterpret_cast<T*>(dv.p),
                                  dout.p, heads, st, ctx_sum);
        dk.download(static_cast<uint8_t*>(kpool), pool, st); dv.download(static_cast<uint8_t*>(vpool), pool, st);
        download_f32(dout.p, type_code<TO>(), out, (size_t)M * Hq, st);
    });
}

// One beam step on caller arrays for one group of nb beams in slots 0..nb-1: logprob, select, reorder and the partial-page
// copy (launch_beam_step without the gather), every input and output on the host (include/xtts_b200.h)
void debug_beam_step(const HarnessCtx& c, int kv_type, int heads, int layers, int Vn, const xtts_sampling& sp,
                     const xtts_beam& bm, int first, int advance, const float* logits, int32_t* n_gen, int32_t* ctx_len,
                     int32_t* last_tok, uint32_t* seen, int mp, int32_t* block_tables, int n_pages, int32_t* pool, int cap,
                     int32_t* hist, xtts_beam_state* state, void* kpool, void* vpool, float* scores) {
    static_assert(sizeof(xtts_beam_state) == sizeof(BeamState), "xtts_beam_state mirrors BeamState");
    const int nb = bm.num_beams;
    auto bad = [](const char* m) { throw std::runtime_error(std::string("debug_beam_step: ") + m); };
    const size_t esz = with_kv(kv_type, "debug_beam_step: kv_type", [](auto* tag, auto*) { return sizeof(*tag); });
    if (nb < 2 || nb > kMaxBeams) bad("num_beams 2..8");
    if (heads < 1 || layers < 1 || Vn < 2 * nb || n_pages < 1 || cap < 1 || mp < 1) bad("empty problem");
    if (!beam_supported(Vn, mp, cap)) bad("geometry outside the beam kernels' limits");
    const int W = ceil_div(Vn, 32), pool_cap = nb * mp;
    BeamState bs;
    std::memcpy(&bs, state, sizeof(bs));
    if (bs.n_free < nb || bs.n_free > pool_cap) bad("the pool must hold nb .. nb * max_pages pages");
    check_pages(pool, bs.n_free, n_pages, "debug_beam_step: pool page outside the pool");
    // every beam that owns pages holds exactly those of its KV positions [0, L), L = ctx_len + advance; the pool and the
    // tables together never exceed nb * max_pages entries
    const int L = ctx_len[0] + advance;
    if (L < 1 || L / kPageTokens >= mp) bad("the next position must lie inside the block table");
    int held = 0;
    for (int j = 0; j < nb; ++j) {
        if (n_gen[j] != n_gen[0] || ctx_len[j] != ctx_len[0]) bad("the beams of a group share n_gen and ctx_len");
        const int np = first && j > 0 ? 0 : bs.n_pages[j];
        if (np != (first && j > 0 ? 0 : ceil_div(L, kPageTokens))) bad("n_pages must cover the KV positions [0, ctx_len + advance)");
        check_pages(block_tables + (size_t)j * mp, np, n_pages, "debug_beam_step: page id outside the pool");
        held += np;
    }
    if (held + bs.n_free > pool_cap) bad("pool and tables exceed nb * max_pages pages");
    if (n_gen[0] < 0 || n_gen[0] >= cap) bad("n_gen outside the history");
    const cudaStream_t st = c.st;
    const size_t page_bytes = (size_t)heads * kv_block_bytes((int)esz), pool_bytes = (size_t)layers * n_pages * page_bytes;
    BeamDesc d{};
    d.primary = 0; d.nb = nb; d.first = first != 0; d.advance = advance; d.do_sample = bm.do_sample != 0;
    d.length_penalty = bm.length_penalty;
    for (int j = 0; j < kMaxBeams; ++j) { d.slot[j] = j < nb ? j : -1; d.row[j] = j < nb ? (first ? 0 : j) : 0; }
    DBuf<int> dng = to_dev(n_gen, nb, st), dctx = to_dev(ctx_len, nb, st), dlast, dfin, dtok,
              dbt = to_dev(block_tables, (size_t)nb * mp, st), dpool = to_dev(pool, pool_cap, st);
    dlast.alloc(nb); dfin.alloc(nb); dtok.alloc((size_t)nb * cap);
    dfin.zero(st); dtok.zero(st);
    DBuf<float> dlog, dsc;
    dlog.alloc((size_t)nb * Vn); dsc.alloc((size_t)nb * Vn);
    dlog.upload(logits, (size_t)(first ? 1 : nb) * Vn, st);
    DBuf<unsigned> dseen = to_dev(seen, (size_t)nb * W, st);
    DBuf<BeamState> dstate = to_dev(&bs, 1, st);
    DBuf<BeamDesc> ddesc = to_dev(&d, 1, st);
    DBuf<int2> dhist = to_dev(reinterpret_cast<const int2*>(hist), (size_t)cap * kMaxBeams, st);
    DBuf<uint8_t> dk = to_dev(static_cast<const uint8_t*>(kpool), pool_bytes, st), dv = to_dev(static_cast<const uint8_t*>(vpool), pool_bytes, st);
    std::vector<void*> ptr(2 * layers);
    for (int l = 0; l < layers; ++l) { ptr[l] = dk.p + l * n_pages * page_bytes; ptr[layers + l] = dv.p + l * n_pages * page_bytes; }
    DBuf<void*> dptr = to_dev(ptr.data(), 2 * layers, st);
    Sampling smp = upload_sampling(&sp, nb, true, st);
    SampleState& S = smp.S;
    S.last_tok = dlast.p; S.n_gen = dng.p; S.ctx_len = dctx.p; S.finished = dfin.p; S.tokens = dtok.p; S.seen = dseen.p;
    S.tokens_cap = cap; S.seen_words = W;
    BeamArgs a{};
    a.desc = ddesc.p; a.n_groups = 1; a.state = dstate.p; a.hist = dhist.p; a.pool = dpool.p; a.pool_cap = pool_cap;
    a.scores = dsc.p; a.block_tables = dbt.p; a.max_pages = mp; a.latents = nullptr; a.H = 0;
    launch_beam_step(dlog.p, Vn, Vn, S, a, dptr.p, dptr.p + layers, layers, heads, (int)esz, st, false);
    dng.download(n_gen, nb, st); dctx.download(ctx_len, nb, st); dlast.download(last_tok, nb, st);
    dseen.download(seen, (size_t)nb * W, st); dbt.download(block_tables, (size_t)nb * mp, st); dpool.download(pool, pool_cap, st);
    dstate.download(&bs, 1, st); dhist.download(reinterpret_cast<int2*>(hist), (size_t)cap * kMaxBeams, st);
    dk.download(static_cast<uint8_t*>(kpool), pool_bytes, st); dv.download(static_cast<uint8_t*>(vpool), pool_bytes, st);
    dsc.download(scores, (size_t)nb * Vn, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::memcpy(state, &bs, sizeof(bs));
}

// One launch of the prefill / encoder attention (launch_attn_generic).  q rows and k / v rows are addressed with the given
// strides (k at kv + k_off, v at kv + v_off); out is [out_rows][heads * 64], rows no sequence covers keep their NaN fill.
void debug_attn_prefill(const HarnessCtx& c, int out_type, int heads, const int32_t* seqs, int nseq, int causal, float scale,
                        const float* q, int64_t q_len, int q_row_stride, int q_head_stride, const float* kv, int64_t kv_len,
                        int kv_row_stride, int kv_head_stride, int64_t k_off, int64_t v_off, float* out, int out_rows) {
    with_elem(out_type, "debug_attn_prefill: out_type", [&](auto* tag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        if (heads < 1 || nseq < 1 || out_rows < 1 || q_len < 1 || kv_len < 1) throw std::runtime_error("debug_attn_prefill: empty problem");
        const int Hq = heads * kHeadDim;
        int max_nq = 0;
        auto last = [&](int64_t row, int64_t rs, int64_t hs) { return row * rs + (int64_t)(heads - 1) * hs + kHeadDim - 1; };
        for (int i = 0; i < nseq; ++i) {
            const int32_t* s = seqs + 4 * i;        // q_start, nq, kv_start, nk
            if (s[0] < 0 || s[1] < 1 || s[2] < 0 || s[3] < 1 || s[0] + s[1] > out_rows)
                throw std::runtime_error("debug_attn_prefill: sequence outside the output rows");
            if (causal && s[3] < s[1]) throw std::runtime_error("debug_attn_prefill: causal attention needs nk >= nq");
            if (last(s[0] + s[1] - 1, q_row_stride, q_head_stride) >= q_len ||
                std::max(k_off, v_off) + last(s[2] + s[3] - 1, kv_row_stride, kv_head_stride) >= kv_len || std::min(k_off, v_off) < 0)
                throw std::runtime_error("debug_attn_prefill: sequence outside the q / kv buffers");
            max_nq = std::max(max_nq, (int)s[1]);
        }
        const cudaStream_t st = c.st;
        const size_t n_out = (size_t)out_rows * Hq;
        DBuf<float> dq = to_dev(q, q_len, st), dkv = to_dev(kv, kv_len, st);
        DBuf<AttnSeq> dseq = to_dev(reinterpret_cast<const AttnSeq*>(seqs), nseq, st);
        DBuf<T> dout;
        dout.alloc(n_out);
        CUDA_CHECK(cudaMemsetAsync(dout.p, 0xFF, n_out * sizeof(T), st));        // NaN in every output type
        AttnLayout A;
        A.q = dq.p; A.k = dkv.p + k_off; A.v = dkv.p + v_off;
        A.q_row_stride = q_row_stride; A.kv_row_stride = kv_row_stride; A.q_head_stride = q_head_stride; A.kv_head_stride = kv_head_stride;
        A.heads = heads; A.scale = scale; A.causal = causal ? 1 : 0;
        launch_attn_generic<T>(A, dseq.p, nseq, max_nq, dout.p, Hq, st);
        download_f32(dout.p, out_type, out, n_out, st);
    });
}

// The decode step's split-K projection + residual / LayerNorm pair, as layers_forward runs it: the 16-bit GEMM into fp32
// partials, then X += bias + sum of the partials and Y = LN(X) (Y skipped without ln_w / ln_b: the last layer's form).
void debug_splitk_ln(const HarnessCtx& c, int mode, int M, int N, int K, int splits, const float* A, const float* W,
                     const float* bias, float* X, const float* ln_w, const float* ln_b, float* Y) {
    if (mode != 1 && mode != 2) throw std::runtime_error("debug_splitk_ln: mode 1 (bf16) or 2 (fp16)");
    if (M < 1 || N < 32 || N % 32 != 0 || N > 8192 || K < 64 || K % 64 != 0 || splits < 1 || splits > 8 || (K / 64) % splits != 0)
        throw std::runtime_error("debug_splitk_ln: need N % 32 == 0 (<= 8192), K % 64 == 0, 1 <= splits <= 8 dividing K / 64");
    if (!bias || (ln_w == nullptr) != (ln_b == nullptr) || (ln_w && !Y)) throw std::runtime_error("debug_splitk_ln: bias, and ln_w / ln_b / Y together");
    std::string err;
    if (!gemm_tc_init(&err)) throw std::runtime_error(err);
    const cudaStream_t st = c.st;
    DBuf<float> dA = to_dev(A, (size_t)M * K, st), dW = to_dev(W, (size_t)N * K, st), db = to_dev(bias, N, st),
                dX = to_dev(X, (size_t)M * N, st), dlw = to_dev(ln_w, N, st), dlb = to_dev(ln_b, N, st), dpart;
    dpart.alloc((size_t)splits * M * N);
    DBuf<__nv_bfloat16> hA, hW, dY;                 // 16-bit operands / output (IEEE fp16 bits in mode 2)
    hA.alloc((size_t)M * K); hW.alloc((size_t)N * K);
    if (ln_w) dY.alloc((size_t)M * N);
    to16(mode, dA.p, hA.p, (size_t)M * K, st); to16(mode, dW.p, hW.p, (size_t)N * K, st);
    launch_gemm_bf16_tc_splitk(hA.p, hW.p, dpart.p, M, N, K, splits, st, false, mode == 2 ? GEMM_F16 : 0);
    with_elem(mode, "debug_splitk_ln: mode", [&](auto* tag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        launch_residual_reduce_layernorm<T>(dX.p, dpart.p, splits, db.p, dlw.p, dlb.p, reinterpret_cast<T*>(dY.p), M, N, c.ln_eps, st);
    });
    dX.download(X, (size_t)M * N, st);
    if (ln_w) download_f32(dY.p, mode, Y, (size_t)M * N, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// The decode step's LayerNorm -> GEMM pair as decode_layers_rows launches it: the 16-bit LayerNorm into the operand buffer,
// then the one-tile GEMM on it.  launch 0: plain launches; 1: both with PDL.
void debug_ln_gemm(const HarnessCtx& c, int mode, int launch, int M, int N, int K, const float* X, const float* ln_w,
                   const float* ln_b, const float* W, const float* bias, const float* resid, int dflags, float* Y, float* out) {
    if (mode != 1 && mode != 2) throw std::runtime_error("debug_ln_gemm: mode 1 (bf16) or 2 (fp16)");
    if (launch < 0 || launch > 1) throw std::runtime_error("debug_ln_gemm: launch 0 (plain) or 1 (PDL)");
    if (M < 1 || N < 32 || N % 32 != 0 || K < 64 || K % 64 != 0 || K > 8192) throw std::runtime_error("debug_ln_gemm: need M >= 1, N % 32 == 0, K % 64 == 0 (<= 8192)");
    if (dflags & ~(XTTS_DEBUG_GEMM_GELU | XTTS_DEBUG_GEMM_OUT16)) throw std::runtime_error("debug_ln_gemm: flags GELU / OUT16 only");
    if (!X || !ln_w || !ln_b || !W || !Y || !out) throw std::runtime_error("debug_ln_gemm: only bias and resid may be NULL");
    if (resid && (dflags & XTTS_DEBUG_GEMM_OUT16)) throw std::runtime_error("debug_ln_gemm: a residual needs fp32 output");
    std::string err;
    if (!gemm_tc_init(&err)) throw std::runtime_error(err);
    const cudaStream_t st = c.st;
    const bool out16 = dflags & XTTS_DEBUG_GEMM_OUT16;
    DBuf<float> dX = to_dev(X, (size_t)M * K, st), dlw = to_dev(ln_w, K, st), dlb = to_dev(ln_b, K, st),
                dW = to_dev(W, (size_t)N * K, st), db = to_dev(bias, N, st), dr = to_dev(resid, (size_t)M * N, st), dout;
    DBuf<__nv_bfloat16> hW, dY, dout16;
    hW.alloc((size_t)N * K); dY.alloc((size_t)M * K);
    if (out16) dout16.alloc((size_t)M * N); else dout.alloc((size_t)M * N);
    to16(mode, dW.p, hW.p, (size_t)N * K, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
    const bool pdl = launch == 1;
    with_elem(mode, "debug_ln_gemm: mode", [&](auto* tag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        launch_layernorm<T>(dX.p, dlw.p, dlb.p, reinterpret_cast<T*>(dY.p), M, K, c.ln_eps, st, pdl);
    });
    const int flags = ((dflags & XTTS_DEBUG_GEMM_GELU) ? GEMM_GELU : 0) | (out16 ? GEMM_OUT_BF16 : 0) | (resid ? GEMM_RESID : 0) |
                      (mode == 2 ? GEMM_F16 : 0);
    void* op = out16 ? (void*)dout16.p : (void*)dout.p;
    launch_gemm_bf16_tc(dY.p, hW.p, db.p, dr.p, op, M, N, K, flags, st, pdl);
    download_f32(dY.p, mode, Y, (size_t)M * K, st);
    download_f32(op, out16 ? mode : 0, out, (size_t)M * N, st);
}

// launch_layernorm (w2 == NULL) or launch_head_norms (w2 != NULL) in the output type `out_type` on private buffers
void debug_norms(const HarnessCtx& c, int out_type, int M, int H, const float* X, int x_rows, const int32_t* row_index,
                 const float* w1, const float* b1, const float* w2, const float* b2, float* Y, float* latents, int n_slots,
                 int lat_rows, const int32_t* slots, const int32_t* lat_pos, const int32_t* n_gen) {
    with_elem(out_type, "debug_norms: out_type", [&](auto* tag) {
        using T = std::remove_pointer_t<decltype(tag)>;
        if (M < 1 || H < 1 || H > 8192 || x_rows < 1) throw std::runtime_error("debug_norms: need M >= 1, 1 <= H <= 8192, x_rows >= 1");
        if (!X || !w1 || !b1 || !Y || (w2 == nullptr) != (b2 == nullptr)) throw std::runtime_error("debug_norms: X, w1, b1, Y, and w2 / b2 together");
        const bool head = w2 != nullptr;
        if (!head && (row_index || latents || x_rows < M)) throw std::runtime_error("debug_norms: a plain LayerNorm reads rows 0 .. M-1 and has no latents");
        if (row_index)
            for (int i = 0; i < M; ++i)
                if (row_index[i] < 0 || row_index[i] >= x_rows) throw std::runtime_error("debug_norms: row_index outside X");
        if (!row_index && x_rows < M) throw std::runtime_error("debug_norms: X has fewer than M rows");
        if (latents) {
            if (!slots || n_slots < 1 || lat_rows < 1 || (!lat_pos && !n_gen)) throw std::runtime_error("debug_norms: latents need slots, n_slots, lat_rows and lat_pos or n_gen");
            for (int i = 0; i < M; ++i)
                if (slots[i] < 0 || slots[i] >= n_slots) throw std::runtime_error("debug_norms: slot outside n_slots");
        }
        const cudaStream_t st = c.st;
        const size_t nlat = latents ? (size_t)n_slots * lat_rows * H : 0;
        DBuf<float> dX = to_dev(X, (size_t)x_rows * H, st), dw1 = to_dev(w1, H, st), db1 = to_dev(b1, H, st),
                    dw2 = to_dev(w2, H, st), db2 = to_dev(b2, H, st), dlat = to_dev(latents, nlat, st);
        DBuf<int> dri = to_dev(row_index, M, st), dsl = to_dev(latents ? slots : nullptr, M, st),
                  dlp = to_dev(latents ? lat_pos : nullptr, M, st), dng = to_dev(latents ? n_gen : nullptr, n_slots, st);
        DBuf<T> dY;
        dY.alloc((size_t)M * H);
        if (!head) launch_layernorm<T>(dX.p, dw1.p, db1.p, dY.p, M, H, c.ln_eps, st);
        else launch_head_norms<T>(dX.p, dri.p, dw1.p, db1.p, dw2.p, db2.p, dY.p, dlat.p, dsl.p, dlp.p, dng.p, lat_rows, M, H,
                                  c.ln_eps, st);
        if (latents) dlat.download(latents, nlat, st);
        download_f32(dY.p, out_type, Y, (size_t)M * H, st);
    });
}

// launch_kv_write (the prefill's paged-cache write) over raw pools in the device layout, updated in place
void debug_kv_write(const HarnessCtx& c, int kv_type, int heads, int M, const float* qkv, const int32_t* row_slot,
                    const int32_t* row_pos, int n_slots, const int32_t* ctx_len, const int32_t* block_tables, int mp,
                    int n_pages, void* kpool, void* vpool) {
    with_kv(kv_type, "debug_kv_write: kv_type", [&](auto* tag, auto*) {
        using T = std::remove_pointer_t<decltype(tag)>;
        if (heads < 1 || M < 1 || n_slots < 1 || mp < 1 || n_pages < 1) throw std::runtime_error("debug_kv_write: empty problem");
        if (!qkv || !row_slot || !block_tables || !kpool || !vpool || (!row_pos && !ctx_len)) throw std::runtime_error("debug_kv_write: row_pos or ctx_len, and every other pointer");
        for (int r = 0; r < M; ++r) {
            const int s = row_slot[r];
            if (s < 0 || s >= n_slots) throw std::runtime_error("debug_kv_write: row slot outside n_slots");
            const int pos = row_pos ? row_pos[r] : ctx_len[s];
            if (pos < 0 || pos / kPageTokens >= mp) throw std::runtime_error("debug_kv_write: position outside the block table");
            check_pages(block_tables + (size_t)s * mp + pos / kPageTokens, 1, n_pages, "debug_kv_write: page id outside the pool");
        }
        const cudaStream_t st = c.st;
        const size_t pool = (size_t)n_pages * heads * kv_block_bytes(sizeof(T)), Hq = (size_t)heads * kHeadDim;
        DBuf<int> dslot = to_dev(row_slot, M, st), dpos = to_dev(row_pos, M, st), dctx = to_dev(ctx_len, n_slots, st),
                  dbt = to_dev(block_tables, (size_t)n_slots * mp, st);
        DBuf<float> dqkv = to_dev(qkv, (size_t)M * 3 * Hq, st);
        DBuf<uint8_t> dk = to_dev(static_cast<const uint8_t*>(kpool), pool, st), dv = to_dev(static_cast<const uint8_t*>(vpool), pool, st);
        launch_kv_write<T>(dqkv.p, M, dslot.p, dpos.p, dctx.p, dbt.p, mp, reinterpret_cast<T*>(dk.p), reinterpret_cast<T*>(dv.p), heads, st);
        dk.download(static_cast<uint8_t*>(kpool), pool, st); dv.download(static_cast<uint8_t*>(vpool), pool, st);
        CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

// launch_build_rows over private embedding tables: rows [n_rows][4] = RowDesc (kind, a, b, c)
void debug_build_rows(const HarnessCtx& c, int Hd, int n_cond, const float* text_emb, int n_text, const float* text_pos,
                      int n_tpos, const float* wte, int n_audio, const float* wpe, int n_wpe, const float* spk, int n_spk,
                      const int32_t* rows, int n_rows, float* X) {
    if (Hd < 4 || Hd % 4 != 0 || n_rows < 1 || n_cond < 1 || n_text < 1 || n_tpos < 1 || n_audio < 1 || n_wpe < 1 || n_spk < 1)
        throw std::runtime_error("debug_build_rows: need H % 4 == 0 and non-empty tables and rows");
    if (!text_emb || !text_pos || !wte || !wpe || !spk || !rows || !X) throw std::runtime_error("debug_build_rows: NULL argument");
    for (int i = 0; i < n_rows; ++i) {
        const int32_t* r = rows + 4 * i;
        const bool ok = r[0] == 0 ? (r[1] >= 0 && r[1] < n_cond && r[3] >= 0 && r[3] < n_spk)
                      : r[0] == 1 ? (r[1] >= 0 && r[1] < n_text && r[2] >= 0 && r[2] < n_tpos)
                      : r[0] == 2 ? (r[1] >= 0 && r[1] < n_audio && r[2] >= 0 && r[2] < n_wpe) : false;
        if (!ok) throw std::runtime_error("debug_build_rows: row kind outside 0..2 or index outside its table");
    }
    const cudaStream_t st = c.st;
    static_assert(sizeof(RowDesc) == 4 * sizeof(int32_t), "RowDesc crosses the ABI as four int32");
    DBuf<float> dte = to_dev(text_emb, (size_t)n_text * Hd, st), dtp = to_dev(text_pos, (size_t)n_tpos * Hd, st),
                dwte = to_dev(wte, (size_t)n_audio * Hd, st), dwpe = to_dev(wpe, (size_t)n_wpe * Hd, st),
                dspk = to_dev(spk, (size_t)n_spk * n_cond * Hd, st), dX;
    dX.alloc((size_t)n_rows * Hd);
    DBuf<RowDesc> drows = to_dev(reinterpret_cast<const RowDesc*>(rows), n_rows, st);
    GptTables t; t.text_emb = dte.p; t.text_pos = dtp.p; t.wte = dwte.p; t.wpe = dwpe.p; t.spk_cond = dspk.p; t.H = Hd; t.n_cond = n_cond;
    launch_build_rows(drows.p, n_rows, t, dX.p, st);
    dX.download(X, (size_t)n_rows * Hd, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// launch_build_decode_rows over private tables and slot arrays
void debug_build_decode_rows(const HarnessCtx& c, int Hd, const float* wte, int n_audio, const float* wpe, int n_wpe, int M,
                             const int32_t* active, int n_slots, const int32_t* last_tok, const int32_t* n_gen, float* X) {
    if (Hd < 4 || Hd % 4 != 0 || M < 1 || n_slots < 1 || n_audio < 1 || n_wpe < 1) throw std::runtime_error("debug_build_decode_rows: need H % 4 == 0, M >= 1 and non-empty tables");
    if (!wte || !wpe || !active || !last_tok || !n_gen || !X) throw std::runtime_error("debug_build_decode_rows: NULL argument");
    for (int i = 0; i < M; ++i) {
        const int s = active[i];
        if (s < 0 || s >= n_slots) throw std::runtime_error("debug_build_decode_rows: active slot outside n_slots");
        if (last_tok[s] < 0 || last_tok[s] >= n_audio || n_gen[s] < 0 || n_gen[s] >= n_wpe)
            throw std::runtime_error("debug_build_decode_rows: last_tok / n_gen outside the tables");
    }
    const cudaStream_t st = c.st;
    DBuf<float> dwte = to_dev(wte, (size_t)n_audio * Hd, st), dwpe = to_dev(wpe, (size_t)n_wpe * Hd, st), dX;
    dX.alloc((size_t)M * Hd);
    DBuf<int> dact = to_dev(active, M, st), dlast = to_dev(last_tok, n_slots, st), dng = to_dev(n_gen, n_slots, st);
    GptTables t{}; t.wte = dwte.p; t.wpe = dwpe.p; t.H = Hd;
    launch_build_decode_rows(dact.p, M, dlast.p, dng.p, t, dX.p, st, c.pdl);
    dX.download(X, (size_t)M * Hd, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// One launch of the fast-mode vocoder convolution (launch_conv1d_tc, or launch_convT_tc for up > 0) with the weights
// packed and planned as make_conv does.  The input atom image is NaN except each item's signal rows; the production pad
// routine then clears what it claims the kernel reads, so any other read reaches a stored output as NaN.  out32 / out16
// are in/out: their incoming contents are the accumulate base and the sentinels of every row the kernel must not write.
void debug_conv_tc(const HarnessCtx& c, int up, int Cin, int Cout, int K, int dil, int batch, int L, const int32_t* item_len,
                   const float* w, const float* bias, const float* cbias, int cbias_stride, const float* x, const float* resid,
                   int mode, float slope_out, float scale16, int max_ctas, float* out32, float* out16) {
    if (up != 0 && up != 2 && up != 4 && up != 8) throw std::runtime_error("debug_conv_tc: up 0 (Conv1d) or 2, 4, 8 (ConvTranspose1d)");
    if (up == 0 && (K < 1 || K % 2 == 0 || dil < 1)) throw std::runtime_error("debug_conv_tc: Conv1d needs an odd K and dil >= 1");
    if (up > 0 && (K != 2 * up || dil != 1)) throw std::runtime_error("debug_conv_tc: ConvTranspose1d needs K = 2 * up and dil = 1");
    if (up > 0 && (resid || mode != CONV_STORE || scale16 != 1.0f))
        throw std::runtime_error("debug_conv_tc: ConvTranspose1d takes no resid, mode STORE and scale16 1");
    if (mode != CONV_STORE && mode != CONV_ACCUM) throw std::runtime_error("debug_conv_tc: mode 0 (store) or 1 (accumulate)");
    if (mode == CONV_ACCUM && !out32) throw std::runtime_error("debug_conv_tc: accumulate mode needs out32");
    if (up == 0 && (K - 1) / 2 * dil > kAtomPadL) throw std::runtime_error("debug_conv_tc: halo (K-1)/2*dil exceeds the atom head pad");
    if (batch < 1 || batch > kVocMaxItems) throw std::runtime_error("debug_conv_tc: batch must be 1..32");
    if (L < 1) throw std::runtime_error("debug_conv_tc: L must be >= 1");
    if (!w) throw std::runtime_error("debug_conv_tc: w is required");
    if (!x) throw std::runtime_error("debug_conv_tc: x is required");
    std::vector<int> lens(batch, L);
    for (int i = 0; i < batch && item_len; ++i) {
        if (item_len[i] < 0 || item_len[i] > L) throw std::runtime_error("debug_conv_tc: item_len must lie in [0, L]");
        lens[i] = item_len[i];
    }
    if (Cin < 1 || Cout < 1) throw std::runtime_error("debug_conv_tc: empty channel count");
    const ConvTcPlan pl = up ? conv1d_tc_plan(Cin, up * Cout, 2) : conv1d_tc_plan(Cin, Cout, K);
    if (!pl.ok) throw std::runtime_error("debug_conv_tc: no tensor-core plan for these channel counts");
    if (up > 0 && Cout % 32 != 0) throw std::runtime_error("debug_conv_tc: ConvTranspose1d needs Cout % 32 == 0");
    if (out16 && Cout % 8 != 0) throw std::runtime_error("debug_conv_tc: out16 needs Cout % 8 == 0");
    if (cbias && cbias_stride < Cout) throw std::runtime_error("debug_conv_tc: cbias_stride < Cout");
    if (max_ctas < 0) throw std::runtime_error("debug_conv_tc: max_ctas must be >= 0");
    const cudaStream_t st = c.st;
    const int Lout = up ? L * up : L, lpad = atoms_lpad(L), lpad_out = atoms_lpad(Lout);
    std::vector<__half> blob(pl.blob_halves);
    if (up) convT_tc_pack(w, Cin, Cout, up, pl, blob.data());
    else conv1d_tc_pack(w, Cin, Cout, K, pl, blob.data());
    __half_raw nan_raw; nan_raw.x = 0x7e00;
    const size_t n_in = (size_t)batch * Cin * lpad, n32 = (size_t)batch * Cout * Lout, n16 = (size_t)batch * Cout * lpad_out;
    std::vector<__half> a(n_in, __half(nan_raw));
    for (int b = 0; b < batch; ++b)
        for (int ch = 0; ch < Cin; ++ch)
            for (int t = 0; t < lens[b]; ++t)
                a[(((size_t)b * (Cin / 8) + ch / 8) * lpad + kAtomPadL + t) * 8 + ch % 8] = __float2half_rn(x[((size_t)b * Cin + ch) * L + t]);
    std::vector<__half> o16(out16 ? n16 : 0);
    for (size_t i = 0; i < o16.size(); ++i) o16[i] = __float2half_rn(out16[i]);
    DBuf<__half> da = to_dev(a.data(), n_in, st), dblob = to_dev(blob.data(), blob.size(), st),
                 do16 = to_dev(out16 ? o16.data() : nullptr, n16, st);
    DBuf<float> dbias = to_dev(bias, Cout, st), dcb = to_dev(cbias, (size_t)batch * cbias_stride, st),
                dres = to_dev(resid, n32, st), do32 = to_dev(out32, n32, st);
    launch_atoms_zero_pads(da.p, batch * Cin / 8, lpad, L, st, batch, lens.data());
    const int* il = item_len ? lens.data() : nullptr;
    struct CapRestore { int& cap; int prev; ~CapRestore() { cap = prev; } } restore{g_voc_sm_cap, g_voc_sm_cap};
    g_voc_sm_cap = max_ctas;
    if (up)
        launch_convT_tc(da.p, dblob.p, pl, dbias.p, dcb.p, do32.p, do16.p, Cin, Cout, L, lpad, lpad_out, up, slope_out, batch,
                        cbias_stride, st, il);
    else
        launch_conv1d_tc(da.p, dblob.p, pl, dbias.p, dcb.p, dres.p, do32.p, do16.p, Cin, Cout, L, lpad, K, dil, slope_out,
                         scale16, mode, batch, cbias_stride, st, il);
    if (out32) do32.download(out32, n32, st);
    if (out16) download_f32(do16.p, 2, out16, n16, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// One vocoder ResBlock1 of C channels on host data, through the fused kernel (launch_resblock_tc) or through the six
// launch_conv1d_tc calls it replaces, issued as Engine::run_vocoder_tc issues them.  Weights w [6][C][C][K] and biases
// [6][C] in the order c1_0, c2_0, c1_1, c2_1, c1_2, c2_2.  The input atoms are lrelu(x, 0.1) as fp16, NaN outside each
// item's signal until the production pad routine clears its pads (the six-launch workspaces too), and the fp32 rows past
// an item's length are NaN: a read of anything else reaches a stored output as NaN.  zs / pa are in/out as in
// debug_conv_tc.
void debug_resblock_tc(const HarnessCtx& c, int C, int K, const int32_t* dil, int batch, int L, const int32_t* item_len,
                       const float* w, const float* bias, const float* x, int mode, float scale16, int max_ctas, int fused,
                       float* zs, float* pa) {
    if (!dil || !w || !bias || !x || !zs) throw std::runtime_error("debug_resblock_tc: dil, w, bias, x and zs are required");
    if (fused && resblock_tc_tile_rows(C, K, dil, L) == 0)
        throw std::runtime_error("debug_resblock_tc: fused needs C 32 or 64, K odd, dilations >= 1 and a halo that is a multiple of 4 and fits the tile");
    if (!fused && (C % 8 != 0 || K % 2 == 0 || dil[0] < 1 || dil[1] < 1 || dil[2] < 1 || !conv1d_tc_plan(C, C, K).ok))
        throw std::runtime_error("debug_resblock_tc: no tensor-core plan for these channel counts, an even K or a dilation < 1");
    if (mode != CONV_STORE && mode != CONV_ACCUM) throw std::runtime_error("debug_resblock_tc: mode 0 (store) or 1 (accumulate)");
    if (batch < 1 || batch > kVocMaxItems) throw std::runtime_error("debug_resblock_tc: batch must be 1..32");
    if (L < 4 || L % 4 != 0) throw std::runtime_error("debug_resblock_tc: L must be a positive multiple of 4");
    if (max_ctas < 0) throw std::runtime_error("debug_resblock_tc: max_ctas must be >= 0");
    for (int t = 0; t < 3; ++t)
        if ((K - 1) / 2 * dil[t] > kAtomPadL) throw std::runtime_error("debug_resblock_tc: halo (K-1)/2*dil exceeds the atom head pad");
    std::vector<int> lens(batch, L);
    for (int i = 0; i < batch && item_len; ++i) {
        if (item_len[i] < 0 || item_len[i] > L) throw std::runtime_error("debug_resblock_tc: item_len must lie in [0, L]");
        lens[i] = item_len[i];
    }
    const cudaStream_t st = c.st;
    const int lpad = atoms_lpad(L), PL = C / 8;
    const ConvTcPlan pl = conv1d_tc_plan(C, C, K);
    std::vector<__half> blob(6 * pl.blob_halves);
    for (int i = 0; i < 6; ++i) conv1d_tc_pack(w + (size_t)i * C * C * K, C, C, K, pl, blob.data() + i * pl.blob_halves);
    __half_raw nan_raw; nan_raw.x = 0x7e00;
    const size_t n32 = (size_t)batch * C * L, n16 = (size_t)batch * C * lpad;
    std::vector<__half> a(n16, __half(nan_raw));
    std::vector<float> x32(n32, std::numeric_limits<float>::quiet_NaN());
    for (int b = 0; b < batch; ++b)
        for (int ch = 0; ch < C; ++ch)
            for (int t = 0; t < lens[b]; ++t) {
                const float v = x[((size_t)b * C + ch) * L + t];
                x32[((size_t)b * C + ch) * L + t] = v;
                a[(((size_t)b * PL + ch / 8) * lpad + kAtomPadL + t) * 8 + ch % 8] = __float2half_rn(v > 0.f ? v : v * 0.1f);
            }
    std::vector<__half> o16(pa ? n16 : 0);
    for (size_t i = 0; i < o16.size(); ++i) o16[i] = __float2half_rn(pa[i]);
    DBuf<__half> dxa = to_dev(a.data(), n16, st), dblob = to_dev(blob.data(), blob.size(), st),
                 dpa = to_dev(pa ? o16.data() : nullptr, n16, st);
    DBuf<float> dx = to_dev(x32.data(), n32, st), dzs = to_dev(zs, n32, st), dbias = to_dev(bias, (size_t)6 * C, st);
    const int* il = item_len ? lens.data() : nullptr;
    launch_atoms_zero_pads(dxa.p, batch * PL, lpad, L, st, batch, lens.data());
    struct CapRestore { int& cap; int prev; ~CapRestore() { cap = prev; } } restore{g_voc_sm_cap, g_voc_sm_cap};
    g_voc_sm_cap = max_ctas;
    const __half* wb[6]; const float* bs[6];
    for (int i = 0; i < 6; ++i) { wb[i] = dblob.p + i * pl.blob_halves; bs[i] = dbias.p + (size_t)i * C; }
    if (fused) {
        launch_resblock_tc(dxa.p, dx.p, wb, bs, dzs.p, dpa.p, C, L, lpad, K, dil, mode, scale16, batch, il, st);
    } else {
        DBuf<__half> ta = to_dev(a.data(), n16, st), ra0 = to_dev(a.data(), n16, st), ra1 = to_dev(a.data(), n16, st);
        DBuf<float> r[2];
        for (auto& rr : r) rr = to_dev(x32.data(), n32, st);
        for (__half* b : {ta.p, ra0.p, ra1.p}) launch_atoms_zero_pads(b, batch * PL, lpad, L, st, batch, lens.data());
        const __half* in16 = dxa.p;
        const float* resid = dx.p;
        __half* ra[2] = {ra0.p, ra1.p};
        for (int t = 0; t < 3; ++t) {
            launch_conv1d_tc(in16, wb[2 * t], pl, bs[2 * t], nullptr, nullptr, nullptr, ta.p, C, C, L, lpad, K, dil[t], 0.1f,
                             1.0f, CONV_STORE, batch, 0, st, il);
            if (t < 2) {
                launch_conv1d_tc(ta.p, wb[2 * t + 1], pl, bs[2 * t + 1], nullptr, resid, r[t].p, ra[t], C, C, L, lpad, K, 1, 0.1f,
                                 1.0f, CONV_STORE, batch, 0, st, il);
                in16 = ra[t]; resid = r[t].p;
            } else {
                launch_conv1d_tc(ta.p, wb[2 * t + 1], pl, bs[2 * t + 1], nullptr, resid, dzs.p, dpa.p, C, C, L, lpad, K, 1, 0.1f,
                                 scale16, mode, batch, 0, st, il);
            }
        }
        CUDA_CHECK(cudaStreamSynchronize(st));
    }
    dzs.download(zs, n32, st);
    if (pa) download_f32(dpa.p, 2, pa, n16, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// One launch of a CUDA-core vocoder kernel (launch_interp, launch_conv1d, launch_conv_transpose1d, launch_conv_post) on
// private buffers, as the engine's vocoder passes.  Op layouts: include/xtts_b200.h.
void debug_vocoder(const HarnessCtx& c, int op, const int32_t* dims, int n_dims, const float* scal, int n_scal,
                   const float* const* in, const int64_t* in_len, int n_in, float* out, int64_t out_len) {
    auto bad = [](const std::string& s) { return std::runtime_error("debug_vocoder: " + s); };
    static const int kBaseDims[XTTS_VOC_N_OPS] = {9, 11, 9, 6};
    if (op < 0 || op >= XTTS_VOC_N_OPS) throw bad("unknown op " + std::to_string(op));
    if (n_dims < kBaseDims[op] || !dims) throw bad("op " + std::to_string(op) + " takes at least " + std::to_string(kBaseDims[op]) + " dims");
    if ((n_scal && !scal) || (n_in > 0 && (!in || !in_len)) || !out) throw bad("NULL argument");
    const int batch = dims[op == XTTS_VOC_INTERP ? 1 : op == XTTS_VOC_CONV_POST ? 3 : 5];
    if (batch < 1 || batch > kVocMaxItems) throw bad("batch must be 1..32");
    const int want_dims = op == XTTS_VOC_INTERP ? 9 + 5 * batch : op == XTTS_VOC_CONV_POST && dims[5] ? 6 + batch : kBaseDims[op];
    const int want_scal = op == XTTS_VOC_INTERP ? batch : 2;
    if (n_dims != want_dims || n_scal != want_scal)
        throw bad("op " + std::to_string(op) + " takes " + std::to_string(want_dims) + " dims and " + std::to_string(want_scal) + " scalars");
    for (int i = 0; i < n_dims; ++i)
        if (dims[i] < 0) throw bad("negative dim");
    auto d = [&](int i) { return (int64_t)dims[i]; };
    auto pos = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (dims[i] < 1) throw bad("dim " + std::to_string(i) + " must be >= 1");
    };
    auto flag = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (dims[i] > 1) throw bad("dim " + std::to_string(i) + " is a flag: 0 or 1");
    };
    std::vector<int64_t> need;       // in_len each input must have
    int64_t need_out = 0, n16 = 0;   // n16: floats of the INTERP atom image at the end of out
    std::vector<InterpItem> items;
    switch (op) {
    case XTTS_VOC_INTERP: {          // C, batch, Lz, atoms, lpad, code_stride, hop, in_sr, out_sr, [T, T0, T1, z0, nz] x batch
        pos({0, 2, 5, 6, 7, 8});
        flag({3});
        if (d(3) && (d(0) % 8 != 0 || d(4) < kAtomPadL + d(2))) throw bad("the atom image needs C % 8 == 0 and lpad >= 64 + Lz");
        for (int i = 0; i < batch; ++i) {
            const int32_t* it = dims + 9 + 5 * i;
            const float r0 = scal[i];
            if (it[0] < 1 || it[2] < 1) throw bad("item " + std::to_string(i) + ": T and T1 must be >= 1");
            if (!(r0 >= 0.f) || r0 > 1e4f || (r0 > 0.f && it[1] < 1)) throw bad("item " + std::to_string(i) + ": r0 must be 0, or > 0 with T0 >= 1");
            if (it[4] > d(2)) throw bad("item " + std::to_string(i) + ": nz > Lz");
            InterpItem ii{nullptr, it[0], it[2], it[3], it[4]};
            ii.T0 = it[1]; ii.r0 = r0;
            items.push_back(ii);
            need.push_back(d(0) * it[0]);
        }
        n16 = d(3) ? batch * d(0) * d(4) : 0;
        need_out = batch * d(0) * d(2) + n16;
        break;
    }
    case XTTS_VOC_CONV1D:            // Cin, Cout, K, dil, L, batch, mode, has_bias, has_cbias, cbias_stride, has_resid
        pos({0, 1, 3, 4});
        flag({6, 7, 8, 10});
        if (d(2) != 3 && d(2) != 7 && d(2) != 11) throw bad("conv1d takes K 3, 7 or 11");
        if ((d(2) - 1) / 2 * d(3) > 64) throw bad("conv1d halo (K-1)/2*dil above 64");
        if (d(8) && d(9) < d(1)) throw bad("cbias_stride < Cout");
        need = {batch * d(0) * d(4), d(1) * d(0) * d(2)};
        if (d(7)) need.push_back(d(1));
        if (d(8)) need.push_back(batch * d(9));
        if (d(10)) need.push_back(batch * d(1) * d(4));
        need_out = batch * d(1) * d(4);
        break;
    case XTTS_VOC_CONV_T:            // Cin, Cout, u, K, Lin, batch, has_bias, has_cbias, cbias_stride
        pos({0, 1, 2, 4});
        flag({6, 7});
        if (d(3) != 2 * d(2) || d(2) % 2 != 0 || 128 % d(2) != 0 || d(2) > 32)
            throw bad("conv_transpose1d takes K = 2u with u even, dividing 128 and <= 32");
        if (d(7) && d(8) < d(1)) throw bad("cbias_stride < Cout");
        need = {batch * d(0) * d(4), d(0) * d(1) * d(3)};
        if (d(6)) need.push_back(d(1));
        if (d(7)) need.push_back(batch * d(8));
        need_out = batch * d(1) * d(4) * d(2);
        break;
    case XTTS_VOC_CONV_POST:         // Cin, K, L, batch, wav_stride, has_lens, [L_i] x batch
        pos({0, 1, 2});
        flag({5});
        if (d(1) % 2 == 0 || d(0) * d(1) > 12288) throw bad("conv_post takes an odd K with Cin * K <= 12288");
        if (d(4) < d(2)) throw bad("wav_stride < L");
        for (int i = 0; i < batch && d(5); ++i)
            if (d(6 + i) > d(2)) throw bad("item " + std::to_string(i) + ": length > L");
        need = {batch * d(0) * d(2), d(0) * d(1)};
        need_out = batch * d(4);
        break;
    }
    if (n_in != (int)need.size()) throw bad("op " + std::to_string(op) + " takes " + std::to_string(need.size()) + " inputs");
    for (int i = 0; i < n_in; ++i) {
        if (in_len[i] != need[i])
            throw bad("input " + std::to_string(i) + " has " + std::to_string(in_len[i]) + " floats, expected " + std::to_string(need[i]));
        if (!in[i]) throw bad("input " + std::to_string(i) + " is NULL");
    }
    if (out_len < 1 || out_len != need_out) throw bad("out has " + std::to_string(out_len) + " floats, expected " + std::to_string(need_out));

    const cudaStream_t st = c.st;
    std::vector<DBuf<float>> din(n_in);
    for (int i = 0; i < n_in; ++i) din[i] = to_dev(in[i], (size_t)in_len[i], st);
    auto I = [&](int i) -> const float* { return din[i].p; };
    const size_t n32 = (size_t)(out_len - n16);
    Guarded<uint32_t> o32(reinterpret_cast<const uint32_t*>(out), n32, st);
    float* o = reinterpret_cast<float*>(o32.p());
    const int* D = dims;
    DBuf<float> dw;                  // conv weights as the engine packs them
    switch (op) {
    case XTTS_VOC_INTERP: {
        std::vector<uint16_t> h16(n16);
        for (int64_t i = 0; i < n16; ++i) { const __half_raw r = __float2half_rn(out[n32 + i]); h16[i] = r.x; }
        Guarded<uint16_t> o16(h16.data(), h16.size(), st);
        for (int i = 0; i < batch; ++i) items[i].lat = I(i);
        launch_interp(items.data(), batch, o, D[3] ? reinterpret_cast<__half*>(o16.p()) : nullptr, D[4], D[0], D[2],
                      interp_scale1(D[5], D[6]), interp_scale2(D[7], D[8]), st);
        if (n16) {
            o16.fetch(h16.data(), st, "interp (atoms)");
            for (int64_t i = 0; i < n16; ++i) { __half_raw r; r.x = h16[i]; out[n32 + i] = __half2float(__half(r)); }
        }
        break;
    }
    case XTTS_VOC_CONV1D: {
        std::vector<float> wt(d(1) * d(0) * d(2));
        conv_weight_ckc(in[1], D[0], D[1], D[2], false, wt.data());
        dw = to_dev(wt.data(), wt.size(), st);
        int k = 2;
        const float* bias = D[7] ? I(k++) : nullptr;
        const float* cbias = D[8] ? I(k++) : nullptr;
        const float* resid = D[10] ? I(k++) : nullptr;
        launch_conv1d(I(0), dw.p, bias, cbias, resid, o, D[0], D[1], D[4], D[2], D[3], scal[0], scal[1], D[6], batch, D[9], st);
        break;
    }
    case XTTS_VOC_CONV_T: {
        std::vector<float> wt(d(0) * d(1) * d(3));
        conv_weight_ckc(in[1], D[0], D[1], D[3], true, wt.data());
        dw = to_dev(wt.data(), wt.size(), st);
        int k = 2;
        const float* bias = D[6] ? I(k++) : nullptr;
        const float* cbias = D[7] ? I(k++) : nullptr;
        launch_conv_transpose1d(I(0), dw.p, bias, cbias, o, D[0], D[1], D[4], D[3], D[2], scal[0], scal[1], batch, D[8], st);
        break;
    }
    case XTTS_VOC_CONV_POST:
        launch_conv_post(I(0), I(1), o, D[0], D[2], D[1], scal[0], scal[1], batch, st, D[5] ? D + 6 : nullptr, D[4]);
        break;
    }
    o32.fetch(reinterpret_cast<uint32_t*>(out), st, "op " + std::to_string(op));
}

}  // namespace xtts
