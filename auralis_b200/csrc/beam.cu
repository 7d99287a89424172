// Beam search on the device: transformers 5.5 GenerationMixin._beam_search (generation/utils.py:2876-3372) for one batch
// item per group, num_return_sequences 1, early_stopping unset — its selection, stop flags, finished-set merge and
// early-stop heuristic — plus the paged-KV fork that replaces its cache reorder.  Every kernel runs between two decode
// steps on the decode stream; the host learns that a group ended from the finished flag it already reads back.
#include "kernels.h"

namespace xtts {
namespace {

constexpr int BV = 2048;                 // vocabulary cap (the sampler's)
constexpr int kMaxTablePages = 128;      // block-table entries a group fork keeps in shared memory

// ------------------------------------------------------------------------------------------------
// one CTA per beam: log_softmax of the beam's logits row -> repetition penalty over prompt ∪ hypothesis ->
// (do_sample) temperature, top-k, top-p with min_tokens_to_keep 2 -> + the beam's running score
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
beam_logprob_kernel(const float* __restrict__ logits, int ld, int V, SampleState S, BeamArgs A) {
    __shared__ float zs[BV];
    __shared__ float sv[BV];
    __shared__ short si[BV];
    __shared__ float red[32];
    __shared__ float scan_part[256];
    const BeamDesc& d = A.desc[blockIdx.x / kMaxBeams];
    const int j = blockIdx.x % kMaxBeams;
    if (j >= d.nb) return;
    const int tid = threadIdx.x;
    const int slot = d.slot[j];
    const float* z = logits + (size_t)d.row[j] * ld;
    float mx = -INFINITY;
    for (int v = tid; v < V; v += 256) mx = fmaxf(mx, z[v]);
    mx = block_max(mx, red);
    float se = 0.f;
    for (int v = tid; v < V; v += 256) se += expf(z[v] - mx);
    const float lse = logf(block_sum(se, red));
    const float pen = S.penalty[slot];
    const unsigned* seen = S.seen + (size_t)slot * S.seen_words;
    for (int v = tid; v < BV; v += 256) {
        float x = -INFINITY;
        if (v < V) {
            x = (z[v] - mx) - lse;
            if ((seen[v >> 5] >> (v & 31)) & 1u) x = (x < 0.f) ? x * pen : x / pen;
        }
        zs[v] = x;
    }
    __syncthreads();
    if (d.do_sample) {
        const float T = S.temperature[slot];
        const int tk = S.top_k[slot];
        const float tp = S.top_p[slot];
        if (T > 0.f && T != 1.0f)
            for (int v = tid; v < V; v += 256) zs[v] = zs[v] / T;
        __syncthreads();
        // ascending bitonic sort of (value, index); the BV - V pads (-inf) go to the front
        for (int v = tid; v < BV; v += 256) { sv[v] = zs[v]; si[v] = (short)v; }
        __syncthreads();
        for (int k = 2; k <= BV; k <<= 1)
            for (int jj = k >> 1; jj > 0; jj >>= 1) {
                for (int t = tid; t < BV; t += 256) {
                    const int ixj = t ^ jj;
                    if (ixj > t) {
                        const float a = sv[t], b = sv[ixj];
                        const short ai = si[t], bi = si[ixj];
                        const bool sw = ((t & k) == 0) ? (b < a || (b == a && bi < ai)) : (a < b || (a == b && ai < bi));
                        if (sw) { sv[t] = b; si[t] = bi; sv[ixj] = a; si[ixj] = ai; }
                    }
                }
                __syncthreads();
            }
        // TopKLogitsWarper: keep >= the k-th largest, k = min(max(top_k, 2), V)
        if (tk > 0) {
            const int k = min(max(tk, 2), V);
            const float kth = sv[BV - k];
            __syncthreads();
            for (int v = tid; v < BV; v += 256) if (sv[v] < kth) sv[v] = -INFINITY;
            __syncthreads();
        }
        // TopPLogitsWarper: drop while the ascending cumulative softmax <= 1 - top_p, never the last 2
        if (tp < 1.0f) {
            const float smx = sv[BV - 1];
            float e[8], loc = 0.f;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const float x = sv[tid * 8 + u];
                e[u] = (x == -INFINITY) ? 0.f : expf(x - smx);
                loc += e[u];
            }
            const float total = block_sum(loc, red);
            scan_part[tid] = loc;
            __syncthreads();
            for (int off = 1; off < 256; off <<= 1) {
                const float add = (tid >= off) ? scan_part[tid - off] : 0.f;
                __syncthreads();
                scan_part[tid] += add;
                __syncthreads();
            }
            float run = (tid == 0) ? 0.f : scan_part[tid - 1];
            const float thr = (float)(1.0 - (double)tp);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                run += e[u];
                const int pos = tid * 8 + u;
                if (pos < BV - 2 && run / total <= thr) sv[pos] = -INFINITY;
            }
            __syncthreads();
        }
        for (int v = tid; v < BV; v += 256) { const int id = si[v]; if (id < V) zs[id] = sv[v]; }
        __syncthreads();
    }
    const float run = d.first ? (j == 0 ? 0.f : -1e9f) : A.state[d.primary].run_score[j];
    float* out = A.scores + (size_t)slot * ld;
    for (int v = tid; v < V; v += 256) out[v] = zs[v] + run;
}

// order of the candidate list: larger key first, then the lower flat index beam * V + token
__device__ __forceinline__ bool cand_before(float ka, int fa, float kb, int fb) {
    return ka > kb || (ka == kb && fa < fb);
}

// ------------------------------------------------------------------------------------------------
// one CTA per group: K = 2 nb candidates over nb x V (top K, or K draws without replacement from softmax of the
// accumulated scores by an Exp(1) race), stop flags, the next running beams, the finished-set merge, the heuristic
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
beam_select_kernel(int ld, int V, SampleState S, BeamArgs A) {
    extern __shared__ float keys[];          // [nb * V]
    __shared__ float red[32];
    __shared__ float wk[8];
    __shared__ int wf[8];
    __shared__ int cand[2 * kMaxBeams];
    const BeamDesc& d = A.desc[blockIdx.x];
    BeamState& bs = A.state[d.primary];
    const int tid = threadIdx.x, nb = d.nb, K = 2 * nb, N = nb * V;
    const int p0 = d.slot[0];
    const int t = S.n_gen[p0];               // tokens so far = this step's index
    for (int f = tid; f < N; f += 256) keys[f] = A.scores[(size_t)d.slot[f / V] * ld + f % V];
    __syncthreads();
    if (d.do_sample) {
        float mx = -INFINITY;
        for (int f = tid; f < N; f += 256) mx = fmaxf(mx, keys[f]);
        mx = block_max(mx, red);
        float loc = 0.f;
        for (int f = tid; f < N; f += 256) { const float x = keys[f]; loc += (x == -INFINITY) ? 0.f : expf(x - mx); }
        const float total = block_sum(loc, red);
        const unsigned long long seed = S.seed[p0];
        const uint32_t k0 = (uint32_t)(seed & 0xffffffffull), k1 = (uint32_t)(seed >> 32);
        const uint32_t sseed = (uint32_t)S.seq_seed[p0];
        __syncthreads();
        for (int f = tid; f < N; f += 256) {
            uint32_t r[4];
            philox4x32_10((uint32_t)(f >> 2), (uint32_t)t, sseed, 0u, k0, k1, r);
            const float x = keys[f];
            const float p = (x == -INFINITY) ? 0.f : expf(x - mx) / total;
            const float uu = ((float)(r[f & 3] >> 9) + 0.5f) * (1.0f / 8388608.0f);
            keys[f] = p / (-logf(uu));
        }
        __syncthreads();
    }
    // K rounds of a block arg-max over the candidates after the previous pick in candidate order
    float lk = INFINITY; int lf = -1;
    for (int r = 0; r < K; ++r) {
        float bk = -INFINITY; int bf = 0x7fffffff;
        for (int f = tid; f < N; f += 256) {
            const float k = keys[f];
            if (r > 0 && !cand_before(lk, lf, k, f)) continue;
            if (bf == 0x7fffffff || cand_before(k, f, bk, bf)) { bk = k; bf = f; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
            const int of = __shfl_xor_sync(0xffffffffu, bf, o);
            if (of != 0x7fffffff && (bf == 0x7fffffff || cand_before(ok, of, bk, bf))) { bk = ok; bf = of; }
        }
        if ((tid & 31) == 0) { wk[tid >> 5] = bk; wf[tid >> 5] = bf; }
        __syncthreads();
        if (tid == 0) {
            float k = wk[0]; int f = wf[0];
            for (int w = 1; w < 8; ++w)
                if (wf[w] != 0x7fffffff && (f == 0x7fffffff || cand_before(wk[w], wf[w], k, f))) { k = wk[w]; f = wf[w]; }
            cand[r] = f; wk[0] = k; wf[0] = f;
        }
        __syncthreads();
        lk = wk[0]; lf = wf[0];
        __syncthreads();
    }
    if (tid != 0) return;
    const int stop = S.stop_token[p0], max_tok = S.max_tokens[p0];
    float cs[2 * kMaxBeams], rs[2 * kMaxBeams];
    int cb[2 * kMaxBeams], ct[2 * kMaxBeams];
    bool fl[2 * kMaxBeams];
    bool all_flag = true;
    for (int i = 0; i < K; ++i) {
        const int f = cand[i];
        cb[i] = f / V; ct[i] = f % V;
        cs[i] = A.scores[(size_t)d.slot[cb[i]] * ld + ct[i]];
        fl[i] = ct[i] == stop || t + 1 >= max_tok;
        all_flag = all_flag && fl[i];
        rs[i] = fl[i] ? cs[i] + -1.0e9f : cs[i];
    }
    // next running beams: the best nb of rs (ties: earlier candidate)
    bool used[2 * kMaxBeams];
    for (int i = 0; i < K; ++i) used[i] = false;
    float new_run[kMaxBeams];
    int2* hist = A.hist + ((size_t)d.primary * S.tokens_cap + t) * kMaxBeams;
    for (int jb = 0; jb < nb; ++jb) {
        int best = -1;
        for (int i = 0; i < K; ++i) if (!used[i] && (best < 0 || rs[i] > rs[best])) best = i;
        used[best] = true;
        new_run[jb] = rs[best];
        bs.sel_parent[jb] = cb[best]; bs.sel_tok[jb] = ct[best];
        hist[jb] = make_int2(cb[best], ct[best]);
    }
    // finished beams: length penalty, then the -1e9 masks, merged with the previous best nb (ties: the earlier entry)
    const float den = (float)pow((double)(t + 1), (double)d.length_penalty);
    const int M = nb + K;
    float ms[3 * kMaxBeams]; int mv[3 * kMaxBeams], mt[3 * kMaxBeams], mb[3 * kMaxBeams], mk[3 * kMaxBeams];
    for (int i = 0; i < nb; ++i) {
        ms[i] = bs.fin_score[i]; mv[i] = bs.fin_valid[i]; mt[i] = bs.fin_step[i]; mb[i] = bs.fin_beam[i]; mk[i] = bs.fin_tok[i];
    }
    for (int i = 0; i < K; ++i) {
        const bool did = i < nb && fl[i];
        float s = cs[i] / den;
        if (!bs.heur_unsat) s += -1.0e9f;
        if (!did) s += -1.0e9f;
        ms[nb + i] = s; mv[nb + i] = did; mt[nb + i] = t; mb[nb + i] = cb[i]; mk[nb + i] = ct[i];
    }
    bool taken[3 * kMaxBeams];
    for (int i = 0; i < M; ++i) taken[i] = false;
    for (int jb = 0; jb < nb; ++jb) {
        int best = -1;
        for (int i = 0; i < M; ++i) if (!taken[i] && (best < 0 || ms[i] > ms[best])) best = i;
        taken[best] = true;
        bs.fin_score[jb] = ms[best]; bs.fin_valid[jb] = mv[best]; bs.fin_step[jb] = mt[best];
        bs.fin_beam[jb] = mb[best]; bs.fin_tok[jb] = mk[best];
    }
    for (int jb = 0; jb < nb; ++jb) bs.run_score[jb] = new_run[jb];
    // _check_early_stop_heuristic (early_stopping False: the best running score at the current length)
    const float best_possible = new_run[0] / den;
    float mn = bs.fin_score[0];
    for (int i = 1; i < nb; ++i) mn = fminf(mn, bs.fin_score[i]);
    bool any = false;
    for (int i = 0; i < nb; ++i) any = any || best_possible > (bs.fin_valid[i] ? mn : -1.0e9f);
    bs.heur_unsat = bs.heur_unsat && any;
    bs.done = !(bs.heur_unsat && !all_flag);
}

// ------------------------------------------------------------------------------------------------
// one CTA per group: fork slot state and block tables to the new running beams.  Full pages of a parent's prefix are
// shared by its children; the partial page stays with the first child and is copied for the others; a beam whose next
// position starts a page gets a fresh one.  Pages no new table references go back to the group's pool first: none of
// them is a copy source, so the copies below may land in them.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
beam_reorder_kernel(SampleState S, BeamArgs A) {
    __shared__ int tb[kMaxBeams][kMaxTablePages];
    __shared__ unsigned seen_old[kMaxBeams][BV / 32];
    __shared__ int n_old[kMaxBeams], par[kMaxBeams], tok[kMaxBeams], first_child[kMaxBeams], n_old_max;
    __shared__ int ctx0, t0;
    const BeamDesc& d = A.desc[blockIdx.x];
    BeamState& bs = A.state[d.primary];
    if (bs.done) return;
    const int tid = threadIdx.x, nb = d.nb, W = S.seen_words;
    for (int i = tid; i < nb * A.max_pages; i += blockDim.x)
        tb[i / A.max_pages][i % A.max_pages] = A.block_tables[(size_t)d.slot[i / A.max_pages] * A.max_pages + i % A.max_pages];
    for (int i = tid; i < nb * W; i += blockDim.x) seen_old[i / W][i % W] = S.seen[(size_t)d.slot[i / W] * W + i % W];
    if (tid == 0) {
        int m = 0;
        for (int j = 0; j < nb; ++j) {
            n_old[j] = d.first && j > 0 ? 0 : bs.n_pages[j];
            m = max(m, n_old[j]);
            par[j] = bs.sel_parent[j]; tok[j] = bs.sel_tok[j];
            int fc = 1;
            for (int i = 0; i < j; ++i) if (bs.sel_parent[i] == bs.sel_parent[j]) fc = 0;
            first_child[j] = fc;
        }
        n_old_max = m;
        ctx0 = S.ctx_len[d.slot[0]] + d.advance;
        t0 = S.n_gen[d.slot[0]];
        bs.n_copy = 0;
    }
    __syncthreads();
    const int Lkv = ctx0, f = Lkv / kPageTokens, part = Lkv % kPageTokens;
    int* pool = A.pool + (size_t)d.primary * A.pool_cap;
    // pages at table index k that no new table references
    for (int k = tid; k < n_old_max; k += blockDim.x) {
        for (int j = 0; j < nb; ++j) {
            if (k >= n_old[j]) continue;
            const int pg = tb[j][k];
            bool dup = false;
            for (int i = 0; i < j; ++i) dup = dup || (k < n_old[i] && tb[i][k] == pg);
            if (dup) continue;
            bool ref = false;
            for (int i = 0; i < nb; ++i) {
                const int p = par[i];
                if (k < f || (k == f && part && first_child[i])) ref = ref || tb[p][k] == pg;
            }
            if (!ref) pool[atomicAdd(&bs.n_free, 1)] = pg;
        }
    }
    __syncthreads();
    if (tid == 0) {
        for (int i = 0; i < nb; ++i) {
            const int p = par[i];
            int pg;
            if (part && first_child[i]) pg = tb[p][f];
            else {
                pg = pool[--bs.n_free];
                if (part) {
                    const int c = bs.n_copy++;
                    bs.copy_src[c] = tb[p][f]; bs.copy_dst[c] = pg; bs.copy_ntok[c] = part;
                }
            }
            n_old[i] = pg;                                  // (reused: page at index f of beam i)
            bs.n_pages[i] = f + 1;
        }
    }
    __syncthreads();
    for (int i = tid; i < nb * (f + 1); i += blockDim.x) {
        const int b = i / (f + 1), k = i % (f + 1);
        A.block_tables[(size_t)d.slot[b] * A.max_pages + k] = k < f ? tb[par[b]][k] : n_old[b];
    }
    for (int i = tid; i < nb * W; i += blockDim.x) {
        const int b = i / W, w = i % W;
        unsigned v = seen_old[par[b]][w];
        if (w == (tok[b] >> 5)) v |= 1u << (tok[b] & 31);
        S.seen[(size_t)d.slot[b] * W + w] = v;
    }
    if (tid < nb) {
        const int s = d.slot[tid];
        S.last_tok[s] = tok[tid]; S.n_gen[s] = t0 + 1; S.ctx_len[s] = Lkv; S.finished[s] = 0;
        if (t0 < S.tokens_cap) S.tokens[(size_t)s * S.tokens_cap + t0] = tok[tid];
    }
}

// grid (groups * kMaxBeams, layers, 2): the valid tokens of one partial page of one layer's K (z = 0) or V (z = 1) pool
// K page: [head][64 / X][32 tok][X], V page: [head][32 tok][64], X * elem = 16 bytes
__global__ void __launch_bounds__(256)
kv_page_copy_kernel(BeamArgs A, void* const* kpool, void* const* vpool, int heads, int elem) {
    const BeamDesc& d = A.desc[blockIdx.x / kMaxBeams];
    const BeamState& bs = A.state[d.primary];
    const int c = blockIdx.x % kMaxBeams;
    if (bs.done || c >= bs.n_copy) return;
    const size_t page_vec = (size_t)heads * kPageTokens * kHeadDim * elem / 16;
    uint4* base = reinterpret_cast<uint4*>(blockIdx.z == 0 ? kpool[blockIdx.y] : vpool[blockIdx.y]);
    const uint4* src = base + (size_t)bs.copy_src[c] * page_vec;
    uint4* dst = base + (size_t)bs.copy_dst[c] * page_vec;
    const int ntok = bs.copy_ntok[c];
    const int vpr = kHeadDim * elem / 16;              // 16-byte vectors per V token row
    for (size_t q = threadIdx.x; q < page_vec; q += blockDim.x) {
        const int tk = blockIdx.z == 0 ? (int)(q % kPageTokens) : (int)((q / vpr) % kPageTokens);
        if (tk < ntok) dst[q] = src[q];
    }
}

// one CTA per group that ended this step: backtrack the best finished hypothesis through the history and write its
// tokens and latents into the primary slot, position by position (the latent of position t is in the ring of the beam
// that ran step t), then raise the primary slot's finished flag with the hypothesis length
__global__ void __launch_bounds__(256)
beam_gather_kernel(SampleState S, BeamArgs A) {
    extern __shared__ int src_slot[];        // [tokens_cap]
    __shared__ int n_tok;
    const BeamDesc& d = A.desc[blockIdx.x];
    const BeamState& bs = A.state[d.primary];
    if (!bs.done) return;
    const int P = d.primary, cap = S.tokens_cap;
    if (threadIdx.x == 0) {
        const int te = bs.fin_step[0];
        int b = bs.fin_beam[0];
        S.tokens[(size_t)P * cap + te] = bs.fin_tok[0];
        src_slot[te] = d.slot[b];
        for (int t = te - 1; t >= 0; --t) {
            const int2 h = A.hist[((size_t)P * cap + t) * kMaxBeams + b];
            S.tokens[(size_t)P * cap + t] = h.y;
            b = h.x;
            src_slot[t] = d.slot[b];
        }
        n_tok = te + 1;
    }
    __syncthreads();
    const int n = n_tok, H = A.H;
    for (size_t i = threadIdx.x; i < (size_t)n * H; i += blockDim.x) {
        const int t = (int)(i / H), h = (int)(i % H);
        const int s = src_slot[t];
        if (s != P) A.latents[((size_t)P * cap + t) * H + h] = A.latents[((size_t)s * cap + t) * H + h];
    }
    if (threadIdx.x == 0) { S.n_gen[P] = n; S.finished[P] = 1; }
}

}  // namespace

bool beam_supported(int V, int max_pages, int tokens_cap) {
    return V <= BV && max_pages <= kMaxTablePages && (size_t)tokens_cap * sizeof(int) <= 200 * 1024;
}

void beam_init_device() {
    // the largest the kernels may take (V = 2048, the largest token list beam_supported admits), the same for every
    // engine on the device: an attribute below 48 KB would lower the default limit
    CUDA_CHECK(cudaFuncSetAttribute(beam_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)(kMaxBeams * BV * sizeof(float))));
    CUDA_CHECK(cudaFuncSetAttribute(beam_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
}

void launch_beam_step(const float* logits, int ld_logits, int V, SampleState s, BeamArgs a, void* const* kpool,
                      void* const* vpool, int layers, int heads, int elem, cudaStream_t st, bool gather) {
    if (a.n_groups <= 0) return;
    if (!beam_supported(V, a.max_pages, s.tokens_cap)) throw CudaError("beam search: unsupported geometry");
    const size_t sel_smem = (size_t)kMaxBeams * V * sizeof(float);
    const int G = a.n_groups;
    ProfScope ps(KF_MISC, st, 0, (double)G * kMaxBeams * V * 12.0);
    beam_logprob_kernel<<<G * kMaxBeams, 256, 0, st>>>(logits, ld_logits, V, s, a);
    COUNT_LAUNCH(); KERNEL_CHECK();
    beam_select_kernel<<<G, 256, sel_smem, st>>>(ld_logits, V, s, a);
    COUNT_LAUNCH(); KERNEL_CHECK();
    beam_reorder_kernel<<<G, 128, 0, st>>>(s, a);
    COUNT_LAUNCH(); KERNEL_CHECK();
    kv_page_copy_kernel<<<dim3(G * kMaxBeams, layers, 2), 256, 0, st>>>(a, kpool, vpool, heads, elem);
    COUNT_LAUNCH(); KERNEL_CHECK();
    if (!gather) return;
    beam_gather_kernel<<<G, 256, (size_t)s.tokens_cap * sizeof(int), st>>>(s, a);
    COUNT_LAUNCH(); KERNEL_CHECK();
}

}  // namespace xtts
