// Shared helpers for the sm_90a kernels of the XTTSv2 hot path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

namespace xtts {

struct CudaError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

inline void cuda_check(cudaError_t e, const char* what, const char* file, int line) {
    if (e != cudaSuccess) {
        char buf[512];
        snprintf(buf, sizeof(buf), "CUDA error %s (%d) at %s:%d in %s", cudaGetErrorString(e), (int)e, file, line, what);
        throw CudaError(buf);
    }
}
#define CUDA_CHECK(x) ::xtts::cuda_check((x), #x, __FILE__, __LINE__)
#define KERNEL_CHECK() ::xtts::cuda_check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__)

// Per-engine launcher state.  Several engines (one per GPU) may live in one process, each with its own scheduler thread:
// what used to be process globals is a KernelCtx owned by the engine and bound to whichever thread issues that engine's
// work (the scheduler thread, or an API thread inside a synchronous entry point).  Unbound threads see a default context.
struct KernelCtx;
extern thread_local KernelCtx* t_kctx;
KernelCtx& kctx_default();
inline KernelCtx& kctx() { return t_kctx ? *t_kctx : kctx_default(); }
// Every kernel launch of this library goes through this counter (bench.py "gpu_launches").
#define g_launch_count (::xtts::kctx().launch_count)
#define COUNT_LAUNCH() (++::xtts::kctx().launch_count)

// Optional per-kernel-family timing with CUDA events on the launching stream (bench.py "roofline").
// Off by default; when on, every launcher records an event pair and its algorithmic FLOPs / bytes.
enum KernelFamily : int {
    KF_GEMM_TC = 0, KF_GEMM_F32, KF_ATTN_DECODE, KF_ATTN_PREFILL, KF_NORM, KF_SAMPLE, KF_KV_WRITE, KF_EMBED,
    KF_CONV1D, KF_CONVT, KF_CONV_POST, KF_INTERP, KF_COND, KF_MISC, KF_CONV1D_TC, KF_DECODE_CHAIN, KF_COUNT
};
struct KernelProfiler {
    bool enabled = false;
    struct Rec { cudaEvent_t a, b; int fam; };
    // Events bracketing the kernels of ONE captured graph (cudaEventRecordExternal nodes): re-recorded by every replay and
    // read back after the replay's synchronize.  Inside a graph there is no host launch gap between the event and the
    // kernel, so these are true device durations even for 5-us kernels (eager event pairs include the CPU launch latency).
    struct GraphRecs {
        std::vector<Rec> recs;
        double flops[KF_COUNT] = {0}, bytes[KF_COUNT] = {0};
        unsigned long long launches[KF_COUNT] = {0};
        double ctx_sum = 0;            // cached tokens summed over the step's rows when the graph was captured
    };
    GraphRecs* cap = nullptr;          // non-null while a profiled graph is being captured
    std::vector<Rec> recs;
    std::vector<cudaEvent_t> pool;
    double ms[KF_COUNT] = {0}, flops[KF_COUNT] = {0}, bytes[KF_COUNT] = {0};
    unsigned long long launches[KF_COUNT] = {0};
    cudaEvent_t get() {
        if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
        cudaEvent_t e; cudaEventCreate(&e); return e;
    }
    void collect() {           // call with the device idle (after a synchronize)
        for (auto& r : recs) {
            float t = 0.f;
            if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) ms[r.fam] += t;
            pool.push_back(r.a); pool.push_back(r.b);
        }
        recs.clear();
    }
    // after the replay has been synchronized.  The paged-attention work of a replay scales with the tokens cached NOW,
    // not with those cached when the graph was captured: `ctx_sum_now` rescales that family's algorithmic bytes / FLOPs.
    void collect_graph(const GraphRecs& g, double ctx_sum_now) {
        for (auto& r : g.recs) {
            float t = 0.f;
            if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) ms[r.fam] += t;
        }
        const double attn_scale = (g.ctx_sum > 0 && ctx_sum_now > 0) ? ctx_sum_now / g.ctx_sum : 1.0;
        for (int i = 0; i < KF_COUNT; ++i) {
            const double sc = (i == KF_ATTN_DECODE) ? attn_scale : 1.0;
            flops[i] += sc * g.flops[i]; bytes[i] += sc * g.bytes[i]; launches[i] += g.launches[i];
        }
        (void)cudaGetLastError();
    }
    void reset() { collect(); for (int i = 0; i < KF_COUNT; ++i) { ms[i] = flops[i] = bytes[i] = 0; launches[i] = 0; } }
};
struct KernelCtx {
    unsigned long long launch_count = 0;
    KernelProfiler prof;
    bool use_pdl = true;
    int voc_sm_cap = 0;           // > 0: persistent tensor-core conv grids take at most this many SMs (set per vocoder batch)
    int attn_ctas_per_sm = 0;     // 0 = uncapped decode-attention grid; > 0: at most this many CTAs per SM
    int gemm_decode_bn = 0;       // 0 = heuristic; 32/64/128 forces the tile width of decode-shaped tensor-core GEMMs
    int attn_warps = 4;           // warps per (row, head) item of the bf16 decode attention (4, or 8: measured slower, run 7)
    int attn_bulk = 0;            // > 0: 16-bit decode attention streams cache pages with cp.async.bulk, this many CTAs per SM
    int attn_stages = 8;          // ring depth of that kernel (8 KB per stage)
    int attn_l2_pages = 0;        // register-load decode attention: every warp prefetches the page this many of its pages ahead into L2
    int attn_l2_ahead = 1;        // that kernel prefetches the next item's pages into L2 (cp.async.bulk.prefetch.L2)
    int gemm_deep_ring = 0;       // decode-shaped unsplit GEMMs use a ring that fills the SM (BN 32: 10 stages, BN 64: 8) instead of 5 / 4
    int gemm_l2_prefetch = 0;     // one-tile GEMM: weight tiles beyond the first ring pass are prefetched into L2 before the dependency wait
    int gemm_wide = 4;            // large shapes (M >= 256) go to the persistent wide-tile kernel (gemm_wgmma_wide.cu) with this ring depth (2-4); 0: off
};
#define g_prof (::xtts::kctx().prof)
#define g_use_pdl (::xtts::kctx().use_pdl)
#define g_voc_sm_cap (::xtts::kctx().voc_sm_cap)
#define g_attn_ctas_per_sm (::xtts::kctx().attn_ctas_per_sm)
#define g_gemm_decode_bn (::xtts::kctx().gemm_decode_bn)
#define g_gemm_wide (::xtts::kctx().gemm_wide)
#define g_attn_warps (::xtts::kctx().attn_warps)
#define g_gemm_l2_prefetch (::xtts::kctx().gemm_l2_prefetch)
#define g_gemm_deep_ring (::xtts::kctx().gemm_deep_ring)
#define g_attn_bulk (::xtts::kctx().attn_bulk)
#define g_attn_stages (::xtts::kctx().attn_stages)
#define g_attn_l2_ahead (::xtts::kctx().attn_l2_ahead)
#define g_attn_l2_pages (::xtts::kctx().attn_l2_pages)

// true the first time it is called with the current CUDA device for this flag set (function attributes are per device)
inline bool first_on_device(bool (&done)[64]) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || done[dev]) return false;
    done[dev] = true;
    return true;
}

// SM count of the current CUDA device (persistent grids, tile heuristics); cached per device
inline int sm_count() {
    static int n[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (n[dev] <= 0 && cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        (void)cudaGetLastError();
        n[dev] = 0;
        throw CudaError("cudaDevAttrMultiProcessorCount query failed");
    }
    return n[dev];
}

struct ProfScope {
    cudaStream_t st; cudaEvent_t b; bool on; bool ext;
    ProfScope(int fam, cudaStream_t s, double fl = 0, double by = 0) : st(s), b(nullptr), on(g_prof.enabled), ext(false) {
        if (!on) return;
        if (g_prof.cap) {                          // capturing a profiled graph: event-record nodes owned by that graph
            ext = true;
            cudaEvent_t a; cudaEventCreate(&a); cudaEventCreate(&b);
            cudaEventRecordWithFlags(a, st, cudaEventRecordExternal);
            g_prof.cap->recs.push_back({a, b, fam});
            g_prof.cap->flops[fam] += fl; g_prof.cap->bytes[fam] += by; g_prof.cap->launches[fam] += 1;
            return;
        }
        cudaEvent_t a = g_prof.get(); b = g_prof.get();
        cudaEventRecord(a, st);
        g_prof.recs.push_back({a, b, fam});
        g_prof.flops[fam] += fl; g_prof.bytes[fam] += by; g_prof.launches[fam] += 1;
    }
    ~ProfScope() {
        if (!on) return;
        if (ext) cudaEventRecordWithFlags(b, st, cudaEventRecordExternal); else cudaEventRecord(b, st);
    }
};
inline const char* kernel_family_name(int f) {
    static const char* n[KF_COUNT] = {"gemm_bf16_wgmma", "gemm_f32", "attn_decode_paged", "attn_prefill", "layernorm",
                                      "sample", "kv_write", "embed", "conv1d", "conv_transpose1d", "conv_post_tanh",
                                      "interp", "conditioning", "misc", "conv1d_tc_f16_wgmma", "decode_chain_wgmma"};
    return (f >= 0 && f < KF_COUNT) ? n[f] : "?";
}

// ---- device-side timeline (debug, option "trace"): the first and the last CTA of a traced kernel stamp %globaltimer at
// entry, after the dependency wait and at exit.  Unlike event brackets this does not serialise anything, so it shows the
// decode step as it really runs (PDL overlap, concurrent branches).  One buffer per translation unit (no -rdc).
struct TraceBuf { unsigned long long* rec; unsigned* n; unsigned cap; };
static __device__ TraceBuf g_trace_tu = {nullptr, nullptr, 0};
enum { TR_GEMM = 1, TR_ATTN = 2, TR_REDUCE_LN = 3, TR_LN = 4, TR_HEAD = 5, TR_SAMPLE = 6, TR_ROWS = 7, TR_CONV = 8 };
__device__ __forceinline__ void trace_pt(int id, int phase) {
    if (threadIdx.x != 0 || threadIdx.y != 0) return;
    const bool first = (blockIdx.x | blockIdx.y | blockIdx.z) == 0;
    const bool last = blockIdx.x == gridDim.x - 1 && blockIdx.y == gridDim.y - 1 && blockIdx.z == gridDim.z - 1;
    if (!first && !last) return;
    const TraceBuf tb = g_trace_tu;
    if (tb.rec == nullptr) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned i = atomicAdd(tb.n, 1u);
    if (i < tb.cap) {
        tb.rec[2 * i] = t;
        tb.rec[2 * i + 1] = ((unsigned long long)id << 32) | ((unsigned long long)(first ? 0 : 1) << 8) | (unsigned long long)phase |
                            ((unsigned long long)(gridDim.x * gridDim.y * gridDim.z) << 40);
    }
}
#define XTTS_TRACE_SETTER(name) void name(TraceBuf b) { cudaMemcpyToSymbol(g_trace_tu, &b, sizeof(b)); }

// ---- programmatic dependent launch (PDL): the decode step is a chain of ~200 short dependent kernels; with the
// programmatic-serialization attribute kernel N+1 is launched while kernel N still runs, does its prologue (barrier
// init, weight-tile prefetch) and only blocks at griddepcontrol.wait before touching N's outputs.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- fine-grained dependencies along the decode chain.  `griddepcontrol.wait` resolves only when the whole prerequisite
// grid has drained and flushed (measured: 1.2-5 us after its last CTA's exit, tools/trace_step.py).  With a DepFlag the
// consumer instead polls a counter that every producer CTA bumps (release) right after its own stores: ~1 us.  The consumer
// kernel is still launched with the PDL attribute (so it is resident early) but never executes griddepcontrol.wait; ordering
// with everything older follows transitively, because its producer waited on ITS producer's flag before finishing.
// wait == nullptr: fall back to griddepcontrol.wait.  One thread of the CTA calls dep_wait, then the CTA synchronises.
struct DepFlag {
    const unsigned* wait = nullptr;     // counter of the producer kernel (device)
    unsigned target = 0;                // its value once every producer CTA has arrived
    unsigned* arrive = nullptr;         // this kernel's own counter (nullptr: nobody polls it)
};
__device__ __forceinline__ void dep_wait(const DepFlag& d) {
    if (d.wait == nullptr) { pdl_wait(); return; }
    const long long t0 = clock64();
    int polls = 0;
    unsigned v;
    while (true) {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(d.wait) : "memory");
        if (v >= d.target) break;
        __nanosleep(polls < 8 ? 100 : 400);          // hundreds of CTAs poll one line that the producers are also adding to
        if ((++polls & 255) == 0 && clock64() - t0 > 4000000000LL) __trap();     // watchdog (no printf: see hopper.cuh)
    }
}
// every thread that stored results calls this; `leader` (one thread, after a CTA barrier) publishes the CTA's arrival
__device__ __forceinline__ void dep_arrive(const DepFlag& d, bool leader) {
    if (d.arrive == nullptr) return;
    __threadfence();
    __syncthreads();
    if (leader) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(d.arrive) : "memory");
}

template <typename... KArgs, typename... Args>
inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    if (pdl && g_use_pdl) {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
    }
    cuda_check(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...), "cudaLaunchKernelEx", __FILE__, __LINE__);
}

constexpr int kHeadDim = 64;       // 16 heads x 64 (xttsv2_gpt_config.py:136-138); kernels specialise on it
constexpr int kPageTokens = 32;    // KV page = one warp of tokens

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// block-wide sum for blockDim.x <= 1024 (multiple of 32); `red` is >= 32 floats of smem
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();               // protect `red` from the previous use
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : -INFINITY;
    r = warp_max(r);
    return r;
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// two fp32 -> one 32-bit word of 16-bit values: IEEE fp16 when f16, bf16 otherwise (the GEMMs' 16-bit epilogue)
__device__ __forceinline__ uint32_t pack16(float a, float b, bool f16) {
    if (f16) { __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// tanh-GELU ("gelu_new", checkpoint_converter.py:197)
__device__ __forceinline__ float gelu_new(float x) {
    const float k = 0.7978845608028654f;   // sqrt(2/pi)
    return 0.5f * x * (1.0f + tanhf(k * (x + 0.044715f * x * x * x)));
}

}  // namespace xtts
