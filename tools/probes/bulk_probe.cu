// cp.async.bulk streaming rate per SM as a function of copy size, ring depth and issuing threads (one CTA per SM, consumers
// only hand the slot back).   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bulk_probe bulk_probe.cu && ./bulk_probe
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void bar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void bar_expect(uint64_t* b, uint32_t n) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_wait(uint64_t* b, uint32_t ph) {
    uint32_t ok = 0;
    while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(s32(b)), "r"(ph) : "memory");
}
__device__ __forceinline__ void bulk(void* dst, const void* src, uint32_t n, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(dst)), "l"(src), "r"(n), "r"(s32(bar)) : "memory");
}
// each CTA streams `per_cta` bytes: stage = `copies` bulk copies of `csize` bytes (scattered `stride` apart), `depth` stages.
// `np` producer lanes each own stages s % np == lane (np = 1: one thread issues everything).  mode 1: consumers also read the
// stage into registers (LDS.128) before handing it back.
__global__ void __launch_bounds__(160) probe(const uint8_t* src, size_t per_cta, int csize, int copies, int depth, int np, int mode, size_t stride, float* sink, unsigned long long nblocks) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[32], empty[32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) for (int s = 0; s < depth; ++s) { bar_init(&full[s], 1); bar_init(&empty[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const size_t stage_bytes = (size_t)csize * copies;
    const uint32_t n = (uint32_t)(per_cta / stage_bytes);
    const uint8_t* base = src + (size_t)blockIdx.x * per_cta;
    if (w == 4) {
        if (lane < np)
            for (uint32_t c = lane; c < n; c += np) {
                const int s = c % depth;
                bar_wait(&empty[s], ((c / depth) & 1) ^ 1);
                bar_expect(&full[s], (uint32_t)stage_bytes);
                for (int k = 0; k < copies; ++k)
                    if (stride != 0) bulk(ring + (size_t)s * stage_bytes + (size_t)k * csize, base + ((size_t)c * copies + k) * stride, csize, &full[s]);
                    else {          // scattered: every copy reads a pseudo-randomly placed csize-aligned block of the whole buffer
                        const unsigned long long i = ((unsigned long long)blockIdx.x * n + c) * copies + k;
                        const unsigned long long blk = (i * 0x9E3779B1ull + 12345ull) % nblocks;
                        bulk(ring + (size_t)s * stage_bytes + (size_t)k * csize, src + blk * (size_t)csize, csize, &full[s]);
                    }
            }
        return;
    }
    float acc = 0.f;
    for (uint32_t c = w; c < n; c += 4) {
        const int s = c % depth;
        bar_wait(&full[s], (c / depth) & 1);
        if (mode == 1) {
            const uint4* p = reinterpret_cast<const uint4*>(ring + (size_t)s * stage_bytes);
            for (int i = lane; i < (int)(stage_bytes / 16); i += 32) { const uint4 v = p[i]; acc += __uint_as_float(v.x ^ v.y ^ v.z ^ v.w); }
        }
        __syncwarp();
        if (lane == 0) bar_arrive(&empty[s]);
    }
    if (acc == 123.456f) sink[0] = acc;
}
int main() {
    int nsm = 0; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
    const size_t total = (size_t)4 << 30;
    uint8_t* src; cudaMalloc(&src, total); cudaMemset(src, 1, total);
    float* sink; cudaMalloc(&sink, 4);
    cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    struct Cfg { int csize, copies, depth, np, mode, ctas_per_sm, scatter; };
    const Cfg cfgs[] = {{4096, 2, 16, 8, 0, 1, 0}, {4096, 2, 16, 8, 0, 1, 1}, {4096, 2, 8, 8, 0, 2, 0}, {4096, 2, 8, 8, 0, 2, 1},
                         {4096, 2, 8, 8, 0, 1, 1}, {16384, 1, 8, 2, 0, 1, 0}, {16384, 1, 8, 2, 0, 1, 1}, {65536, 1, 2, 1, 0, 1, 0}, {65536, 1, 2, 1, 0, 1, 1},
                         {1024, 8, 16, 8, 0, 1, 1}, {512, 16, 16, 8, 0, 1, 1}, {4096, 2, 8, 8, 0, 3, 1}};
    for (const Cfg& c : cfgs) {
        const int grid = nsm * c.ctas_per_sm;
        const size_t stage = (size_t)c.csize * c.copies;
        size_t per_cta = (total / grid) / stage * stage;
        per_cta = per_cta > ((size_t)24 << 20) ? ((size_t)24 << 20) / stage * stage : per_cta;       // 24 MB per CTA
        const size_t smem = stage * c.depth;
        float best = 1e9f;
        for (int rep = 0; rep < 3; ++rep) {
            cudaEventRecord(a);
            probe<<<grid, 160, smem>>>(src, per_cta, c.csize, c.copies, c.depth, c.np, c.mode, c.scatter ? 0 : (size_t)c.csize, sink, (unsigned long long)(total / c.csize));
            cudaEventRecord(b); cudaEventSynchronize(b);
            float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best;
        }
        cudaError_t e = cudaGetLastError();
        const double gbs = (double)per_cta * grid / best / 1e6;
        printf("%s copy %6d B x %d per stage, depth %2d (%3zu KB in flight/CTA), %d issuing lane(s), %d CTA/SM, consumers %s: %8.1f GB/s total, %6.1f GB/s per SM  %s\n",
               c.scatter ? "scattered " : "sequential", c.csize, c.copies, c.depth, smem >> 10, c.np, c.ctas_per_sm, c.mode ? "read stage" : "idle", gbs, gbs / nsm, e == cudaSuccess ? "" : cudaGetErrorString(e));
    }
    return 0;
}
