// The fp8 paged-KV format (engine option "kv_fp8"): e4m3 bytes with one power-of-two scale per (token, head), for K and V
// separately.  Everything that reads or writes fp8 pages (kv_write, the decode attention, the beam fork's page copy, the
// isolation harness) takes the layout and the quantiser from here.
//
// One (page, head) block of a K or V pool, kKv8Block = 2080 bytes (a multiple of 32, so blocks stay sector-aligned):
//   K: [64/16][32 tok][16] e4m3   (16 dims of one token per 16-byte atom: a lane = a token reads 16 B, as in the 16-bit K)
//   V: [32 tok][64] e4m3
//   then 32 int8 exponents, one per token: value = e4m3 * 2^e.
// Quantiser of one 64-dim row x: amax = max |x|, e = the smallest integer with amax * 2^-e <= 448 (e4m3's largest finite),
// clamped to int8 (an all-zero row gets -128); byte = e4m3 round-to-nearest-even of x * 2^-e, which never saturates.
#pragma once
#include <cuda_fp8.h>
#include "common.cuh"

namespace xtts {

constexpr int kKv8X = 16;                                           // e4m3 elements per 16-byte K atom
constexpr int kKv8Data = kPageTokens * kHeadDim;                    // 2048 bytes of e4m3 per block
constexpr int kKv8Block = kKv8Data + kPageTokens;                   // + the 32 exponents
static_assert(kKv8Block % 32 == 0, "fp8 KV blocks must stay 32-byte aligned");

// bytes of one (page, head) block of a K or V pool of `elem`-byte elements (1: fp8, exponents included)
__host__ __device__ constexpr size_t kv_block_bytes(int elem) {
    return elem == 1 ? (size_t)kKv8Block : (size_t)kPageTokens * kHeadDim * elem;
}

__host__ __device__ inline size_t kv8_block(int page, int heads, int h) { return ((size_t)page * heads + h) * kKv8Block; }
__host__ __device__ inline int kv8_k_off(int tk, int d) { return ((d / kKv8X) * kPageTokens + tk) * kKv8X + d % kKv8X; }
__host__ __device__ inline int kv8_v_off(int tk, int d) { return tk * kHeadDim + d; }
__host__ __device__ inline int kv8_e_off(int tk) { return kKv8Data + tk; }

// 2^e exactly, for e in [-149, 127]
__device__ __forceinline__ float kv8_pow2(int e) {
    return e >= -126 ? __int_as_float((e + 127) << 23) : __int_as_float(1 << (e + 149));
}

// the scale exponent of a row whose largest magnitude is amax
__device__ __forceinline__ int kv8_exponent(float amax) {
    if (!(amax > 0.f)) return -128;
    int E;
    const float m = frexpf(amax, &E);                 // amax = m * 2^E, m in [0.5, 1); 448 = 0.875 * 2^9
    const int e = (m <= 0.875f) ? E - 9 : E - 8;
    return max(-128, min(127, e));
}

__device__ __forceinline__ uint8_t kv8_quant(float x, int e) {
    return (uint8_t)__nv_cvt_float_to_fp8(ldexpf(x, -e), __NV_SATFINITE, __NV_E4M3);
}

__device__ __forceinline__ float kv8_dequant(uint8_t q, int e) {
    const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)q, __NV_E4M3);
    return __half2float(__half(h)) * kv8_pow2(e);
}

// one 16-byte atom = 16 e4m3 values -> fp32 (unscaled), through the hardware e4m3x2 -> f16x2 conversion
__device__ __forceinline__ void kv8_unpack16(const uint4& raw, float* f) {
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> (16 * j)), __NV_E4M3);
            const float2 t = __half22float2(__half2(h));
            f[4 * i + 2 * j] = t.x; f[4 * i + 2 * j + 1] = t.y;
        }
    }
}

// The append of one token of one head by a 128-thread CTA: thread t < 64 holds k[t], thread 64 + d holds v[d].  Writes the
// bytes and the exponents into the K / V blocks (kv8_block) at token slot tk and returns the dequantised value of this
// thread's element.  `red` is 4 floats of shared memory; every thread of the CTA must call it.
__device__ __forceinline__ float kv8_append(float x, uint8_t* __restrict__ kblk, uint8_t* __restrict__ vblk, int tk, float* red) {
    const int t = threadIdx.x, d = t & 63;
    const float a = warp_max(fabsf(x));
    if ((t & 31) == 0) red[t >> 5] = a;
    __syncthreads();
    const int e = kv8_exponent(fmaxf(red[(t >> 6) * 2], red[(t >> 6) * 2 + 1]));
    const uint8_t q = kv8_quant(x, e);
    uint8_t* blk = t < 64 ? kblk : vblk;
    blk[t < 64 ? kv8_k_off(tk, d) : kv8_v_off(tk, d)] = q;
    if (d == 0) blk[kv8_e_off(tk)] = (uint8_t)(int8_t)e;
    return kv8_dequant(q, e);
}

}  // namespace xtts
