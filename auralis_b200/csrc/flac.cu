// FLAC encoder (see cond.h): mono 16-bit PCM -> a complete FLAC stream (RFC 9639), for TTSOutput.to_bytes("flac").
//
// Stream: "fLaC", one STREAMINFO block (flagged last), then one frame per block of 4096 samples (the last block holds
// the remainder).  Fixed blocking, one channel, 16 bits per sample, no wasted bits.
//
// Per block (flac_analyse_kernel, one CTA) every candidate subframe is costed exactly in bits and the smallest is kept;
// on a tie the first in this order: CONSTANT (all samples equal), VERBATIM, FIXED orders 0..4, LPC orders 1..12 at a
// precision of 12 bits.  A predictor of order o is a candidate only when the block holds more than o samples; a
// 1-sample block is CONSTANT.  The LPC coefficients come from one Tukey(0.5)-windowed fp64 autocorrelation and
// Levinson-Durbin, quantised with a carried rounding error; an order whose residual would reach |r| >= 2^31 is dropped.
// Residuals are partitioned Rice codes (method 00, parameters 0..14, no escape), partition orders 0..6 where the block
// allows; each partition's parameter is chosen by exact cost from the sums S_k = sum (u >> k), which are accumulated
// once at the finest partition order and merged upward.  So no subframe costs more than VERBATIM, and a frame is at
// most 8211 bytes.
//
// flac_scan_kernel turns the frame sizes of a batch into byte offsets; flac_write_kernel (one CTA per frame) writes
// the header and its CRC-8, the warm-up samples and coefficients, and the Rice codes at bit offsets from a block-wide
// prefix sum of code lengths, MSB-first into shared memory, then a CRC-16 computed in 256 byte-serial pieces combined
// by polynomial multiplication.  Every sum is integer or in a fixed order, so the stream does not depend on the batch
// size and is the same from run to run.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <stdexcept>

#include "cond.h"

namespace xtts {
namespace {

constexpr int kBlock = 4096, kThreads = 256, kPerThread = kBlock / kThreads;
constexpr int kMaxLpc = 12, kPrec = 12, kMaxPorder = 6, kNumK = 15;
constexpr int kMaxFrameBytes = 8211, kWords = (kMaxFrameBytes + 3) / 4;
constexpr int kStreamHeader = 42;                          // "fLaC" + block header + STREAMINFO
enum : int { SUB_CONSTANT = 0, SUB_VERBATIM = 1, SUB_FIXED = 2, SUB_LPC = 3 };

struct FrameDesc {
    int32_t type, order, shift, porder;
    int32_t bits;                  // subframe bits
    int32_t bytes;                 // the whole frame: header, subframe, padding, CRC-16
    int32_t q[kMaxLpc];
    uint8_t k[1 << kMaxPorder];    // Rice parameter of each partition
};

// frame-header sample-rate code; 0 = "see STREAMINFO" for rates without one
__host__ __device__ inline int rate_code(int sr) {
    switch (sr) {
        case 88200: return 1;  case 176400: return 2; case 192000: return 3; case 8000: return 4;
        case 16000: return 5;  case 22050: return 6;  case 24000: return 7;  case 32000: return 8;
        case 44100: return 9;  case 48000: return 10; case 96000: return 11; default: return 0;
    }
}

__device__ int block_size_code(int nb) {
    if (nb == 192) return 1;
    for (int c = 2; c <= 5; ++c) if (nb == 576 << (c - 2)) return c;
    for (int c = 8; c <= 15; ++c) if (nb == 256 << (c - 8)) return c;
    return nb <= 256 ? 6 : 7;                              // (size - 1) in 8 / 16 bits after the frame number
}

// The frame header of frame `frame` (nb samples) with its CRC-8, into h; returns its length (at most 16 bytes).
__device__ int frame_header(uint8_t* h, int64_t frame, int nb, int rcode) {
    int i = 0;
    const int bc = block_size_code(nb);
    h[i++] = 0xFF; h[i++] = 0xF8;                          // sync, reserved 0, fixed blocking
    h[i++] = (uint8_t)(bc << 4 | rcode);
    h[i++] = 0x08;                                         // mono, 16 bits, reserved 0
    if (frame < 0x80) {
        h[i++] = (uint8_t)frame;
    } else {                                               // an n-byte code carries 5n + 1 bits
        int nbytes = 2;
        while (frame >> (5 * nbytes + 1)) ++nbytes;
        h[i++] = (uint8_t)(((0xFF00 >> nbytes) & 0xFF) | (frame >> (6 * (nbytes - 1))));
        for (int c = nbytes - 2; c >= 0; --c) h[i++] = (uint8_t)(0x80 | ((frame >> (6 * c)) & 0x3F));
    }
    if (bc == 6) h[i++] = (uint8_t)(nb - 1);
    else if (bc == 7) { h[i++] = (uint8_t)((nb - 1) >> 8); h[i++] = (uint8_t)(nb - 1); }
    uint8_t crc = 0;
    for (int j = 0; j < i; ++j) {
        crc ^= h[j];
        for (int b = 0; b < 8; ++b) crc = (uint8_t)(crc & 0x80 ? (crc << 1) ^ 0x07 : crc << 1);
    }
    h[i++] = crc;
    return i;
}

__device__ __forceinline__ uint32_t fold(int64_t r) { return (uint32_t)(r >= 0 ? 2 * r : -2 * r - 1); }

// the largest partition order the block allows for a predictor of this order
__device__ int max_porder(int nb, int order) {
    int p = 0;
    while (p < kMaxPorder && (nb & ((2 << p) - 1)) == 0 && (nb >> (p + 1)) > order) ++p;
    return p;
}

__device__ __forceinline__ int fixed_residual(const int32_t* s, int i, int order) {
    switch (order) {
        case 0: return s[i];
        case 1: return s[i] - s[i - 1];
        case 2: return s[i] - 2 * s[i - 1] + s[i - 2];
        case 3: return s[i] - 3 * s[i - 1] + 3 * s[i - 2] - s[i - 3];
        default: return s[i] - 4 * s[i - 1] + 6 * s[i - 2] - 4 * s[i - 3] + s[i - 4];
    }
}

__device__ __forceinline__ int64_t lpc_residual(const int32_t* s, int i, int order, const int32_t* q, int shift) {
    int64_t acc = 0;
    for (int j = 0; j < order; ++j) acc += (int64_t)q[j] * s[i - 1 - j];
    return (int64_t)s[i] - (acc >> shift);
}

struct AnalyseShared {
    int32_t s[kBlock];
    unsigned long long sums[(1 << kMaxPorder) * kNumK];   // S_k per finest partition
    uint32_t pbits[(2 << kMaxPorder) - 1];                 // best cost of partition j at order p, at index 2^p - 1 + j
    uint8_t pk[(2 << kMaxPorder) - 1];
    double red[kThreads / 32][kMaxLpc + 1];
    double lpc[kMaxLpc][kMaxLpc];                          // Levinson-Durbin coefficients of each order
    int32_t q[kMaxLpc];
    int n_lpc, shift, skip, bad, take, cost_p;
    uint32_t cost_bits;
    FrameDesc best;
};

// Residual cost of samples order .. nb-1 with folded residuals u(i): sets cost_bits (method, partition order and every
// partition) and cost_p, and leaves the chosen parameters in pk.  Called by every thread.
template <class U>
__device__ void rice_cost(AnalyseShared& sh, int nb, int order, U u_of) {
    const int tid = threadIdx.x;
    const int pm = max_porder(nb, order), L = nb >> pm;
    for (int i = tid; i < (kNumK << pm); i += kThreads) sh.sums[i] = 0;
    __syncthreads();
    const int C = (nb + kThreads - 1) / kThreads;
    const int i1 = min(nb, (tid + 1) * C);
    unsigned long long acc[kNumK];
    int cur = -1;
    for (int i = max(tid * C, order); i < i1; ++i) {
        const int part = i / L;
        if (part != cur) {
            if (cur >= 0)
                for (int k = 0; k < kNumK; ++k) atomicAdd(&sh.sums[cur * kNumK + k], acc[k]);
            cur = part;
            for (int k = 0; k < kNumK; ++k) acc[k] = 0;
        }
        const uint32_t u = u_of(i);
        for (int k = 0; k < kNumK; ++k) acc[k] += u >> k;
    }
    if (cur >= 0)
        for (int k = 0; k < kNumK; ++k) atomicAdd(&sh.sums[cur * kNumK + k], acc[k]);
    __syncthreads();
    if (tid < (2 << pm) - 1) {                             // one thread per (order p, partition j)
        const int p = 31 - __clz(tid + 1), j = tid + 1 - (1 << p), span = 1 << (pm - p);
        const unsigned long long cnt = (unsigned long long)((nb >> p) - (j == 0 ? order : 0));
        unsigned long long best = ULLONG_MAX;
        int bk = 0;
        for (int k = 0; k < kNumK; ++k) {
            unsigned long long c = cnt * (k + 1);
            for (int f = j * span; f < (j + 1) * span; ++f) c += sh.sums[f * kNumK + k];
            if (c < best) { best = c; bk = k; }
        }
        sh.pbits[tid] = 4 + (uint32_t)best;                // the parameter, then the codes
        sh.pk[tid] = (uint8_t)bk;
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t best = UINT_MAX;
        int bp = 0;
        for (int p = 0; p <= pm; ++p) {
            uint32_t c = 6;                                // method 00 and the partition order
            for (int j = 0; j < 1 << p; ++j) c += sh.pbits[(1 << p) - 1 + j];
            if (c < best) { best = c; bp = p; }
        }
        sh.cost_bits = best; sh.cost_p = bp;
    }
    __syncthreads();
}

// Keep the candidate just costed by rice_cost if it is strictly smaller than the best so far.
__device__ void consider(AnalyseShared& sh, int type, int order, uint32_t head_bits) {
    const int tid = threadIdx.x;
    if (tid == 0) {
        const uint32_t total = head_bits + sh.cost_bits;
        sh.take = total < (uint32_t)sh.best.bits;
        if (sh.take) {
            sh.best.type = type; sh.best.order = order; sh.best.porder = sh.cost_p; sh.best.bits = (int32_t)total;
            sh.best.shift = type == SUB_LPC ? sh.shift : 0;
            for (int j = 0; j < kMaxLpc; ++j) sh.best.q[j] = type == SUB_LPC && j < order ? sh.q[j] : 0;
        }
    }
    __syncthreads();
    if (sh.take && tid < (1 << sh.cost_p)) sh.best.k[tid] = sh.pk[(1 << sh.cost_p) - 1 + tid];
    __syncthreads();
}

// One CTA per block: frames frame0 .. frame0 + gridDim.x - 1 of the stream; pcm holds this batch's samples (ns).
__global__ void __launch_bounds__(kThreads) flac_analyse_kernel(const int16_t* __restrict__ pcm, int64_t ns,
                                                                 int64_t frame0, int rcode, FrameDesc* __restrict__ desc) {
    extern __shared__ double xs[];                         // the windowed block [kBlock]
    __shared__ AnalyseShared sh;
    const int tid = threadIdx.x, f = blockIdx.x;
    const int nb = (int)min((int64_t)kBlock, ns - (int64_t)f * kBlock);
    const int16_t* x = pcm + (size_t)f * kBlock;
    for (int i = tid; i < nb; i += kThreads) sh.s[i] = x[i];
    for (int i = tid; i < (1 << kMaxPorder); i += kThreads) sh.best.k[i] = 0;
    __syncthreads();

    bool same = true;
    for (int i = tid; i < nb; i += kThreads) same &= sh.s[i] == sh.s[0];
    const bool constant = __syncthreads_and(same);
    if (tid == 0) {
        sh.best.type = constant ? SUB_CONSTANT : SUB_VERBATIM;
        sh.best.bits = constant ? 8 + 16 : 8 + 16 * nb;
        sh.best.order = sh.best.shift = sh.best.porder = 0;
        for (int j = 0; j < kMaxLpc; ++j) sh.best.q[j] = 0;
    }
    __syncthreads();

    if (nb > 1) {
        for (int order = 0; order <= 4 && order < nb; ++order) {
            rice_cost(sh, nb, order, [&](int i) { return fold(fixed_residual(sh.s, i, order)); });
            consider(sh, SUB_FIXED, order, 8 + 16 * order);
        }

        // Tukey(0.5) window, fp64 autocorrelation at lags 0..12 (per thread, then a fixed-order tree)
        const int max_order = min(kMaxLpc, nb - 1);
        const double half = 0.25 * (nb - 1);               // alpha (N - 1) / 2: the length of each cosine taper
        for (int i = tid; i < nb; i += kThreads) {
            const int e = min(i, nb - 1 - i);
            const double w = e < half ? 0.5 * (1.0 - cos(kPi * e / half)) : 1.0;
            xs[i] = w * sh.s[i];
        }
        __syncthreads();
#pragma unroll
        for (int l = 0; l <= kMaxLpc; ++l) {
            double a = 0.0;
            if (l <= max_order)
                for (int i = tid; i + l < nb; i += kThreads) a += xs[i] * xs[i + l];
            for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
            if ((tid & 31) == 0) sh.red[tid >> 5][l] = a;
        }
        __syncthreads();
        if (tid == 0) {                                    // Levinson-Durbin
            double R[kMaxLpc + 1], a[kMaxLpc + 1] = {0}, tmp[kMaxLpc + 1];
            for (int l = 0; l <= max_order; ++l) {
                R[l] = 0.0;
                for (int w = 0; w < kThreads / 32; ++w) R[l] += sh.red[w][l];
            }
            double err = R[0];
            int n_lpc = 0;
            for (int i = 1; i <= max_order && err > 0.0; ++i) {
                double acc = R[i];
                for (int j = 1; j < i; ++j) acc -= a[j] * R[i - j];
                const double k = acc / err;
                for (int j = 1; j < i; ++j) tmp[j] = a[j] - k * a[i - j];
                for (int j = 1; j < i; ++j) a[j] = tmp[j];
                a[i] = k;
                err *= 1.0 - k * k;
                for (int j = 0; j < i; ++j) sh.lpc[i - 1][j] = a[j + 1];
                n_lpc = i;
            }
            sh.n_lpc = n_lpc;
        }
        __syncthreads();

        const int n_lpc = sh.n_lpc;
        for (int order = 1; order <= n_lpc; ++order) {
            __syncthreads();                               // every thread has read the last order's skip / bad
            if (tid == 0) {                                // quantise to 12 bits with a carried rounding error
                double cmax = 0.0;
                for (int j = 0; j < order; ++j) cmax = fmax(cmax, fabs(sh.lpc[order - 1][j]));
                int shift = 0;
                bool skip = !isfinite(cmax);
                if (!skip && cmax > 0.0) {
                    int ex;
                    frexp(cmax, &ex);                      // cmax = m 2^ex, m in [0.5, 1): floor(log2 cmax) = ex - 1
                    shift = min(15, (kPrec - 1) - (ex - 1) - 1);
                    skip = shift < 0;
                }
                if (!skip) {
                    double err = 0.0;
                    const int qmax = (1 << (kPrec - 1)) - 1, qmin = -(1 << (kPrec - 1));
                    for (int j = 0; j < order; ++j) {
                        err += sh.lpc[order - 1][j] * (double)(1 << shift);
                        const int qj = (int)fmax((double)qmin, fmin((double)qmax, round(err)));
                        sh.q[j] = qj;
                        err -= qj;
                    }
                }
                sh.shift = shift; sh.skip = skip; sh.bad = 0;
            }
            __syncthreads();
            if (sh.skip) continue;
            const int shift = sh.shift;
            rice_cost(sh, nb, order, [&](int i) {
                const int64_t r = lpc_residual(sh.s, i, order, sh.q, shift);
                if (r >= ((int64_t)1 << 31) || r <= -((int64_t)1 << 31)) { sh.bad = 1; return 0u; }
                return fold(r);
            });
            if (sh.bad) continue;                          // read after rice_cost's closing barrier: uniform
            consider(sh, SUB_LPC, order, 8 + 16 * order + 4 + 5 + kPrec * order);
        }
    }

    if (tid == 0) {
        uint8_t h[16];
        sh.best.bytes = frame_header(h, frame0 + f, nb, rcode) + (sh.best.bits + 7) / 8 + 2;
    }
    __syncthreads();
    uint32_t* dst = reinterpret_cast<uint32_t*>(desc + f);
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&sh.best);
    for (int i = tid; i < (int)(sizeof(FrameDesc) / 4); i += kThreads) dst[i] = src[i];
}

// off[f] = bytes of frames 0 .. f-1 of the batch; stats = {total, min, max} frame bytes
__global__ void __launch_bounds__(1024) flac_scan_kernel(const FrameDesc* __restrict__ desc, int nf,
                                                         int64_t* __restrict__ off, int64_t* __restrict__ stats) {
    __shared__ int64_t part[1024];
    __shared__ int mn[32], mx[32];
    const int tid = threadIdx.x, per = (nf + 1023) / 1024;
    const int f0 = min(nf, tid * per), f1 = min(nf, f0 + per);
    int64_t sum = 0;
    int lo = INT_MAX, hi = 0;
    for (int f = f0; f < f1; ++f) { const int b = desc[f].bytes; sum += b; lo = min(lo, b); hi = max(hi, b); }
    part[tid] = sum;
    lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
    if ((tid & 31) == 0) { mn[tid >> 5] = lo; mx[tid >> 5] = hi; }
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {                   // inclusive Hillis-Steele scan of the thread sums
        const int64_t v = tid >= d ? part[tid - d] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    int64_t o = part[tid] - sum;
    for (int f = f0; f < f1; ++f) { off[f] = o; o += desc[f].bytes; }
    if (tid == 0) {
        for (int w = 1; w < 32; ++w) { lo = min(lo, mn[w]); hi = max(hi, mx[w]); }
        stats[0] = part[1023]; stats[1] = lo; stats[2] = hi;
    }
}

// bits [pos, pos + n) of the big-endian bit string W = v (n in 1..32, v < 2^n, the bits still zero)
__device__ __forceinline__ void put_bits(uint32_t* W, uint32_t pos, uint32_t v, int n) {
    const uint32_t w = pos >> 5, o = pos & 31;
    if (o + n <= 32) {
        atomicOr(&W[w], v << (32 - o - n));
    } else {
        const int lo = (int)(o + n - 32);                  // bits that spill into the next word
        atomicOr(&W[w], v >> lo);
        atomicOr(&W[w + 1], v << (32 - lo));
    }
}

__device__ __forceinline__ uint32_t get_byte(const uint32_t* W, int b) { return (W[b >> 2] >> (24 - 8 * (b & 3))) & 0xFF; }

// a * b mod the CRC-16 polynomial x^16 + x^15 + x^2 + 1
__device__ __forceinline__ uint32_t crc16_mulmod(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int i = 15; i >= 0; --i) {
        r <<= 1;
        if (r & 0x10000) r ^= 0x18005;
        if (a >> i & 1) r ^= b;
    }
    return r;
}

// One CTA per frame of the batch: writes frame f at out + off[f].
__global__ void __launch_bounds__(kThreads) flac_write_kernel(const int16_t* __restrict__ pcm, int64_t ns,
                                                               int64_t frame0, int rcode,
                                                               const FrameDesc* __restrict__ desc,
                                                               const int64_t* __restrict__ off,
                                                               uint8_t* __restrict__ out) {
    __shared__ uint32_t W[kWords + 1];
    __shared__ int32_t s[kBlock];
    __shared__ uint16_t tab[256];
    __shared__ uint32_t scan[kThreads / 32];
    __shared__ uint32_t wcrc[kThreads / 32];
    __shared__ FrameDesc d;
    __shared__ int hlen;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, f = blockIdx.x;
    const int nb = (int)min((int64_t)kBlock, ns - (int64_t)f * kBlock);
    const int16_t* x = pcm + (size_t)f * kBlock;
    for (int i = tid; i < kWords + 1; i += kThreads) W[i] = 0;
    for (int i = tid; i < nb; i += kThreads) s[i] = x[i];
    {
        uint32_t c = (uint32_t)tid << 8;
        for (int b = 0; b < 8; ++b) c = c & 0x8000 ? (c << 1) ^ 0x8005 : c << 1;
        tab[tid] = (uint16_t)c;
    }
    if (tid == 0) d = desc[f];
    __syncthreads();
    if (tid == 0) {
        uint8_t h[16];
        hlen = frame_header(h, frame0 + f, nb, rcode);
        for (int i = 0; i < hlen; ++i) put_bits(W, 8 * i, h[i], 8);
    }
    __syncthreads();

    const uint32_t pos0 = 8u * hlen;
    const int order = d.order;
    if (tid == 0) {
        const int t6 = d.type == SUB_CONSTANT ? 0 : d.type == SUB_VERBATIM ? 1 : d.type == SUB_FIXED ? 8 | order : 32 | (order - 1);
        put_bits(W, pos0, (uint32_t)t6 << 1, 8);
    }
    if (d.type == SUB_CONSTANT) {
        if (tid == 0) put_bits(W, pos0 + 8, (uint16_t)s[0], 16);
    } else if (d.type == SUB_VERBATIM) {
        for (int i = tid; i < nb; i += kThreads) put_bits(W, pos0 + 8 + 16 * i, (uint16_t)s[i], 16);
    } else {
        if (tid < order) put_bits(W, pos0 + 8 + 16 * tid, (uint16_t)s[tid], 16);
        uint32_t rb = pos0 + 8 + 16 * order;
        if (d.type == SUB_LPC) {
            if (tid == 0) { put_bits(W, rb, kPrec - 1, 4); put_bits(W, rb + 4, d.shift, 5); }
            if (tid < order) put_bits(W, rb + 9 + kPrec * tid, (uint32_t)d.q[tid] & ((1u << kPrec) - 1), kPrec);
            rb += 9 + kPrec * order;
        }
        if (tid == 0) put_bits(W, rb, d.porder, 6);        // method 00, partition order
        const uint32_t codes = rb + 6;
        const int L = nb >> d.porder, C = (nb + kThreads - 1) / kThreads;
        const int i0 = max(tid * C, order), i1 = min(nb, (tid + 1) * C);
        uint32_t u[kPerThread], len = 0;
        for (int i = i0; i < i1; ++i) {
            const int64_t r = d.type == SUB_FIXED ? fixed_residual(s, i, order) : lpc_residual(s, i, order, d.q, d.shift);
            const int k = d.k[i / L];
            u[i - i0] = fold(r);
            len += (u[i - i0] >> k) + 1 + k;
        }
        // exclusive block scan of the code lengths
        uint32_t incl = len;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) scan[warp] = incl;
        __syncthreads();
        uint32_t pre = incl - len;
        for (int w = 0; w < warp; ++w) pre += scan[w];
        for (int i = i0; i < i1; ++i) {
            const int part = i / L, k = d.k[part];
            if (i == (part == 0 ? order : part * L)) put_bits(W, codes + 4 * part + pre, k, 4);
            const uint32_t v = u[i - i0], at = codes + 4 * (part + 1) + pre;
            put_bits(W, at + (v >> k), 1u << k | (v & ((1u << k) - 1)), k + 1);
            pre += (v >> k) + 1 + k;
        }
    }
    __syncthreads();

    // CRC-16 of bytes 0 .. nd-1: each thread runs the table over Lc bytes of the message right-aligned in
    // kThreads * Lc bytes (leading zeros leave a zero-init CRC unchanged); then crc(A || B) = crc(A) x^(8|B|) + crc(B)
    // combines the pieces in a tree.
    const int nd = d.bytes - 2, Lc = (nd + kThreads - 1) / kThreads, lead = kThreads * Lc - nd;
    uint32_t c = 0;
    for (int v = tid * Lc; v < (tid + 1) * Lc; ++v) {
        const uint32_t b = v >= lead ? get_byte(W, v - lead) : 0;
        c = ((c << 8) ^ tab[(c >> 8) ^ b]) & 0xFFFF;
    }
    uint32_t m = 1;                                        // x^(8 Lc) mod P: the register run over Lc zero bytes
    for (int v = 0; v < Lc; ++v) m = ((m << 8) ^ tab[m >> 8]) & 0xFFFF;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t other = __shfl_down_sync(0xffffffffu, c, o);
        if ((lane & (2 * o - 1)) == 0) c = crc16_mulmod(c, m) ^ other;
        m = crc16_mulmod(m, m);
    }
    if (lane == 0) wcrc[warp] = c;
    __syncthreads();

    uint8_t* dst = out + off[f];
    for (int b = tid; b < nd; b += kThreads) dst[b] = (uint8_t)get_byte(W, b);
    if (tid == 0) {
        uint32_t crc = wcrc[0];
        for (int w = 1; w < kThreads / 32; ++w) crc = crc16_mulmod(crc, m) ^ wcrc[w];
        dst[nd] = (uint8_t)(crc >> 8); dst[nd + 1] = (uint8_t)crc;
    }
}

void invalid(const std::string& s) { throw std::invalid_argument("encode_flac: " + s); }

constexpr int64_t kMaxSamples = ((int64_t)1 << 36) - 1;   // STREAMINFO's 36-bit total

}  // namespace

struct FlacEncoder::Impl {
    cudaStream_t st;
    Dev<int16_t> pcm;
    Dev<FrameDesc> desc;
    Dev<int64_t> off, stats;
    Dev<uint8_t> bytes;
    bool attr_set = false;
};

FlacEncoder::FlacEncoder(cudaStream_t st) : impl(new Impl()) { impl->st = st; }
FlacEncoder::~FlacEncoder() = default;

int64_t FlacEncoder::max_bytes(int64_t n) {
    return n < 0 ? 0 : kStreamHeader + (n + kBlock - 1) / kBlock * kMaxFrameBytes;
}

int64_t FlacEncoder::run(const int16_t* pcm, int64_t n, int sample_rate, const uint8_t* md5, uint8_t* out, int64_t cap,
                         int batch_frames, int64_t* n_out) {
    Impl& m = *impl;
    cudaStream_t st = m.st;
    *n_out = 0;
    if (sample_rate < 1 || sample_rate > (1 << 20) - 1) invalid("sample rate outside 1 .. 1048575 Hz");
    if (n < 0 || (n > 0 && !pcm)) invalid("no input");
    if (n > kMaxSamples) invalid("more than 2^36 - 1 samples");
    if (batch_frames < 1) invalid("batch_frames < 1");
    if (!out) cap = 0;
    const int rcode = rate_code(sample_rate);
    const int64_t frames = (n + kBlock - 1) / kBlock;
    const int B = (int)std::min<int64_t>(batch_frames, std::max<int64_t>(frames, 1));
    if (frames > 0) {
        m.pcm.ensure((size_t)B * kBlock); m.desc.ensure((size_t)B); m.off.ensure((size_t)B); m.stats.ensure(3);
        m.bytes.ensure((size_t)B * kMaxFrameBytes);
        if (!m.attr_set) {
            CUDA_CHECK(cudaFuncSetAttribute(flac_analyse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            kBlock * (int)sizeof(double)));
            m.attr_set = true;
        }
    }

    int64_t pos = kStreamHeader, fmin = 0, fmax = 0;
    for (int64_t f0 = 0; f0 < frames; f0 += B) {
        const int nf = (int)std::min<int64_t>(B, frames - f0);
        const int64_t s0 = f0 * kBlock, ns = std::min<int64_t>(n - s0, (int64_t)nf * kBlock);
        CUDA_CHECK(cudaMemcpyAsync(m.pcm.p, pcm + s0, (size_t)ns * sizeof(int16_t), cudaMemcpyHostToDevice, st));
        flac_analyse_kernel<<<nf, kThreads, kBlock * sizeof(double), st>>>(m.pcm.p, ns, f0, rcode, m.desc.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        flac_scan_kernel<<<1, 1024, 0, st>>>(m.desc.p, nf, m.off.p, m.stats.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        flac_write_kernel<<<nf, kThreads, 0, st>>>(m.pcm.p, ns, f0, rcode, m.desc.p, m.off.p, m.bytes.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        int64_t stats[3];
        CUDA_CHECK(cudaMemcpyAsync(stats, m.stats.p, sizeof(stats), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (pos + stats[0] <= cap) {
            CUDA_CHECK(cudaMemcpyAsync(out + pos, m.bytes.p, (size_t)stats[0], cudaMemcpyDeviceToHost, st));
            CUDA_CHECK(cudaStreamSynchronize(st));
        }
        pos += stats[0];
        fmin = f0 == 0 ? stats[1] : std::min(fmin, stats[1]);
        fmax = std::max(fmax, stats[2]);
    }
    *n_out = pos;
    if (cap < pos) invalid("output buffer too small");

    // "fLaC", the last-metadata-block flag with type 0 (STREAMINFO) and length 34, then STREAMINFO
    uint8_t h[kStreamHeader] = {'f', 'L', 'a', 'C', 0x80, 0, 0, 34};
    uint8_t* si = h + 8;
    si[0] = kBlock >> 8; si[1] = kBlock & 0xFF; si[2] = kBlock >> 8; si[3] = kBlock & 0xFF;
    for (int i = 0; i < 3; ++i) { si[4 + i] = (uint8_t)(fmin >> (16 - 8 * i)); si[7 + i] = (uint8_t)(fmax >> (16 - 8 * i)); }
    // 20 bits rate, 3 bits channels - 1 (0), 5 bits bits per sample - 1 (15), 36 bits total samples
    const uint64_t packed = (uint64_t)sample_rate << 44 | (uint64_t)15 << 36 | (uint64_t)n;
    for (int i = 0; i < 8; ++i) si[10 + i] = (uint8_t)(packed >> (56 - 8 * i));
    for (int i = 0; i < 16; ++i) si[18 + i] = md5 ? md5[i] : 0;
    std::memcpy(out, h, kStreamHeader);
    return pos;
}

}  // namespace xtts
