// FLAC encoder (see cond.h): mono 16-bit PCM -> a complete FLAC stream (RFC 9639), for TTSOutput.to_bytes("flac").
// (The decoder, for FLAC input, is the second half of this file.)
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

// tab[i] = the CRC-16 table entry of byte i (one entry per thread of a kThreads CTA)
__device__ __forceinline__ void crc16_table(uint16_t* tab) {
    uint32_t c = (uint32_t)threadIdx.x << 8;
    for (int b = 0; b < 8; ++b) c = c & 0x8000 ? (c << 1) ^ 0x8005 : c << 1;
    tab[threadIdx.x] = (uint16_t)c;
}

// CRC-16 of bytes 0 .. nd-1 (byte_at(i)) by the whole CTA; wcrc: kThreads / 32 words of shared memory.  Each thread runs
// the table over Lc bytes of the message right-aligned in kThreads * Lc bytes (leading zeros leave a zero-init CRC
// unchanged); then crc(A || B) = crc(A) x^(8|B|) + crc(B) combines the pieces in a tree.  Valid in thread 0.
template <class ByteAt>
__device__ uint32_t cta_crc16(ByteAt byte_at, int64_t nd, const uint16_t* tab, uint32_t* wcrc) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t Lc = (nd + kThreads - 1) / kThreads, lead = kThreads * Lc - nd;
    uint32_t c = 0;
    for (int64_t v = tid * Lc; v < (tid + 1) * Lc; ++v) {
        const uint32_t b = v >= lead ? byte_at(v - lead) : 0;
        c = ((c << 8) ^ tab[(c >> 8) ^ b]) & 0xFFFF;
    }
    uint32_t m = 1;                                        // x^(8 Lc) mod P: the register run over Lc zero bytes
    for (int64_t v = 0; v < Lc; ++v) m = ((m << 8) ^ tab[m >> 8]) & 0xFFFF;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t other = __shfl_down_sync(0xffffffffu, c, o);
        if ((lane & (2 * o - 1)) == 0) c = crc16_mulmod(c, m) ^ other;
        m = crc16_mulmod(m, m);
    }
    if (lane == 0) wcrc[warp] = c;
    __syncthreads();
    uint32_t crc = wcrc[0];
    for (int w = 1; w < kThreads / 32; ++w) crc = crc16_mulmod(crc, m) ^ wcrc[w];
    return crc;
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
    crc16_table(tab);
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

    const int nd = d.bytes - 2;
    const uint32_t crc = cta_crc16([&](int64_t b) { return get_byte(W, (int)b); }, nd, tab, wcrc);

    uint8_t* dst = out + off[f];
    for (int b = tid; b < nd; b += kThreads) dst[b] = (uint8_t)get_byte(W, b);
    if (tid == 0) { dst[nd] = (uint8_t)(crc >> 8); dst[nd + 1] = (uint8_t)crc; }
}

void invalid(const std::string& s) { throw std::invalid_argument("encode_flac: " + s); }

constexpr int64_t kMaxSamples = ((int64_t)1 << 36) - 1;   // STREAMINFO's 36-bit total

}  // namespace

struct FlacEncoder::Impl {
    cudaStream_t st;
    DBuf<int16_t> pcm;
    DBuf<FrameDesc> desc;
    DBuf<int64_t> off, stats;
    DBuf<uint8_t> bytes;
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

// ================================================================================================================
// FLAC decoder (see cond.h): a FLAC stream (RFC 9639) -> planar int32 samples.
//
// The host parses the ID3v2 tag and the metadata blocks (a handful of block headers) and uploads the stream.  Frame
// boundaries are found on the device: flac_sync_count_kernel tests every byte position of the frame region for a
// frame header (sync code, no reserved value, fields that agree with STREAMINFO, a correct CRC-8, a frame / sample
// number the total allows), flac_excl_scan_kernel and flac_sync_emit_kernel compact them into a position-ordered
// candidate list.  The host chains candidates by frame / sample number: the frame after a confirmed frame is taken
// to be the first later candidate with the next number.  Each batch of chained frames is then decoded one frame per
// thread (flac_parse_kernel: subframe headers, warm-up samples, LPC coefficients and the Rice / escape residuals, to
// the frame's end), its CRC-16 checked one CTA per frame (flac_crc_kernel), its predictors restored one thread per
// subframe (flac_restore_kernel: FIXED / LPC in int64, sample by sample, because the shift makes the recursion
// non-linear) and its channels decorrelated one CTA per frame (flac_decorrelate_kernel).  A frame is accepted only
// when every frame before it was and the previous one's parsed end is exactly its start, so a false sync inside a
// payload is found when the frame holding it is parsed past it: the batch is cut there and the next one starts at
// the parsed end.  The output is what a strictly sequential decoder returns, whatever the batch size.
namespace {

constexpr int kScanPer = 16;                               // byte positions per thread of the sync scan
constexpr int kMaxOrder = 32, kMaxChannels = 8;
constexpr int kParseThreads = 64;

struct StreamParams { int64_t total; int32_t rate, channels, bps, max_block; };
struct Cand { int64_t pos, num; int32_t bs, hlen, ca, var; };                 // a frame header
struct DFrame { int64_t pos, off; int32_t hlen, bs, ca, pad; };              // off: per-channel offset in the batch
struct DSub { int32_t type, order, shift, wasted, width; int32_t coef[kMaxOrder]; };
struct DRes { int64_t end; int32_t status, pad; };                           // end: the byte after the CRC-16

enum : int { D_OK = 0, D_TRUNC, D_PAD, D_TYPE, D_WASTED, D_ORDER, D_LPC, D_METHOD, D_RESID, D_RANGE, D_CRC };
const char* const kDecodeError[] = {"", "frame runs past the end of the data", "non-zero padding bit",
                                    "reserved subframe type", "wasted bits leave no sample bits",
                                    "predictor or partition order does not fit the block",
                                    "LPC precision 1111 or a negative LPC shift", "reserved residual coding method",
                                    "a residual does not fit 32 bits", "a decoded sample does not fit its bit depth",
                                    "CRC-16 mismatch"};

__constant__ int kSampleSizes[8] = {0, 8, 12, 0, 16, 20, 24, 32};
__constant__ int kRates[12] = {0, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};

// The frame header at byte p, read no further than `end`, into c; false if it is not a valid header of this stream.
__device__ bool frame_header_at(const uint8_t* __restrict__ d, int64_t p, int64_t end, const StreamParams& sp, Cand& c) {
    if (p + 4 > end || d[p] != 0xFF || (d[p + 1] & 0xFE) != 0xF8) return false;
    const int var = d[p + 1] & 1, b2 = d[p + 2], b3 = d[p + 3];
    const int bc = b2 >> 4, rc = b2 & 15, ca = b3 >> 4, sc = (b3 >> 1) & 7;
    if (bc == 0 || rc == 15 || ca > 10 || sc == 3 || (b3 & 1)) return false;
    if ((ca >= 8 ? 2 : ca + 1) != sp.channels || (sc && kSampleSizes[sc] != sp.bps)) return false;
    int64_t q = p + 4;
    if (q >= end) return false;
    const int b0 = d[q];
    int n = 1;
    uint64_t num = b0;
    if (b0 >= 0x80) {                                      // UTF-8-style: n leading ones, then n - 1 continuation bytes
        n = __clz(~((uint32_t)b0 << 24));
        if (n < 2 || n > (var ? 7 : 6) || q + n > end) return false;
        num = b0 & (0x7F >> n);
        for (int i = 1; i < n; ++i) {
            const int cb = d[q + i];
            if ((cb & 0xC0) != 0x80) return false;
            num = num << 6 | (cb & 0x3F);
        }
    }
    q += n;
    const int extra = (bc == 6 ? 1 : bc == 7 ? 2 : 0) + (rc == 12 ? 1 : (rc == 13 || rc == 14) ? 2 : 0);
    if (q + extra + 1 > end) return false;
    int bs;
    if (bc == 1) bs = 192;
    else if (bc <= 5) bs = 576 << (bc - 2);
    else if (bc == 6) bs = d[q++] + 1;
    else if (bc == 7) { bs = (d[q] << 8 | d[q + 1]) + 1; q += 2; }
    else bs = 256 << (bc - 8);
    int rate;
    if (rc == 12) rate = d[q++] * 1000;
    else if (rc == 13) { rate = d[q] << 8 | d[q + 1]; q += 2; }
    else if (rc == 14) { rate = (d[q] << 8 | d[q + 1]) * 10; q += 2; }
    else rate = rc ? kRates[rc] : sp.rate;
    if (rate != sp.rate || bs > sp.max_block) return false;
    uint32_t crc = 0;
    for (int64_t j = p; j < q; ++j) {
        crc ^= d[j];
        for (int b = 0; b < 8; ++b) crc = (crc & 0x80 ? (crc << 1) ^ 0x07 : crc << 1) & 0xFF;
    }
    if (crc != d[q]) return false;
    if (sp.total > 0 && (var ? num + bs > (uint64_t)sp.total : num >= (uint64_t)sp.total)) return false;
    c.pos = p; c.num = (int64_t)num; c.bs = bs; c.hlen = (int)(q + 1 - p); c.ca = ca; c.var = var;
    return true;
}

// mask[t] bit i = a frame header at p0 + kScanPer * t + i; counts[block] = headers found by the block
__global__ void __launch_bounds__(kThreads) flac_sync_count_kernel(const uint8_t* __restrict__ d, int64_t p0, int64_t end,
                                                                   StreamParams sp, uint16_t* __restrict__ mask,
                                                                   int64_t* __restrict__ counts) {
    __shared__ int part[kThreads / 32];
    const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x, base = p0 + t * kScanPer;
    uint32_t m = 0;
    Cand c;
    for (int i = 0; i < kScanPer; ++i)
        if (base + i < end && d[base + i] == 0xFF && frame_header_at(d, base + i, end, sp, c)) m |= 1u << i;
    if (base < end) mask[t] = (uint16_t)m;
    const int cnt = __reduce_add_sync(0xffffffffu, __popc(m));
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t s = 0;
        for (int w = 0; w < kThreads / 32; ++w) s += part[w];
        counts[blockIdx.x] = s;
    }
}

// v[0 .. n) -> its exclusive prefix sums; *total = the sum
__global__ void __launch_bounds__(1024) flac_excl_scan_kernel(int64_t* __restrict__ v, int64_t n, int64_t* __restrict__ total) {
    __shared__ int64_t part[1024];
    const int tid = threadIdx.x;
    const int64_t per = (n + 1023) / 1024, i0 = min(n, tid * per), i1 = min(n, i0 + per);
    int64_t sum = 0;
    for (int64_t i = i0; i < i1; ++i) sum += v[i];
    part[tid] = sum;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        const int64_t x = tid >= d ? part[tid - d] : 0;
        __syncthreads();
        part[tid] += x;
        __syncthreads();
    }
    int64_t o = part[tid] - sum;
    for (int64_t i = i0; i < i1; ++i) { const int64_t x = v[i]; v[i] = o; o += x; }
    if (tid == 1023) *total = part[1023];
}

// Writes every header found by flac_sync_count_kernel to out, in position order.
__global__ void __launch_bounds__(kThreads) flac_sync_emit_kernel(const uint8_t* __restrict__ d, int64_t p0, int64_t end,
                                                                  StreamParams sp, const uint16_t* __restrict__ mask,
                                                                  const int64_t* __restrict__ block_off,
                                                                  Cand* __restrict__ out) {
    __shared__ int part[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x, base = p0 + t * kScanPer;
    const uint32_t m = base < end ? mask[t] : 0;
    const int cnt = __popc(m);
    int incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += x;
    }
    if (lane == 31) part[warp] = incl;
    __syncthreads();
    int64_t o = block_off[blockIdx.x] + incl - cnt;
    for (int w = 0; w < warp; ++w) o += part[w];
    Cand c;
    for (int i = 0; i < kScanPer; ++i)
        if (m >> i & 1) {
            frame_header_at(d, base + i, end, sp, c);
            out[o++] = c;
        }
}

// MSB-first reader over the big-endian words of the stream; the buffer holds four zero words past the data, so a
// read that starts less than 64 bits past `lim` stays inside it, and callers check pos <= lim after each read.
struct BitReader {
    const uint32_t* __restrict__ w;
    int64_t pos, lim;                                      // bits
    __device__ __forceinline__ uint64_t peek() const {     // at least 33 valid bits at the top
        const int64_t i = pos >> 5;
        const uint64_t a = __byte_perm(w[i], 0, 0x0123), b = __byte_perm(w[i + 1], 0, 0x0123);
        return (a << 32 | b) << (pos & 31);
    }
    __device__ __forceinline__ uint32_t get(int n) {       // n in 0 .. 32
        if (n == 0) return 0;
        const uint32_t v = (uint32_t)(peek() >> (64 - n));
        pos += n;
        return v;
    }
    __device__ __forceinline__ int64_t sget(int n) {       // n in 1 .. 33, two's complement
        uint64_t v = n > 32 ? (uint64_t)get(n - 32) << 32 : 0;
        v |= get(n > 32 ? 32 : n);
        return (int64_t)(v << (64 - n)) >> (64 - n);
    }
    __device__ __forceinline__ bool room(int64_t bits) const { return pos + bits <= lim; }
};

template <class T>
__device__ int parse_residual(BitReader& br, int nb, int order, T* __restrict__ x) {
    if (!br.room(6)) return D_TRUNC;
    const int method = br.get(2);
    if (method > 1) return D_METHOD;
    const int pbits = method ? 5 : 4, esc = (1 << pbits) - 1, porder = br.get(4);
    if ((nb & ((1 << porder) - 1)) || (nb >> porder) < order) return D_ORDER;
    int i = order;
    for (int part = 0; part < 1 << porder; ++part) {
        const int cnt = (nb >> porder) - (part == 0 ? order : 0);
        if (!br.room(pbits)) return D_TRUNC;
        const int k = br.get(pbits);
        if (k == esc) {                                    // escape: raw signed values of n bits (0: all zero)
            if (!br.room(5)) return D_TRUNC;
            const int n = br.get(5);
            if (!br.room((int64_t)cnt * n)) return D_TRUNC;
            for (int j = 0; j < cnt; ++j) x[i++] = n ? (T)br.sget(n) : (T)0;
            continue;
        }
        for (int j = 0; j < cnt; ++j) {
            uint64_t q = 0, v = br.peek();
            while ((v >> 32) == 0) {                       // 32 or more zeros
                q += 32; br.pos += 32;
                if (br.pos > br.lim) return D_TRUNC;
                if (q >> (32 - k)) return D_RESID;
                v = br.peek();
            }
            const int z = __clzll(v);
            q += z; br.pos += z + 1;
            const uint32_t lo = br.get(k);
            if (br.pos > br.lim) return D_TRUNC;
            if (q >> (32 - k)) return D_RESID;             // the folded value would reach 2^32
            const uint32_t u = (uint32_t)(q << k) | lo;
            x[i++] = (T)((int64_t)(u >> 1) ^ -(int64_t)(u & 1));
        }
    }
    return D_OK;
}

// One thread per frame of the batch: parses every subframe into work (warm-up or raw samples, residuals) and subs.
template <class T>
__global__ void __launch_bounds__(kParseThreads) flac_parse_kernel(const uint32_t* __restrict__ words, int64_t lim_bytes,
                                                                   const DFrame* __restrict__ frames, int nf, int C,
                                                                   int bps, int64_t bn, T* __restrict__ work,
                                                                   DSub* __restrict__ subs, DRes* __restrict__ res) {
    const int f = blockIdx.x * kParseThreads + threadIdx.x;
    if (f >= nf) return;
    const DFrame F = frames[f];
    BitReader br{words, (F.pos + F.hlen) * 8, lim_bytes * 8};
    int st = D_OK;
    for (int c = 0; c < C && st == D_OK; ++c) {
        const bool side = (F.ca == 8 && c == 1) || (F.ca == 9 && c == 0) || (F.ca == 10 && c == 1);
        const int sbits = bps + side, nb = F.bs;
        T* x = work + c * bn + F.off;
        DSub& s = subs[(int64_t)f * C + c];
        if (!br.room(8)) { st = D_TRUNC; break; }
        const uint32_t h = br.get(8);
        if (h >> 7) { st = D_PAD; break; }
        const int t = (h >> 1) & 63;
        int wasted = 0;
        if (h & 1) {                                       // wasted bits, unary: w - 1 zeros, then a one
            wasted = 1;
            for (;;) {
                if (!br.room(1)) { st = D_TRUNC; break; }
                if (br.get(1)) break;
                if (++wasted >= sbits) { st = D_WASTED; break; }
            }
            if (st) break;
        }
        const int b = sbits - wasted;
        s.type = t; s.wasted = wasted; s.width = b; s.order = 0; s.shift = 0;
        if (t == 0) {
            if (!br.room(b)) { st = D_TRUNC; break; }
            x[0] = (T)br.sget(b);
        } else if (t == 1) {
            if (!br.room((int64_t)b * nb)) { st = D_TRUNC; break; }
            for (int i = 0; i < nb; ++i) x[i] = (T)br.sget(b);
        } else if ((t >= 8 && t <= 12) || t >= 32) {
            const int order = t <= 12 ? t - 8 : t - 31;
            if (order > nb) { st = D_ORDER; break; }
            if (!br.room((int64_t)b * order)) { st = D_TRUNC; break; }
            for (int i = 0; i < order; ++i) x[i] = (T)br.sget(b);
            s.order = order;
            if (t >= 32) {
                if (!br.room(9)) { st = D_TRUNC; break; }
                const int prec = br.get(4) + 1, shift = (int)br.sget(5);
                if (prec == 16 || shift < 0) { st = D_LPC; break; }
                if (!br.room((int64_t)prec * order)) { st = D_TRUNC; break; }
                for (int j = 0; j < order; ++j) s.coef[j] = (int32_t)br.sget(prec);
                s.shift = shift;
            }
            st = parse_residual(br, nb, order, x);
        } else {
            st = D_TYPE;
        }
    }
    int64_t end = 0;
    if (st == D_OK) {
        const int pad = (int)(-br.pos & 7);
        if (br.get(pad)) st = D_PAD;
        end = br.pos / 8 + 2;
        if (end > lim_bytes) st = D_TRUNC;
    }
    res[f].end = end;
    res[f].status = st;
}

// One CTA per frame whose parse succeeded: the CRC-16 of its bytes against the two that follow them.
__global__ void __launch_bounds__(kThreads) flac_crc_kernel(const uint8_t* __restrict__ d, const DFrame* __restrict__ frames,
                                                            DRes* __restrict__ res) {
    __shared__ uint16_t tab[256];
    __shared__ uint32_t wcrc[kThreads / 32];
    const int f = blockIdx.x;
    if (res[f].status != D_OK) return;
    const int64_t p = frames[f].pos, end = res[f].end;
    crc16_table(tab);
    __syncthreads();
    const uint32_t crc = cta_crc16([&](int64_t i) { return (uint32_t)d[p + i]; }, end - 2 - p, tab, wcrc);
    if (threadIdx.x == 0 && crc != ((uint32_t)d[end - 2] << 8 | d[end - 1])) res[f].status = D_CRC;
}

// One thread per subframe: CONSTANT fill, FIXED / LPC restoration in int64 with every sample inside its width.
template <class T>
__global__ void __launch_bounds__(kParseThreads) flac_restore_kernel(const DFrame* __restrict__ frames, int nf, int C,
                                                                     int64_t bn, const DSub* __restrict__ subs,
                                                                     T* __restrict__ work, DRes* __restrict__ res) {
    const int64_t idx = (int64_t)blockIdx.x * kParseThreads + threadIdx.x;
    if (idx >= (int64_t)nf * C) return;
    const int f = (int)(idx / C), c = (int)(idx % C);
    if (res[f].status != D_OK) return;
    const DFrame F = frames[f];
    const DSub& s = subs[idx];
    T* x = work + c * bn + F.off;
    const int nb = F.bs, order = s.order, t = s.type;
    if (t == 0) {
        const T v = x[0];
        for (int i = 1; i < nb; ++i) x[i] = v;
        return;
    }
    if (t == 1) return;
    const int64_t hi = ((int64_t)1 << (s.width - 1)) - 1, lo = -hi - 1;
    if (t <= 12) {
        for (int i = order; i < nb; ++i) {
            int64_t p = 0;
            switch (order) {
                case 1: p = x[i - 1]; break;
                case 2: p = 2 * (int64_t)x[i - 1] - x[i - 2]; break;
                case 3: p = 3 * ((int64_t)x[i - 1] - x[i - 2]) + x[i - 3]; break;
                case 4: p = 4 * ((int64_t)x[i - 1] + x[i - 3]) - 6 * (int64_t)x[i - 2] - x[i - 4]; break;
                default: break;
            }
            const int64_t v = (int64_t)x[i] + p;
            if (v < lo || v > hi) { res[f].status = D_RANGE; return; }
            x[i] = (T)v;
        }
        return;
    }
    int32_t q[kMaxOrder];
    for (int j = 0; j < order; ++j) q[j] = s.coef[j];
    const int shift = s.shift;
    for (int i = order; i < nb; ++i) {
        int64_t acc = 0;
        for (int j = 0; j < order; ++j) acc += (int64_t)q[j] * x[i - 1 - j];
        const int64_t v = (int64_t)x[i] + (acc >> shift);
        if (v < lo || v > hi) { res[f].status = D_RANGE; return; }
        x[i] = (T)v;
    }
}

// One CTA per frame: wasted bits back, inter-channel decorrelation, every sample inside the stream's bit depth; out
// may alias work (each thread reads all channels of its samples before writing them).
template <class T>
__global__ void __launch_bounds__(kThreads) flac_decorrelate_kernel(const DFrame* __restrict__ frames, int C, int bps,
                                                                    int64_t bn, const DSub* __restrict__ subs,
                                                                    const T* work, int32_t* out, DRes* __restrict__ res) {
    const int f = blockIdx.x;
    if (res[f].status != D_OK) return;
    const DFrame F = frames[f];
    int ws[kMaxChannels];
    for (int c = 0; c < C; ++c) ws[c] = subs[(int64_t)f * C + c].wasted;
    const int64_t lim = (int64_t)1 << (bps - 1);
    bool bad = false;
    for (int i = threadIdx.x; i < F.bs; i += kThreads) {
        int64_t v[kMaxChannels];
        for (int c = 0; c < C; ++c) v[c] = (int64_t)work[c * bn + F.off + i] * ((int64_t)1 << ws[c]);
        if (F.ca == 8) v[1] = v[0] - v[1];
        else if (F.ca == 9) v[0] += v[1];
        else if (F.ca == 10) {
            const int64_t m = v[0] * 2 + (v[1] & 1);
            v[0] = (m + v[1]) >> 1;
            v[1] = (m - v[1]) >> 1;
        }
        for (int c = 0; c < C; ++c) {
            bad |= v[c] < -lim || v[c] >= lim;
            out[c * bn + F.off + i] = (int32_t)v[c];
        }
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) res[f].status = D_RANGE;
}

void dinvalid(const std::string& s) { throw std::invalid_argument("decode_flac: " + s); }

uint64_t be(const uint8_t* p, int n) {
    uint64_t v = 0;
    for (int i = 0; i < n; ++i) v = v << 8 | p[i];
    return v;
}

}  // namespace

struct FlacDecoder::Impl {
    cudaStream_t st;
    DBuf<uint32_t> words;
    DBuf<uint16_t> mask;
    DBuf<int64_t> counts, total;
    DBuf<Cand> cands;
    DBuf<DFrame> frames;
    DBuf<DSub> subs;
    DBuf<DRes> res;
    DBuf<int32_t> w32;
    DBuf<int64_t> w64;
};

FlacDecoder::FlacDecoder(cudaStream_t st) : impl(new Impl()) { impl->st = st; }
FlacDecoder::~FlacDecoder() = default;

int64_t FlacDecoder::run(const uint8_t* data, int64_t n, int32_t* out, int64_t cap, int batch_frames,
                         xtts_flac_info* info) {
    Impl& m = *impl;
    cudaStream_t st = m.st;
    std::memset(info, 0, sizeof(*info));
    if (n < 0 || (n > 0 && !data)) dinvalid("no input");
    if (batch_frames < 1) dinvalid("batch_frames < 1");
    if (!out) cap = 0;

    // ---- ID3v2 tag, "fLaC", metadata blocks (STREAMINFO first)
    int64_t pos = 0;
    if (n >= 3 && std::memcmp(data, "ID3", 3) == 0) {
        if (n < 10 || ((data[6] | data[7] | data[8] | data[9]) & 0x80)) dinvalid("bad ID3v2 header");
        pos = 10 + ((int64_t)data[6] << 21 | data[7] << 14 | data[8] << 7 | data[9]) + (data[5] & 0x10 ? 10 : 0);
    }
    if (pos + 4 > n || std::memcmp(data + pos, "fLaC", 4) != 0) dinvalid("no fLaC marker");
    pos += 4;
    bool last = false, have_si = false;
    StreamParams sp{};
    int min_block = 0;
    while (!last) {
        if (pos + 4 > n) dinvalid("truncated metadata");
        last = data[pos] & 0x80;
        const int type = data[pos] & 0x7F;
        const int64_t len = (int64_t)be(data + pos + 1, 3);
        if (type == 127) dinvalid("metadata block type 127");
        if (pos + 4 + len > n) dinvalid("truncated metadata");
        if (!have_si) {
            if (type != 0 || len != 34) dinvalid("the first metadata block is not a 34-byte STREAMINFO");
            const uint8_t* b = data + pos + 4;
            const uint64_t v = be(b + 10, 8);
            min_block = (int)be(b, 2);
            sp.max_block = (int)be(b + 2, 2);
            sp.rate = (int)(v >> 44);
            sp.channels = (int)((v >> 41) & 7) + 1;
            sp.bps = (int)((v >> 36) & 31) + 1;
            sp.total = (int64_t)(v & (((uint64_t)1 << 36) - 1));
            info->sample_rate = sp.rate; info->channels = sp.channels; info->bits_per_sample = sp.bps;
            info->min_block = min_block; info->max_block = sp.max_block;
            std::memcpy(info->md5, b + 18, 16);
            have_si = true;
        }
        pos += 4 + len;
    }
    if (sp.rate == 0 || sp.bps < 4 || min_block < 16 || sp.max_block < min_block) dinvalid("bad STREAMINFO");
    const int C = sp.channels;
    const int64_t fstart = pos;
    int64_t fend = n;                                      // frames end here (with a known total, trailing bytes are ignored)
    if (sp.total == 0 && n - fstart >= 128 && std::memcmp(data + n - 128, "TAG", 3) == 0) fend = n - 128;
    // every frame takes at least 9 bytes, so a total the data cannot hold is wrong
    if (sp.total > ((fend - fstart) / 9) * sp.max_block) dinvalid("STREAMINFO's total does not fit in the data");
    info->total_samples = sp.total;                        // (only once it is plausible: callers allocate it)
    if (sp.total > 0 && cap < C * sp.total) dinvalid("output buffer too small");

    // ---- the stream on the device, every frame header in it
    const int64_t nwords = (n + 3) / 4 + 4, tail = std::min<int64_t>(nwords, 5);
    m.words.ensure((size_t)nwords);
    CUDA_CHECK(cudaMemsetAsync(m.words.p + nwords - tail, 0, (size_t)tail * sizeof(uint32_t), st));
    CUDA_CHECK(cudaMemcpyAsync(m.words.p, data, (size_t)n, cudaMemcpyHostToDevice, st));
    const uint8_t* d = reinterpret_cast<const uint8_t*>(m.words.p);
    std::vector<Cand> cand;
    if (fend > fstart) {
        const int64_t nthr = (fend - fstart + kScanPer - 1) / kScanPer, nblk = (nthr + kThreads - 1) / kThreads;
        m.mask.ensure((size_t)nthr); m.counts.ensure((size_t)nblk); m.total.ensure(1);
        flac_sync_count_kernel<<<(unsigned)nblk, kThreads, 0, st>>>(d, fstart, fend, sp, m.mask.p, m.counts.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        flac_excl_scan_kernel<<<1, 1024, 0, st>>>(m.counts.p, nblk, m.total.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        int64_t ncand = 0;
        CUDA_CHECK(cudaMemcpyAsync(&ncand, m.total.p, sizeof(ncand), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (ncand > 0) {
            m.cands.ensure((size_t)ncand);
            flac_sync_emit_kernel<<<(unsigned)nblk, kThreads, 0, st>>>(d, fstart, fend, sp, m.mask.p, m.counts.p, m.cands.p);
            COUNT_LAUNCH(); KERNEL_CHECK();
            cand.resize((size_t)ncand);
            CUDA_CHECK(cudaMemcpyAsync(cand.data(), m.cands.p, (size_t)ncand * sizeof(Cand), cudaMemcpyDeviceToHost, st));
            CUDA_CHECK(cudaStreamSynchronize(st));
        }
    }

    // ---- batches of chained frames
    const bool wide = sp.bps == 32;                        // the side channel of 32-bit audio needs 33 bits
    const int64_t batch_cap = (int64_t)batch_frames * 4096;
    std::vector<std::vector<int32_t>> staged(sp.total == 0 ? C : 0);   // total unknown: the samples wait here
    std::vector<int32_t> tmp;
    int64_t done = 0, nframes = 0, start = fstart;
    int strategy = -1, block = -1;
    bool must_end = false;
    std::vector<DFrame> B;
    std::vector<const Cand*> BC;
    std::vector<DRes> R;
    while (sp.total > 0 ? done < sp.total : start < fend) {
        auto it = std::lower_bound(cand.begin(), cand.end(), start, [](const Cand& c, int64_t p) { return c.pos < p; });
        if (it == cand.end() || it->pos != start) dinvalid("no valid frame header at byte " + std::to_string(start));
        size_t k = (size_t)(it - cand.begin());
        const int strat = strategy >= 0 ? strategy : cand[k].var;
        B.clear(); BC.clear();
        int64_t bo = 0, tdone = done, tframes = nframes;
        for (;;) {
            const Cand& c = cand[k];
            B.push_back({c.pos, bo, c.hlen, c.bs, c.ca, 0});
            BC.push_back(&c);
            bo += c.bs; tdone += c.bs; ++tframes;
            if ((sp.total > 0 && tdone >= sp.total) || (int)B.size() >= batch_frames) break;
            const int64_t want = strat ? tdone : tframes;
            size_t j = k + 1;
            while (j < cand.size() && !(cand[j].var == strat && cand[j].num == want)) ++j;
            if (j == cand.size() || (bo + cand[j].bs) * C > batch_cap) break;
            k = j;
        }
        const int nf = (int)B.size();
        const int64_t bn = bo;
        m.frames.ensure((size_t)nf); m.subs.ensure((size_t)nf * C); m.res.ensure((size_t)nf);
        m.w32.ensure((size_t)(bn * C));
        if (wide) m.w64.ensure((size_t)(bn * C));
        CUDA_CHECK(cudaMemcpyAsync(m.frames.p, B.data(), nf * sizeof(DFrame), cudaMemcpyHostToDevice, st));
        const unsigned g1 = (unsigned)((nf + kParseThreads - 1) / kParseThreads);
        const unsigned g2 = (unsigned)(((int64_t)nf * C + kParseThreads - 1) / kParseThreads);
        if (wide) flac_parse_kernel<<<g1, kParseThreads, 0, st>>>(m.words.p, fend, m.frames.p, nf, C, sp.bps, bn, m.w64.p, m.subs.p, m.res.p);
        else flac_parse_kernel<<<g1, kParseThreads, 0, st>>>(m.words.p, fend, m.frames.p, nf, C, sp.bps, bn, m.w32.p, m.subs.p, m.res.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        flac_crc_kernel<<<nf, kThreads, 0, st>>>(d, m.frames.p, m.res.p);
        COUNT_LAUNCH(); KERNEL_CHECK();
        if (wide) {
            flac_restore_kernel<<<g2, kParseThreads, 0, st>>>(m.frames.p, nf, C, bn, m.subs.p, m.w64.p, m.res.p);
            COUNT_LAUNCH(); KERNEL_CHECK();
            flac_decorrelate_kernel<<<nf, kThreads, 0, st>>>(m.frames.p, C, sp.bps, bn, m.subs.p, (const int64_t*)m.w64.p, m.w32.p, m.res.p);
        } else {
            flac_restore_kernel<<<g2, kParseThreads, 0, st>>>(m.frames.p, nf, C, bn, m.subs.p, m.w32.p, m.res.p);
            COUNT_LAUNCH(); KERNEL_CHECK();
            flac_decorrelate_kernel<<<nf, kThreads, 0, st>>>(m.frames.p, C, sp.bps, bn, m.subs.p, (const int32_t*)m.w32.p, m.w32.p, m.res.p);
        }
        COUNT_LAUNCH(); KERNEL_CHECK();
        R.resize((size_t)nf);
        CUDA_CHECK(cudaMemcpyAsync(R.data(), m.res.p, nf * sizeof(DRes), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));

        // accept the frames a sequential decoder reaches: each starts where the one before it ends
        const int64_t done0 = done;
        int acc = 0;
        for (int i = 0; i < nf; ++i) {
            const Cand& c = *BC[i];
            const std::string at = " in the frame at byte " + std::to_string(c.pos);
            if (R[i].status != D_OK) dinvalid(kDecodeError[R[i].status] + at);
            if (strategy < 0) strategy = c.var;
            if (c.var != strategy) dinvalid("blocking strategy changed" + at);
            if (c.num != (strategy ? done : nframes)) dinvalid("frame number out of sequence" + at);
            if (must_end) dinvalid("a block size changed before the last frame of a fixed-blocksize stream");
            if (!strategy) {
                if (block < 0) block = c.bs;
                else if (c.bs != block) must_end = true;
            }
            if (sp.total > 0 && done + c.bs > sp.total) dinvalid("frames hold more samples than STREAMINFO says");
            done += c.bs; ++nframes; ++acc;
            start = R[i].end;
            if (i + 1 < nf && B[i + 1].pos != start) break;
        }
        const int64_t na = B[acc - 1].off + B[acc - 1].bs;  // the accepted frames: the batch's first na samples
        if (sp.total > 0) {
            CUDA_CHECK(cudaMemcpy2DAsync(out + done0, (size_t)sp.total * 4, m.w32.p, (size_t)bn * 4, (size_t)na * 4, C,
                                         cudaMemcpyDeviceToHost, st));
        } else {
            tmp.resize((size_t)(na * C));
            CUDA_CHECK(cudaMemcpy2DAsync(tmp.data(), (size_t)na * 4, m.w32.p, (size_t)bn * 4, (size_t)na * 4, C,
                                         cudaMemcpyDeviceToHost, st));
        }
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (sp.total == 0)
            for (int c = 0; c < C; ++c) staged[c].insert(staged[c].end(), tmp.begin() + c * na, tmp.begin() + (c + 1) * na);
    }
    info->total_samples = done;
    if (sp.total == 0) {
        if (cap < C * done) dinvalid("output buffer too small");
        for (int c = 0; c < C && done > 0; ++c) std::memcpy(out + c * done, staged[c].data(), (size_t)done * sizeof(int32_t));
    }
    return done;
}

}  // namespace xtts
