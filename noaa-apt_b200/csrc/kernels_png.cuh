// Kernels of the PNG encoder (png.hpp, DESIGN.md §11).  Every kernel's output is a pure function of its inputs: the
// encoder's bytes do not depend on launch geometry, scheduling or the device.
#pragma once

#include <cstdint>

#include "launch.hpp"
#include "png.hpp"

namespace aptb200 {

constexpr u32 kPngWindow = 32768;
constexpr u32 kPngMaxMatch = 258;
constexpr u32 kPngMinMatch = 4;
constexpr u32 kPngSpan = 32736;        // positions one match CTA decides: span + window < 0xFFFF (u16 head offsets)
constexpr u32 kPngHdrWords = 80;       // a block header is at most 17 + 57 + 316 * 7 = 2286 bits
constexpr u32 kPngLit = 286, kPngDist = 30, kPngCl = 19;
constexpr u32 kPngEmitThreads = 256;
constexpr u32 kPngCrcChunk = 1024;     // bytes per thread of the CRC pass
constexpr u32 kPngDeflateBase = 43;    // byte offset of the deflate stream in the file

__constant__ unsigned char c_png_len_sym[kPngMaxMatch + 1];   // match length -> length code - 257
__constant__ uint16_t c_png_len_base[29];
__constant__ unsigned char c_png_len_extra[29];
__constant__ uint16_t c_png_dist_base[30];
__constant__ unsigned char c_png_dist_extra[30];
__constant__ unsigned char c_png_cl_order[19];
__constant__ u32 c_png_crc_table[256];
__constant__ u32 c_png_x2n[32];                               // x^(2^k) mod P, reflected (zlib's x2n_table)

// Bounds-checking build (-DAPTB200_PNG_CHECK, tools/png_bounds_check.sh): every global and shared index of the encoder is
// checked against its image's region of the buffer (PngImage: n + 16 bytes of f, n positions, height * width * in_ch
// pixels, out_bytes of out, nblocks blocks); a violation sets a bit of g_png_violation (no fault) and the encode then
// fails with APT_ERR_CUDA.  Ordinary builds compile the checks away.
#ifdef APTB200_PNG_CHECK
__device__ u32 g_png_violation;
#define PNG_CHECK(cond, bit)                                                  \
    do {                                                                      \
        if (!(cond)) atomicOr(&::aptb200::g_png_violation, 1u << (bit));      \
    } while (0)
#else
#define PNG_CHECK(cond, bit) \
    do {                     \
    } while (0)
#endif

// The image of a global index (row, span, block or CRC chunk): the last image whose first index is <= key.
template <u32 PngImage::*First>
__device__ __forceinline__ u32 png_image_of(const PngImage *__restrict__ im, u32 g, u32 key) {
    u32 lo = 0, hi = g;
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) / 2;
        if (im[mid].*First <= key) lo = mid;
        else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ u32 png_dist_sym(u32 d) {   // d >= 1
    const u32 dd = d - 1;
    if (dd < 4) return dd;
    const u32 k = 31 - __clz(dd);
    return 2 * k + ((dd >> (k - 1)) & 1);
}

// ------------------------------------------------------------------------------------------------------ 1. filter

__device__ __forceinline__ int png_paeth(int a, int b, int c) {
    const int p = a + b - c;
    const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// One warp per row of any image of the group: the five residual sums, the winner (ties to the lower type) and the row of
// F it gives; the warp of an image's last row also zeroes the 16 bytes of padding after its stream.
// CIN: channels of the input, C: channels written (C = 3, CIN = 4 drops alpha).
template <int CIN, int C>
__global__ void __launch_bounds__(256) k_png_filter(const PngImage *__restrict__ im, u32 g, u32 rows, u32 width, int fixed,
                                                    unsigned char *__restrict__ f_all) {
    const u32 lane = threadIdx.x & 31;
    const u32 gr = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (gr >= rows) return;
    const PngImage I = im[png_image_of<&PngImage::row0>(im, g, gr)];
    const u32 r = gr - I.row0;
    const unsigned char *__restrict__ px = I.px;
    unsigned char *__restrict__ f = f_all + I.pos;
    const u64 R = static_cast<u64>(width) * C;
    const u64 rin = static_cast<u64>(width) * CIN;
    if (r + 1 == I.height && lane < 16) f[I.n + lane] = 0;
    auto get = [&](u32 rr, u64 x) -> int {
        const u64 k = CIN == C ? rr * rin + x : rr * rin + (x / 3) * 4 + x % 3;
        PNG_CHECK(k < static_cast<u64>(I.height) * rin, 0);
        return px[k];
    };
    auto res = [&](int t, u64 x) -> u32 {
        const int cur = get(r, x);
        const int a = x >= static_cast<u64>(C) ? get(r, x - C) : 0;
        const int b = r ? get(r - 1, x) : 0;
        const int c = (r && x >= static_cast<u64>(C)) ? get(r - 1, x - C) : 0;
        int p = 0;
        switch (t) {
        case 1: p = a; break;
        case 2: p = b; break;
        case 3: p = (a + b) >> 1; break;
        case 4: p = png_paeth(a, b, c); break;
        default: break;
        }
        return static_cast<u32>(cur - p) & 0xFFu;
    };
    int type = fixed;
    if (fixed < 0) {
        u32 s[5] = {0, 0, 0, 0, 0};
        for (u64 x = lane; x < R; x += 32) {
            const int cur = get(r, x);
            const int a = x >= static_cast<u64>(C) ? get(r, x - C) : 0;
            const int b = r ? get(r - 1, x) : 0;
            const int c = (r && x >= static_cast<u64>(C)) ? get(r - 1, x - C) : 0;
            const int pred[5] = {0, a, b, (a + b) >> 1, png_paeth(a, b, c)};
#pragma unroll
            for (int t = 0; t < 5; ++t) {
                const u32 v = static_cast<u32>(cur - pred[t]) & 0xFFu;
                s[t] += min(v, 256u - v);
            }
        }
#pragma unroll
        for (int t = 0; t < 5; ++t)
            for (int o = 16; o; o >>= 1) s[t] += __shfl_xor_sync(0xFFFFFFFFu, s[t], o);
        type = 0;
#pragma unroll
        for (int t = 1; t < 5; ++t)
            if (s[t] < s[type]) type = t;
    }
    unsigned char *row = f + static_cast<u64>(r) * (R + 1);
    PNG_CHECK(static_cast<u64>(r + 1) * (R + 1) <= I.n, 1);
    if (lane == 0) row[0] = static_cast<unsigned char>(type);
    for (u64 x = lane; x < R; x += 32) row[1 + x] = static_cast<unsigned char>(res(type, x));
}

// ------------------------------------------------------------------------------------------------------ 3. matches

__device__ __forceinline__ u32 png_ld32(const unsigned char *f, u32 pos, u32 n) {   // 4 bytes at any offset (F is padded)
    const u32 *w = reinterpret_cast<const u32 *>(f + (pos & ~3u));
    PNG_CHECK((pos & ~3u) + 8ull <= n + 16ull, 2);
    return __funnelshift_r(w[0], w[1], (pos & 3u) * 8);
}

// One warp per span of kPngSpan positions of one image (each image's positions are cut into spans of its own).  It walks the window before the span and the span itself 32 positions at a
// time with a head table (last position of each hash, as a u16 offset from the walk's start) in shared memory; lanes
// with the same hash in one step resolve among themselves with __match_any_sync.  Every position with a hash updates the
// head, so m(i) is the same whatever the parse does.  Positions of the span get lcode (0 or l - 3) and dist (d - 1).
__global__ void __launch_bounds__(32) k_png_match(const PngImage *__restrict__ im, u32 g, const unsigned char *__restrict__ f_all,
                                                  u32 block_bytes, unsigned char *__restrict__ lcode_all,
                                                  uint16_t *__restrict__ dist_all) {
    extern __shared__ uint16_t head[];   // 32768 entries
    const PngImage &I = im[png_image_of<&PngImage::span0>(im, g, blockIdx.x)];
    const u32 n = I.n;
    const unsigned char *__restrict__ f = f_all + I.pos;
    unsigned char *__restrict__ lcode = lcode_all + I.pos;
    uint16_t *__restrict__ dist = dist_all + I.pos;
    const u32 lane = threadIdx.x;
    const u32 s = (blockIdx.x - I.span0) * kPngSpan;
    const u32 e = min(n, s + kPngSpan);
    const u32 b = s > kPngWindow ? s - kPngWindow : 0;
    for (u32 k = lane; k < 32768; k += 32) head[k] = 0xFFFFu;
    __syncwarp();
    for (u32 base = b; base < e; base += 32) {
        const u32 i = base + lane;
        const bool valid = i < e && i + 2 < n;
        u32 h = 0x8000u + lane;   // lanes without a hash get keys no hash equals
        if (valid) h = ((static_cast<u32>(f[i]) << 10) ^ (static_cast<u32>(f[i + 1]) << 5) ^ f[i + 2]) & 0x7FFFu;
        const u32 peers = __match_any_sync(0xFFFFFFFFu, h);
        const u32 lower = peers & ((1u << lane) - 1u);
        int cand = -1;
        if (valid) {
            if (lower) cand = static_cast<int>(base + 31 - __clz(lower));
            else if (head[h] != 0xFFFFu) cand = static_cast<int>(b + head[h]);
        }
        __syncwarp();
        const u32 higher = peers & ~((2u << lane) - 1u);
        if (valid && !higher) head[h] = static_cast<uint16_t>(i - b);
        __syncwarp();
        if (i < s || i >= e) continue;
        u32 len = 0;
        if (cand >= 0 && static_cast<u32>(cand) + kPngWindow >= i) {
            const u32 bend = min(n, (i / block_bytes + 1) * block_bytes);
            const u32 cap = min(kPngMaxMatch, bend - i);
            const u32 j = static_cast<u32>(cand);
            while (len < cap) {
                const u32 x = png_ld32(f, j + len, n) ^ png_ld32(f, i + len, n);
                if (x) {
                    len += (__ffs(x) - 1) >> 3;
                    break;
                }
                len += 4;
            }
            len = min(len, cap);
        }
        PNG_CHECK(i < n && (len < kPngMinMatch || i + len <= n), 3);
        if (len >= kPngMinMatch) {
            lcode[i] = static_cast<unsigned char>(len - 3);
            dist[i] = static_cast<uint16_t>(i - static_cast<u32>(cand) - 1);
        } else {
            lcode[i] = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------------ 4. parse

// One CTA per deflate block of the group: thread 0 walks the greedy jump chain over the block's lcode in shared memory and marks the
// token positions; then the block's literal/length and distance histograms (end of block counted).
__global__ void __launch_bounds__(256) k_png_parse(const PngImage *__restrict__ im, u32 g, const unsigned char *__restrict__ f_all,
                                                   const unsigned char *__restrict__ lcode_all, const uint16_t *__restrict__ dist_all,
                                                   u32 block_bytes, unsigned char *__restrict__ flag_all, u32 *__restrict__ hist) {
    extern __shared__ unsigned char sl[];   // block_bytes
    __shared__ u32 h[kPngLit + kPngDist];
    const PngImage &I = im[png_image_of<&PngImage::blk0>(im, g, blockIdx.x)];
    const u32 n = I.n;
    const unsigned char *__restrict__ f = f_all + I.pos;
    const unsigned char *__restrict__ lcode = lcode_all + I.pos;
    const uint16_t *__restrict__ dist = dist_all + I.pos;
    unsigned char *__restrict__ flag = flag_all + I.pos;
    const u32 start = (blockIdx.x - I.blk0) * block_bytes;
    const u32 len = min(block_bytes, n - start);
    PNG_CHECK(start + len <= n && blockIdx.x - I.blk0 < I.nblocks, 13);
    for (u32 k = threadIdx.x; k < kPngLit + kPngDist; k += blockDim.x) h[k] = 0;
    const u32 nw = len / 4;
    const u32 *src = reinterpret_cast<const u32 *>(lcode + start);   // pos and start are multiples of 4: aligned
    for (u32 k = threadIdx.x; k < nw; k += blockDim.x) reinterpret_cast<u32 *>(sl)[k] = src[k];
    for (u32 k = 4 * nw + threadIdx.x; k < len; k += blockDim.x) sl[k] = lcode[start + k];
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned char *fl = flag + start;
        u32 p = 0;
        while (p < len) {
            PNG_CHECK(start + p < n && p < block_bytes, 4);
            fl[p] = 1;
            const u32 c = sl[p];
            p += c ? c + 3 : 1;
        }
    }
    __syncthreads();
    for (u32 k = threadIdx.x; k < len; k += blockDim.x) {
        if (!flag[start + k]) continue;
        const u32 c = sl[k];
        if (!c) {
            atomicAdd(&h[f[start + k]], 1u);
        } else {
            atomicAdd(&h[257 + c_png_len_sym[c + 3]], 1u);
            atomicAdd(&h[kPngLit + png_dist_sym(dist[start + k] + 1u)], 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) h[256] = 1;
    __syncthreads();
    for (u32 k = threadIdx.x; k < kPngLit + kPngDist; k += blockDim.x) hist[static_cast<u64>(blockIdx.x) * (kPngLit + kPngDist) + k] = h[k];
}

// ------------------------------------------------------------------------------------------------------ 5-6. codes

struct PngPmShared {
    u32 lw[288];             // used symbols' weights, ascending (weight, symbol)
    uint16_t lsym[288];
    u32 a[576], b[576];      // the previous and current level lists
    unsigned char leaf[15][576];
    u32 nleaf[16];
};

// Package-merge code lengths of freq[0..n) limited to `limit` bits, by one warp.  Leaves are ranked by (weight, symbol);
// in each merged list a leaf comes before a package of equal weight.  Fewer than two used symbols: two codes of length 1,
// symbol 0 (or 1 when 0 is the used one) completing the tree.
__device__ void png_package_merge(const u32 *freq, u32 n, u32 limit, unsigned char *len, PngPmShared &sh) {
    const u32 lane = threadIdx.x & 31;
    u32 used = 0;
    for (u32 i = 0; i < n; i += 32) used += __popc(__ballot_sync(0xFFFFFFFFu, i + lane < n && freq[i + lane] > 0));
    for (u32 i = lane; i < n; i += 32) {
        len[i] = 0;
        if (!freq[i]) continue;
        const u32 key = (freq[i] << 9) | i;
        u32 rank = 0;
        for (u32 j = 0; j < n; ++j)
            if (freq[j] && ((freq[j] << 9) | j) < key) ++rank;
        sh.lw[rank] = freq[i];
        sh.lsym[rank] = static_cast<uint16_t>(i);
    }
    __syncwarp();
    if (used < 2) {
        if (lane == 0) {
            u32 s0 = 0xFFFFFFFFu;
            for (u32 i = 0; i < n; ++i)
                if (freq[i]) s0 = i;
            if (s0 != 0xFFFFFFFFu) len[s0] = 1;
            len[s0 == 0 ? 1 : 0] = 1;
            if (s0 == 0xFFFFFFFFu) len[1] = 1;
        }
        __syncwarp();
        return;
    }
    u32 *prev = sh.a, *cur = sh.b;
    for (u32 i = lane; i < used; i += 32) {
        prev[i] = sh.lw[i];
        sh.leaf[0][i] = 1;
    }
    __syncwarp();
    u32 plen = used;
    for (u32 lvl = 1; lvl < limit; ++lvl) {
        const u32 np = plen / 2;
        for (u32 i = lane; i < used; i += 32) {
            const u32 w = sh.lw[i];
            u32 lo = 0, hi = np;                    // packages with weight < w
            while (lo < hi) {
                const u32 mid = (lo + hi) / 2;
                if (prev[2 * mid] + prev[2 * mid + 1] < w) lo = mid + 1;
                else hi = mid;
            }
            cur[i + lo] = w;
            sh.leaf[lvl][i + lo] = 1;
        }
        for (u32 k = lane; k < np; k += 32) {
            const u32 w = prev[2 * k] + prev[2 * k + 1];
            u32 lo = 0, hi = used;                  // leaves with weight <= w
            while (lo < hi) {
                const u32 mid = (lo + hi) / 2;
                if (sh.lw[mid] <= w) lo = mid + 1;
                else hi = mid;
            }
            cur[k + lo] = w;
            sh.leaf[lvl][k + lo] = 0;
        }
        __syncwarp();
        u32 *t = prev;
        prev = cur;
        cur = t;
        plen = used + np;
    }
    u32 c = 2 * used - 2;
    for (int lvl = static_cast<int>(limit) - 1; lvl >= 0; --lvl) {
        u32 cnt = 0;
        for (u32 i = lane; i < c; i += 32) cnt += sh.leaf[lvl][i];
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, o);
        if (lane == 0) sh.nleaf[lvl] = cnt;
        c = 2 * (c - cnt);
    }
    __syncwarp();
    for (u32 r = lane; r < used; r += 32) {
        u32 d = 0;
        for (u32 lvl = 0; lvl < limit; ++lvl) d += sh.nleaf[lvl] > r;
        len[sh.lsym[r]] = static_cast<unsigned char>(d);
    }
    __syncwarp();
}

// RFC 1951 §3.2.2 canonical codes, bit-reversed for LSB-first packing, packed as code | length << 16 (one thread).
__device__ void png_canonical(const unsigned char *len, u32 n, u32 *packed) {
    u32 count[16] = {0}, next[16];
    for (u32 i = 0; i < n; ++i) count[len[i]]++;
    count[0] = 0;
    u32 code = 0;
    for (u32 bits = 1; bits < 16; ++bits) {
        code = (code + count[bits - 1]) << 1;
        next[bits] = code;
    }
    for (u32 i = 0; i < n; ++i) {
        const u32 L = len[i];
        packed[i] = L ? ((__brev(next[L]++) >> (32 - L)) | (L << 16)) : 0u;
    }
}

struct PngBits {   // plain (non-atomic) LSB-first writer into zeroed words
    u32 *w;
    u32 pos;
    __device__ void put(u32 v, u32 nb) {
        if (!nb) return;
        const u32 k = pos >> 5, sh = pos & 31;
        PNG_CHECK(k + 1 < kPngHdrWords || (k < kPngHdrWords && sh + nb <= 32), 5);
        w[k] |= v << sh;
        if (sh + nb > 32) w[k + 1] |= v >> (32 - sh);
        pos += nb;
    }
};

// One warp per block of the group: the three trees, the header bits and the block's bit count.
__global__ void __launch_bounds__(32) k_png_huffman(const PngImage *__restrict__ im, u32 g, const u32 *__restrict__ hist,
                                                    u32 *__restrict__ codes, u32 *__restrict__ hdr, u32 *__restrict__ hdr_bits,
                                                    u64 *__restrict__ bits) {
    __shared__ PngPmShared sh;
    __shared__ u32 fr[kPngLit + kPngDist];
    __shared__ unsigned char len[kPngLit + kPngDist];
    __shared__ u32 pk[kPngLit + kPngDist];
    __shared__ u32 clf[kPngCl];
    __shared__ unsigned char cll[kPngCl];
    __shared__ u32 clc[kPngCl];
    __shared__ u32 seq[kPngLit + kPngDist];   // run-length items: symbol | extra value << 8 | extra bits << 16
    __shared__ u32 hw[kPngHdrWords];
    __shared__ u32 nseq, hlit, hdist;
    const u32 lane = threadIdx.x;
    const u32 blk = blockIdx.x;
    for (u32 k = lane; k < kPngLit + kPngDist; k += 32) fr[k] = hist[static_cast<u64>(blk) * (kPngLit + kPngDist) + k];
    for (u32 k = lane; k < kPngHdrWords; k += 32) hw[k] = 0;
    for (u32 k = lane; k < kPngCl; k += 32) clf[k] = 0;
    __syncwarp();
    png_package_merge(fr, kPngLit, 15, len, sh);
    png_package_merge(fr + kPngLit, kPngDist, 15, len + kPngLit, sh);
    if (lane == 0) {
        u32 hl = 257, hd = 1;
        for (u32 s = 0; s < kPngLit; ++s)
            if (len[s]) hl = max(hl, s + 1);
        for (u32 s = 0; s < kPngDist; ++s)
            if (len[kPngLit + s]) hd = max(hd, s + 1);
        hlit = hl;
        hdist = hd;
        // the HLIT + HDIST lengths as one run-length coded sequence
        const u32 total = hl + hd;
        auto at = [&](u32 i) -> u32 { return i < hl ? len[i] : len[kPngLit + i - hl]; };
        u32 ns = 0, i = 0;
        while (i < total) {
            const u32 v = at(i);
            u32 run = 1;
            while (i + run < total && at(i + run) == v) ++run;
            if (v == 0) {
                u32 r = run;
                while (r >= 11) {
                    const u32 k = min(r, 138u);
                    seq[ns++] = 18u | ((k - 11) << 8) | (7u << 16);
                    r -= k;
                }
                if (r >= 3) {
                    seq[ns++] = 17u | ((r - 3) << 8) | (3u << 16);
                    r = 0;
                }
                for (; r; --r) seq[ns++] = 0;
            } else {
                seq[ns++] = v;
                u32 r = run - 1;
                while (r >= 3) {
                    const u32 k = min(r, 6u);
                    seq[ns++] = 16u | ((k - 3) << 8) | (2u << 16);
                    r -= k;
                }
                for (; r; --r) seq[ns++] = v;
            }
            i += run;
        }
        nseq = ns;
        PNG_CHECK(ns <= kPngLit + kPngDist, 6);
        for (u32 k = 0; k < ns; ++k) clf[seq[k] & 0xFF]++;
    }
    __syncwarp();
    png_package_merge(clf, kPngCl, 7, cll, sh);
    if (lane == 0) {
        png_canonical(cll, kPngCl, clc);
        png_canonical(len, kPngLit, pk);
        png_canonical(len + kPngLit, kPngDist, pk + kPngLit);
        u32 hclen = kPngCl;
        while (hclen > 4 && cll[c_png_cl_order[hclen - 1]] == 0) --hclen;
        PngBits wr{hw, 0};
        const PngImage &I = im[png_image_of<&PngImage::blk0>(im, g, blk)];
        wr.put(blk + 1 == I.blk0 + I.nblocks ? 1u : 0u, 1);   // BFINAL on the image's last block
        wr.put(2u, 2);
        wr.put(hlit - 257, 5);
        wr.put(hdist - 1, 5);
        wr.put(hclen - 4, 4);
        for (u32 k = 0; k < hclen; ++k) wr.put(cll[c_png_cl_order[k]], 3);
        for (u32 k = 0; k < nseq; ++k) {
            const u32 s = seq[k] & 0xFF;
            wr.put(clc[s] & 0xFFFFu, clc[s] >> 16);
            wr.put((seq[k] >> 8) & 0xFF, seq[k] >> 16);
        }
        hdr_bits[blk] = wr.pos;
    }
    __syncwarp();
    u64 tot = 0;
    for (u32 s = lane; s < kPngLit + kPngDist; s += 32) {
        if (!fr[s]) continue;
        u32 extra = 0;
        if (s >= 257 && s < kPngLit) extra = c_png_len_extra[s - 257];
        else if (s >= kPngLit) extra = c_png_dist_extra[s - kPngLit];
        tot += static_cast<u64>(fr[s]) * (len[s] + extra);
    }
    for (int o = 16; o; o >>= 1) tot += __shfl_xor_sync(0xFFFFFFFFu, tot, o);
    if (lane == 0) bits[blk] = tot + hdr_bits[blk];
    for (u32 k = lane; k < kPngLit + kPngDist; k += 32) codes[static_cast<u64>(blk) * (kPngLit + kPngDist) + k] = pk[k];
    for (u32 k = lane; k < kPngHdrWords; k += 32) hdr[static_cast<u64>(blk) * kPngHdrWords + k] = hw[k];
}

// Segmented exclusive scan of the block bit counts, one CTA of 1024 threads per image, and each stream's total.
__global__ void __launch_bounds__(1024) k_png_scan(const PngImage *__restrict__ im, const u64 *__restrict__ bits_all,
                                                   u64 *__restrict__ off_all, PngCtl *__restrict__ ctl_all) {
    __shared__ u64 part[1024];
    const PngImage &I = im[blockIdx.x];
    const u32 nblocks = I.nblocks;
    const u64 *__restrict__ bits = bits_all + I.blk0;
    u64 *__restrict__ off = off_all + I.blk0;
    PngCtl *__restrict__ ctl = ctl_all + blockIdx.x;
    const u32 t = threadIdx.x;
    const u32 per = (nblocks + 1023) / 1024;
    const u32 b0 = min(nblocks, t * per), b1 = min(nblocks, b0 + per);
    u64 s = 0;
    for (u32 k = b0; k < b1; ++k) s += bits[k];
    part[t] = s;
    __syncthreads();
    if (t == 0) {
        u64 acc = 0;
        for (u32 k = 0; k < 1024; ++k) {
            const u64 v = part[k];
            part[k] = acc;
            acc += v;
        }
        ctl->deflate_bits = acc;
    }
    __syncthreads();
    u64 acc = part[t];
    for (u32 k = b0; k < b1; ++k) {
        off[k] = acc;
        acc += bits[k];
    }
}

// ------------------------------------------------------------------------------------------------------ emission

struct PngOut {   // LSB-first writer into zeroed words shared with other threads (atomicOr)
    u32 *w;
    u64 pos;      // bit position of acc's bit 0
    u64 acc;
    u32 nacc;
    u64 lim;      // bytes of w (bounds-checking build)
    __device__ void flush_word(u32 v, u32 nb) {
        const u64 k = pos >> 5;
        const u32 sh = static_cast<u32>(pos & 31);
        if (nb < 32) v &= (1u << nb) - 1u;
        if (v) {
            PNG_CHECK(4 * (k + (sh && (v >> (32 - sh)) ? 2 : 1)) <= lim, 7);
            atomicOr(&w[k], v << sh);
            if (sh && (v >> (32 - sh))) atomicOr(&w[k + 1], v >> (32 - sh));
        }
        pos += nb;
    }
    __device__ void put(u32 v, u32 nb) {   // nb <= 32
        if (!nb) return;
        acc |= static_cast<u64>(v) << nacc;
        nacc += nb;
        if (nacc >= 32) {
            flush_word(static_cast<u32>(acc), 32);
            acc >>= 32;
            nacc -= 32;
        }
    }
    __device__ void done() {
        if (nacc) flush_word(static_cast<u32>(acc), nacc);
        nacc = 0;
    }
};

// One CTA per block of the group, kPngEmitThreads / 32 warps, each owning a contiguous segment of the block's positions.  A warp reads
// its segment 32 consecutive positions at a time (coalesced); a warp scan of the token bit counts places each lane's
// token, the lanes OR their bits into a per-warp staging buffer in shared memory, and the warp ORs the covered words into
// the output.  Pass 1 counts the bits of each segment so that a CTA scan gives the segments' offsets; thread 0 writes the
// header and the end-of-block code.  The Adler-32 partial sums of the block ride along.
constexpr u32 kPngStageWords = 50;   // 32 tokens of at most 48 bits plus an offset of < 32 bits
__global__ void __launch_bounds__(kPngEmitThreads) k_png_emit(const PngImage *__restrict__ im, u32 g,
                                                              const unsigned char *__restrict__ f_all,
                                                              const unsigned char *__restrict__ lcode_all,
                                                              const uint16_t *__restrict__ dist_all,
                                                              const unsigned char *__restrict__ flag_all, u32 block_bytes,
                                                              const u32 *__restrict__ codes, const u32 *__restrict__ hdr,
                                                              const u32 *__restrict__ hdr_bits, const u64 *__restrict__ off,
                                                              unsigned char *__restrict__ out_all, u64 *__restrict__ sums) {
    constexpr u32 kWarps = kPngEmitThreads / 32;
    __shared__ u32 tab[kPngLit + kPngDist];
    __shared__ u64 wsum[kWarps];
    __shared__ u64 red[2][kWarps];
    __shared__ u32 stage[kWarps][kPngStageWords];
    const u32 blk = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const PngImage &I = im[png_image_of<&PngImage::blk0>(im, g, blk)];
    const u32 n = I.n;
    const unsigned char *__restrict__ f = f_all + I.pos;
    const unsigned char *__restrict__ lcode = lcode_all + I.pos;
    const uint16_t *__restrict__ dist = dist_all + I.pos;
    const unsigned char *__restrict__ flag = flag_all + I.pos;
    u32 *__restrict__ out_words = reinterpret_cast<u32 *>(out_all + I.out);
    const u64 out_lim = I.out_bytes;
    const u32 start = (blk - I.blk0) * block_bytes;
    const u32 len = min(block_bytes, n - start);
    PNG_CHECK(start + len <= n && blk - I.blk0 < I.nblocks, 13);
    for (u32 k = t; k < kPngLit + kPngDist; k += blockDim.x) tab[k] = codes[static_cast<u64>(blk) * (kPngLit + kPngDist) + k];
    for (u32 k = lane; k < kPngStageWords; k += 32) stage[wid][k] = 0;
    __syncthreads();
    const u32 per = (len + kWarps * 32 - 1) / (kWarps * 32) * 32;   // segment length, a multiple of 32
    const u32 s0 = min(len, wid * per), s1e = min(len, s0 + per);
    // token at position p: bits, and the (value, count) pieces
    auto token = [&](u32 p, u32 &v0, u32 &n0, u32 &v1, u32 &n1) {
        const u32 c = lcode[start + p];
        if (!c) {
            const u32 e = tab[f[start + p]];
            v0 = e & 0xFFFFu;
            n0 = e >> 16;
            v1 = 0;
            n1 = 0;
            return;
        }
        const u32 L = c + 3, ls = c_png_len_sym[L];
        const u32 d = dist[start + p] + 1u, ds = png_dist_sym(d);
        const u32 el = tab[257 + ls], ed = tab[kPngLit + ds];
        const u32 nl = el >> 16, xl = c_png_len_extra[ls], nd = ed >> 16;
        v0 = (el & 0xFFFFu) | ((L - c_png_len_base[ls]) << nl);   // length code + extra: at most 20 bits
        n0 = nl + xl;
        v1 = (ed & 0xFFFFu) | ((d - c_png_dist_base[ds]) << nd);   // distance code + extra: at most 28 bits
        n1 = nd + c_png_dist_extra[ds];
    };
    u64 mine = 0, a1 = 0, a2 = 0;
    for (u32 p = s0 + lane; p < s1e; p += 32) {
        const u32 v = f[start + p];
        a1 += v;
        a2 += static_cast<u64>(len - p) * v;
        if (flag[start + p]) {
            u32 v0, n0, v1, n1;
            token(p, v0, n0, v1, n1);
            mine += n0 + n1;
        }
    }
    for (int o = 16; o; o >>= 1) {
        mine += __shfl_xor_sync(0xFFFFFFFFu, mine, o);
        a1 += __shfl_xor_sync(0xFFFFFFFFu, a1, o);
        a2 += __shfl_xor_sync(0xFFFFFFFFu, a2, o);
    }
    if (lane == 0) {
        wsum[wid] = mine;
        red[0][wid] = a1;
        red[1][wid] = a2;
    }
    __syncthreads();
    u64 before = 0, toks = 0;
    for (u32 k = 0; k < kWarps; ++k) {
        if (k < wid) before += wsum[k];
        toks += wsum[k];
    }
    const u64 base = static_cast<u64>(kPngDeflateBase) * 8 + off[blk];
    const u32 hb = hdr_bits[blk];
    u64 pos = base + hb + before;   // bit position of the next step's first token
    u32 *st = stage[wid];
    for (u32 p0 = s0; p0 < s1e; p0 += 32) {
        const u32 p = p0 + lane;
        u32 v0 = 0, n0 = 0, v1 = 0, n1 = 0;
        if (p < s1e && flag[start + p]) token(p, v0, n0, v1, n1);
        const u32 nb = n0 + n1;
        u32 x = nb;
        for (int o = 1; o < 32; o <<= 1) {
            const u32 y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if (lane >= static_cast<u32>(o)) x += y;
        }
        const u32 total = __shfl_sync(0xFFFFFFFFu, x, 31);
        const u32 sh = static_cast<u32>(pos & 31);
        auto put = [&](u32 at, u32 v, u32 cnt) {   // cnt <= 28 bits at local bit `at`
            if (!cnt || !v) return;
            const u32 k = at >> 5, b = at & 31;
            PNG_CHECK(k + (b + cnt > 32 ? 1 : 0) < kPngStageWords, 8);
            atomicOr(&st[k], v << b);
            if (b + cnt > 32) atomicOr(&st[k + 1], v >> (32 - b));
        };
        const u32 at = sh + x - nb;
        put(at, v0, n0);
        put(at + n0, v1, n1);
        __syncwarp();
        const u32 nw = (sh + total + 31) >> 5;
        const u64 w0 = pos >> 5;
        for (u32 k = lane; k < nw; k += 32) {
            const u32 v = st[k];
            PNG_CHECK(4 * (w0 + k + 1) <= out_lim, 9);
            if (v) atomicOr(&out_words[w0 + k], v);
            st[k] = 0;
        }
        __syncwarp();
        pos += total;
    }
    if (t == 0) {
        PngOut h{out_words, base, 0, 0, out_lim};
        const u32 *hw = hdr + static_cast<u64>(blk) * kPngHdrWords;
        for (u32 k = 0; k * 32 < hb; ++k) h.put(hw[k], min(32u, hb - k * 32));
        h.done();
        PngOut eob{out_words, base + hb + toks, 0, 0, out_lim};
        eob.put(tab[256] & 0xFFFFu, tab[256] >> 16);
        eob.done();
        u64 x1 = 0, x2 = 0;
        for (u32 k = 0; k < kWarps; ++k) {
            x1 += red[0][k];
            x2 += red[1][k];
        }
        sums[2 * static_cast<u64>(blk)] = x1;
        sums[2 * static_cast<u64>(blk) + 1] = x2;
    }
}

// ------------------------------------------------------------------------------------------------------ framing

__device__ __forceinline__ u32 png_multmodp(u32 a, u32 b) {   // zlib's multmodp: a * b mod P, reflected
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

__device__ __forceinline__ u32 png_x8n(u64 n) {   // x^(8 n) mod P
    u32 p = 1u << 31;
    u32 k = 3;
    while (n) {
        if (n & 1) p = png_multmodp(c_png_x2n[k & 31], p);
        n >>= 1;
        ++k;
    }
    return p;
}

__device__ __forceinline__ void png_be32(unsigned char *p, u32 v) {
    p[0] = static_cast<unsigned char>(v >> 24);
    p[1] = static_cast<unsigned char>(v >> 16);
    p[2] = static_cast<unsigned char>(v >> 8);
    p[3] = static_cast<unsigned char>(v);
}

// One thread per image: Adler-32 from the block sums, the signature, IHDR, the IDAT length and type, the zlib header and
// trailer.
__global__ void k_png_frame(const PngImage *__restrict__ im, u32 g, const u64 *__restrict__ sums_all, u32 block_bytes,
                            unsigned char *__restrict__ out_all, PngCtl *__restrict__ ctl_all) {
    const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= g) return;
    const PngImage &I = im[k];
    const u32 n = I.n, nblocks = I.nblocks;
    const u64 *__restrict__ sums = sums_all + 2 * static_cast<u64>(I.blk0);
    unsigned char *__restrict__ out = out_all + I.out;
    PngCtl *__restrict__ ctl = ctl_all + k;
    const u64 M = 65521;
    u64 s1 = 1, s2 = n % M;
    for (u32 b = 0; b < nblocks; ++b) {
        const u64 end = min(static_cast<u64>(n), static_cast<u64>(b + 1) * block_bytes);
        const u64 sb = sums[2 * static_cast<u64>(b)] % M, wb = sums[2 * static_cast<u64>(b) + 1] % M;
        s1 = (s1 + sb) % M;
        s2 = (s2 + wb + ((n - end) % M) * sb) % M;
    }
    const u32 adler = static_cast<u32>((s2 << 16) | s1);
    ctl->adler = adler;
    const u64 dbytes = (ctl->deflate_bits + 7) / 8;
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    for (int j = 0; j < 8; ++j) out[j] = sig[j];
    for (int j = 0; j < 25; ++j) out[8 + j] = I.ihdr[j];
    png_be32(out + 33, static_cast<u32>(2 + dbytes + 4));
    out[37] = 'I';
    out[38] = 'D';
    out[39] = 'A';
    out[40] = 'T';
    out[41] = 0x78;
    out[42] = 0x9C;
    PNG_CHECK(kPngDeflateBase + dbytes + 20 <= I.out_bytes, 10);
    png_be32(out + kPngDeflateBase + dbytes, adler);
    ctl->total = kPngDeflateBase + dbytes + 4 + 4 + 12;
}

// CRC-32 contributions: each thread takes kPngCrcChunk bytes of one image's "IDAT" + zlib stream, computes their CRC
// from a zero register and shifts it by the bytes that follow (x^(8 k) mod P); the contributions XOR together (CRC
// linearity).  Each image's chunks start at a multiple of 32, so a warp's contributions belong to one image.
__global__ void __launch_bounds__(256) k_png_crc(const PngImage *__restrict__ im, u32 g, u32 chunks,
                                                 const unsigned char *__restrict__ out_all, PngCtl *__restrict__ ctl_all) {
    __shared__ u32 tab[256];
    for (u32 k = threadIdx.x; k < 256; k += blockDim.x) tab[k] = c_png_crc_table[k];
    __syncthreads();
    const u32 gc = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 k = png_image_of<&PngImage::chunk0>(im, g, min(gc, chunks - 1));
    const PngImage &I = im[k];
    const unsigned char *__restrict__ out = out_all + I.out;
    PngCtl *__restrict__ ctl = ctl_all + k;
    const u64 lo = 37, hi = ctl->total - 16;   // IDAT type .. Adler-32 inclusive
    const u64 a = lo + static_cast<u64>(gc - I.chunk0) * kPngCrcChunk;
    u32 contrib = 0;
    if (gc < chunks && a < hi) {
        const u64 b = min(hi, a + kPngCrcChunk);
        u32 c = 0;
        PNG_CHECK(b <= I.out_bytes, 11);
        for (u64 k = a; k < b; ++k) c = tab[(c ^ out[k]) & 0xFF] ^ (c >> 8);
        contrib = png_multmodp(png_x8n(hi - b), c);
    }
    for (int o = 16; o; o >>= 1) contrib ^= __shfl_xor_sync(0xFFFFFFFFu, contrib, o);
    if ((threadIdx.x & 31) == 0 && contrib) atomicXor(&ctl->crc_raw, contrib);
}

// One thread per image: the IDAT CRC (initial register and final XOR applied) and the IEND chunk.
__global__ void k_png_end(const PngImage *__restrict__ im, u32 g, unsigned char *__restrict__ out_all,
                          const PngCtl *__restrict__ ctl_all) {
    const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= g) return;
    const PngImage &I = im[k];
    unsigned char *__restrict__ out = out_all + I.out;
    const PngCtl *__restrict__ ctl = ctl_all + k;
    const u64 hi = ctl->total - 16;
    const u32 crc = ctl->crc_raw ^ png_multmodp(png_x8n(hi - 37), 0xFFFFFFFFu) ^ 0xFFFFFFFFu;
    PNG_CHECK(hi + 16 <= I.out_bytes, 12);
    png_be32(out + hi, crc);
    const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    for (int j = 0; j < 12; ++j) out[hi + 4 + j] = iend[j];
}

}  // namespace aptb200
