// FM demodulation of complex I/Q (DESIGN.md §10): load + convert, mix to 0 Hz, channel FIR decimated by D, discriminator,
// in one kernel that reads the I/Q once and writes only the audio.
//
// A CTA owns a tile of tz consecutive FIR outputs z[zb .. zb + tz) and writes the audio a[zb + 1 .. zb + tz): it recomputes
// z[zb] in front of its tile, so no value crosses CTAs.  The staged input is polyphase-major: plane r holds
// S_r[j] = s[j*D - r], so that z[m] = sum_r sum_q hp[r][q] * S_r[m - q] with hp[r][q] = h[q*D + r] (zero past N taps).
// Each thread makes 16 consecutive outputs of one plane partition; per block of 16 taps it reads 31 samples and issues
// 512 FMAs (a 16 x 16 register-blocked convolution), so shared memory supplies one sample per 16 FMAs.  Each plane is
// stored as 16 sub-planes (u mod 16) so that the lanes of a warp read consecutive words.
// Every output sums planes r = p, p + P, ... per partition p, q descending within each 16-tap block, then the partitions
// p = 0..P-1 in order: the same sequence for every output, wherever the tile, chunk or launch boundaries fall.  A sample
// with a non-finite component after the mix is staged as 0, so the zero-padded taps never turn it into a NaN.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "launch.hpp"

namespace aptb200 {

constexpr u32 kIqBlock = 4096;    // B: the phasor is P[i / B] (x) W[i % B]
constexpr u32 kIqThreads = 256;
constexpr u32 kIqR = 16;          // outputs per thread = taps per register block

struct IqArgs {
    const void *in;               // the address I/Q sample 0 would have (complex samples of the format)
    u64 w_lo, w_hi;               // absolute samples [w_lo, w_hi) are readable at in; every other sample reads as 0
    const float2 *W;              // kIqBlock phasors
    const float *hp;              // D x qpad polyphase taps
    u32 D, qpad;
    u32 fs;                       // iq_rate
    u64 f;                        // offset_hz mod fs, in [0, fs)
    int mix;                      // 0: offset 0, p(i) == 1 and the mix is skipped
    float scale;                  // (float)(audio_rate / 2pi)
    u64 m_begin, m_end;           // audio outputs to write, absolute
    float *out;                   // the address audio output 0 would have
    u32 tz, lp16, ps;             // FIR outputs per tile, sub-plane length, plane stride (float2)
};

template <int FMT> __device__ __forceinline__ float2 iq_load(const void *p, u64 i);
template <> __device__ __forceinline__ float2 iq_load<APT_CU8>(const void *p, u64 i) {
    const uchar2 v = __ldg(static_cast<const uchar2 *>(p) + i);
    return make_float2(__fsub_rn(static_cast<float>(v.x), 127.5f), __fsub_rn(static_cast<float>(v.y), 127.5f));
}
template <> __device__ __forceinline__ float2 iq_load<APT_CS16>(const void *p, u64 i) {
    const short2 v = __ldg(static_cast<const short2 *>(p) + i);
    return make_float2(static_cast<float>(v.x), static_cast<float>(v.y));
}
template <> __device__ __forceinline__ float2 iq_load<APT_CF32>(const void *p, u64 i) {
    return __ldg(static_cast<const float2 *>(p) + i);
}

// complex product in f32, every operation rounded on its own
__device__ __forceinline__ float2 cmul_rn(float2 a, float2 b) {
    return make_float2(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

// The per-channel launch data of k_fm_demod_channels: channel c (blockIdx.y) mixes with W[c], f[c], mix[c] and writes out[c].
constexpr int kIqMaxChannels = 8;
struct IqChannels {
    const float2 *W[kIqMaxChannels];
    float *out[kIqMaxChannels];
    u64 f[kIqMaxChannels];
    int mix[kIqMaxChannels];
};

// One tile of k_fm_demod (blockIdx.x) for the channel whose phasors, offset, mix flag and output are given; every other
// field of `a` is shared by the channels.  Both kernels run this function, so a channel's audio is the same bits in each.
template <int FMT>
__device__ __forceinline__ void fm_demod_tile(const IqArgs &a, const float2 *W, u64 f, int mix, float *out) {
    extern __shared__ float2 sm[];
    const u32 D = a.D, qpad = a.qpad, tz = a.tz, lp16 = a.lp16, ps = a.ps;
    const u32 tid = threadIdx.x;
    const long long zb = static_cast<long long>(a.m_begin) - 1 + static_cast<long long>(blockIdx.x) * (tz - 1);
    const u32 lp = tz + qpad - 1;                                  // samples per plane the tile reads
    const long long i_lo = (zb - static_cast<long long>(qpad) + 1) * D - (D - 1);
    const u64 nstage = static_cast<u64>(lp) * D;
    float2 *P = sm + static_cast<size_t>(D) * ps;                 // phasors P[i / B] of the tile's blocks

    // --- P[q] = exp(-2 pi j ((q B f) mod fs) / fs), evaluated in double and rounded once
    const long long qa = (i_lo < 0 ? 0 : i_lo) >> 12;
    if (mix) {
        const long long last = i_lo + static_cast<long long>(nstage) - 1;
        const u32 nq = last < 0 ? 0u : static_cast<u32>((last >> 12) - qa + 1);
        if (tid < nq) {
            const u64 q = static_cast<u64>(qa) + tid;
            const u64 v = ((q * kIqBlock) % a.fs) * f % a.fs;
            double sv, cv;
            sincospi(-2.0 * static_cast<double>(v) / static_cast<double>(a.fs), &sv, &cv);
            P[tid] = make_float2(static_cast<float>(cv), static_cast<float>(sv));
        }
        __syncthreads();
    }

    // --- stage: load, convert, mix, scatter into the polyphase planes (element e = u*D + (D-1-r), i = i_lo + e)
    {
        u32 u = tid / D, o = tid % D;
        const u32 du = kIqThreads / D, dr = kIqThreads % D;
        for (u64 e = tid; e < nstage; e += kIqThreads) {
            const long long i = i_lo + static_cast<long long>(e);
            float2 x = make_float2(0.f, 0.f);
            if (i >= static_cast<long long>(a.w_lo) && i < static_cast<long long>(a.w_hi)) {
                x = iq_load<FMT>(a.in, static_cast<u64>(i));
                if (mix) {
                    const float2 p = cmul_rn(P[(i >> 12) - qa], __ldg(W + (i & (kIqBlock - 1))));
                    x = cmul_rn(x, p);
                }
                // a NaN or Inf would reach the outputs whose zero-padded taps cover it, and whether those read it
                // depends on where the chunk window starts: staged as 0, every FMA with a zero tap is exact
                if (!isfinite(x.x) || !isfinite(x.y)) x = make_float2(0.f, 0.f);
            }
            const u32 r = D - 1 - o;
            sm[static_cast<size_t>(r) * ps + (u & 15) * lp16 + (u >> 4)] = x;
            u += du;
            o += dr;
            if (o >= D) {
                o -= D;
                ++u;
            }
        }
    }
    __syncthreads();

    // --- channel FIR: thread (g, p) makes z[zb + 16g .. zb + 16g + 16) over the planes r = p, p + P, ...
    const u32 gl = tz / kIqR, P_parts = kIqThreads / gl;
    const u32 g = tid % gl, p = tid / gl;
    float ar[kIqR], ai[kIqR];
#pragma unroll
    for (int k = 0; k < (int)kIqR; ++k) ar[k] = ai[k] = 0.f;
    for (u32 r = p; r < D; r += P_parts) {
        const float4 *hq = reinterpret_cast<const float4 *>(a.hp + static_cast<size_t>(r) * qpad);
        for (u32 q0 = 0; q0 < qpad; q0 += kIqR) {
            float t[kIqR];
#pragma unroll
            for (int k = 0; k < (int)kIqR / 4; ++k) {
                const float4 v = __ldg(hq + q0 / 4 + k);
                t[4 * k] = v.x; t[4 * k + 1] = v.y; t[4 * k + 2] = v.z; t[4 * k + 3] = v.w;
            }
            // output i, tap q reads local sample u = 16g + (qpad - 1 - q0) + (i - q); qpad - 1 - q0 = 16*ch + 15
            const float2 *base = sm + static_cast<size_t>(r) * ps + g + (qpad - q0) / 16 - 1;
#pragma unroll
            for (int d = -(int)kIqR + 1; d < (int)kIqR; ++d) {
                const int c = 15 + d;                                  // in [0, 30]
                const float2 x = base[(c & 15) * lp16 + (c >> 4)];
#pragma unroll
                for (int i = 0; i < (int)kIqR; ++i) {
                    const int q = i - d;
                    if (q >= 0 && q < (int)kIqR) {
                        ar[i] = fmaf(t[q], x.x, ar[i]);
                        ai[i] = fmaf(t[q], x.y, ai[i]);
                    }
                }
            }
        }
    }
    __syncthreads();   // the planes are read: their space takes the partial sums

    // --- partial sums of the P partitions, in partition order (index skewed by 1 per 16 against bank conflicts)
    const u32 pstride = tz + tz / 16;
#pragma unroll
    for (int i = 0; i < (int)kIqR; ++i) sm[static_cast<size_t>(p) * pstride + 17 * g + i] = make_float2(ar[i], ai[i]);
    __syncthreads();
    float2 *zs = sm + static_cast<size_t>(P_parts) * pstride;
    for (u32 zl = tid; zl < tz; zl += kIqThreads) {
        const u32 k = zl + zl / 16;
        float2 z = sm[k];
        for (u32 pp = 1; pp < P_parts; ++pp) {
            const float2 v = sm[static_cast<size_t>(pp) * pstride + k];
            z.x = __fadd_rn(z.x, v.x);
            z.y = __fadd_rn(z.y, v.y);
        }
        zs[zl] = z;
    }
    __syncthreads();

    // --- discriminator: a[m] = atan2f(Im(z[m] conj z[m-1]), Re(..)) * audio_rate / 2pi, a[0] = 0
    for (u32 zl = tid + 1; zl < tz; zl += kIqThreads) {
        const long long m = zb + zl;
        if (m >= static_cast<long long>(a.m_end)) break;
        float v = 0.f;
        if (m > 0) {
            const float2 z1 = zs[zl], z0 = zs[zl - 1];
            const float re = __fadd_rn(__fmul_rn(z1.x, z0.x), __fmul_rn(z1.y, z0.y));
            const float im = __fsub_rn(__fmul_rn(z1.y, z0.x), __fmul_rn(z1.x, z0.y));
            v = __fmul_rn(atan2f(im, re), a.scale);
        }
        out[m] = v;
    }
}

template <int FMT>
__global__ void __launch_bounds__(kIqThreads, 2) k_fm_demod(const IqArgs a) {
    fm_demod_tile<FMT>(a, a.W, a.f, a.mix, a.out);
}

// Several channels of one I/Q window in one launch: blockIdx.y is the channel; a.W, a.f, a.mix and a.out are not read.
template <int FMT>
__global__ void __launch_bounds__(kIqThreads, 2) k_fm_demod_channels(const IqArgs a, const IqChannels ch) {
    const u32 c = blockIdx.y;
    fm_demod_tile<FMT>(a, ch.W[c], ch.f[c], ch.mix[c], ch.out[c]);
}

// The load of k_fm_demod alone: n samples of a push into the streaming decoder's cf32 window (exact for every format).
template <int FMT>
__global__ void __launch_bounds__(256) k_iq_to_cf32(const void *__restrict__ in, u64 n, float2 *__restrict__ out) {
    for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x)
        out[i] = iq_load<FMT>(in, i);
}

}  // namespace aptb200
