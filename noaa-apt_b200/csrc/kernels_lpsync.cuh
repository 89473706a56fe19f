// Fused demodulation low-pass + sync cross-correlation (dsp::filter dsp.rs:386-410 with the 37..61-tap
// Lowpass of decode.rs:95-102, and the correlation loop of find_sync decode.rs:225-233).
//
//   f[i]    = sum_{j < NT, j < i} e[i-j] * c[j]                 (causal; e[0] is never read: strict i > j)
//   corr[i] = sum_{j < 38*PW} guard[j] * f[i+j],   i < n - 38*PW
//
// The template is +-1 in runs of 2*PW samples (19 runs: - | (-,+) x 7 | - - - -), so the correlation is
// computed from box sums B[n] = f[n] + ... + f[n+2*PW-1]:  corr[i] = sum_b sign_b * B[i + 2*PW*b]  -- 24 adds
// per output instead of 114.  The summation order differs from the reference's sequential loop, i.e. the
// values agree to fp32 rounding (~1e-7 relative), not bit for bit; the generic kernel keeps the exact order.  f, the box
// sums and corr are bit for bit those of k_lowpass_records (kernels_sync2.cuh), and f those of k_gather_rows_lp: the three
// share one low-pass order, one box-sum order and one correlation order (tests/_sync_oracle.py restates them).
//
// Tiles start at `base` (BASED instantiations only; a multiple of 16, so every position keeps the parity and the 16-byte alignment it has with
// base 0 and the values are those of a run from 0); there f_out == nullptr skips storing f.
// One CTA handles 1856 consecutive positions: e tile -> f tile -> box sums -> correlation, all on fp32 register pairs
// (fma2: two FMAs / adds):
//   low-pass   : a thread owns 8 consecutive outputs (even warps the first 8 of a block of 16, odd warps the last 8),
//                one FMA chain each, tap 0 first: a window sample broadcast into a register pair meets the tap pair
//                (c[j], c[j+1]) of two neighbouring outputs, a warp-uniform kernel-parameter operand.
//   box sums   : pair sums P[k] = f[2k] + f[2k+1] shared by neighbouring outputs: PW + 2 adds per two outputs.
//   correlation: output pairs (v, v+1), v even, accumulate box pairs (B[m], B[m+1]), m even (2*PW is even), with
//                fma2 by (+-1, +-1): 19 per output pair.
// f and corr go to HBM once each (coalesced float4 from the shared tiles); e is read once (+7 % halo).  Shared-memory
// tiles are skewed by 4 floats every 32 so that 8- and 16-float-strided LDS.128 stay conflict-free.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "kernels_fast.cuh"
#include "launch.hpp"

namespace aptb200 {

struct LpTaps {          // kernel parameter: warp-uniform operands
    float2 p[64];        // p[j+1] = (c[j], c[j+1]), j = -1 .. NT-1 -- one sample x the taps of two neighbouring outputs
    float2 pd[72];       // pd[j+DEC] = (c[j], c[j+DEC]), j = -DEC .. NT-1 -- ... of two neighbouring PIXELS (DEC samples apart)
};

constexpr int kLpTile = 1856;   // (T + 38*PW - 1) / 16 <= 128 for PW <= 5: every phase is one pass of the CTA

__device__ __forceinline__ u32 skew(u32 n) { return n + ((n >> 5) << 2); }   // 4 floats of padding every 32

// Low-pass outputs o .. o+7, o = 16*blk + 8*HALF, from the skewed e tile into the skewed f tile.  Every output is ONE
// chain of FMAs, tap 0 first (f[o] = fma(c[NT-1], e[o-NT+1], ... fma(c[0], e[o], 0))), the order of k_lowpass_records and
// k_gather_rows_lp: one window sample x the taps it has in two neighbouring outputs, (c[j], c[j+1]) -- a warp-uniform tap
// pair -- into the accumulator pair of the outputs (2v, 2v+1).  j = -1 (c[-1] = 0) and the c[NT] = 0 half of j = NT-1 add
// +0 to a chain that starts at +0, which leaves it unchanged.
template <int NT, int HALF>
__device__ __forceinline__ void lp_outputs(const LpTaps &taps, const float *s_e, float *s_f, u32 blk) {
    static_assert(NT % 2 == 1, "odd tap counts only (Kaiser design, filters.rs:79)");
    constexpr int EOFF = (NT - 1 + 3) / 4 * 4;     // e tile starts this many samples before the tile (multiple of 4)
    constexpr int WN = EOFF + 8;                   // window: s_e[o .. o + EOFF + 7] (the oldest tap needs o + EOFF - NT + 1 >= o)
    const u32 o = 16 * blk + 8 * HALF;
    float w[WN];
#pragma unroll
    for (int k = 0; k < WN / 4; ++k) {
        const float4 q = *reinterpret_cast<const float4 *>(s_e + skew(o + 4 * k));
        w[4 * k] = q.x; w[4 * k + 1] = q.y; w[4 * k + 2] = q.z; w[4 * k + 3] = q.w;
    }
    f32x2 acc[4];                                  // 4 independent chain pairs, tap pair outermost
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[v] = 0ull;
#pragma unroll
    for (int j = -1; j < NT; ++j) {
        const f32x2 t2 = pack2(taps.p[j + 1].x, taps.p[j + 1].y);   // (c[j], c[j+1]): outputs 2v and 2v+1 from sample EOFF+2v-j
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const float x = w[EOFF + 2 * v - j];
            acc[v] = fma2(pack2(x, x), t2, acc[v]);
        }
    }
    float r[8];
#pragma unroll
    for (int v = 0; v < 4; ++v) unpack2(acc[v], r[2 * v], r[2 * v + 1]);
    *reinterpret_cast<float4 *>(s_f + skew(o)) = make_float4(r[0], r[1], r[2], r[3]);
    *reinterpret_cast<float4 *>(s_f + skew(o + 4)) = make_float4(r[4], r[5], r[6], r[7]);
}

template <int NT, int PW, bool BASED>
__global__ void __launch_bounds__(256, NT <= 37 && !BASED ? 4 : 2)
k_lowpass_corr(const float *__restrict__ e, u64 base_arg, u64 n, u64 ncorr, const __grid_constant__ LpTaps taps, float *__restrict__ f_out,
               float *__restrict__ corr_out) {
    const u64 base = BASED ? base_arg : 0;     // the whole-recording instantiations keep their register budget
    constexpr int T = kLpTile;
    constexpr int G = 38 * PW;                 // template length
    constexpr int BOX = 2 * PW;                // run length
    constexpr int FN = T + G - 1;              // f values needed by the tile's correlations
    constexpr int FNP = (FN + 15) / 16 * 16;   // computed in blocks of 16 (8 even + 8 odd positions)
    static_assert(FNP / 16 <= 128, "one pass of 8 warps");
    constexpr int EOFF = (NT - 1 + 3) / 4 * 4; // e tile starts this many samples before the tile (multiple of 4)
    constexpr int ENP = FNP + EOFF + 8;        // e values staged (the aligned windows read a few beyond the last output)
    constexpr int BN = T + 18 * BOX;           // box sums needed
    __shared__ __align__(16) float s_e[(ENP + 32) + (ENP + 32) / 8 + 8];
    __shared__ __align__(16) float s_f[(FNP + BOX + 16) + (FNP + BOX + 16) / 8 + 8];
    __shared__ __align__(16) float s_b[(BN + 16) + (BN + 16) / 8 + 8];

    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // e values of a tile, fetched one tile ahead into registers (the loads of tile k+1 are in flight while tile k is
    // computed): staged index m4 = 4*(tid + 256*r) holds e[i0 - EOFF + m4 .. +3]; indices < 1 or >= n read as zero
    // (dsp.rs:399: the sum only takes signal[i-j] with i > j, so signal[0] and anything before it never contribute)
    constexpr int NPRE = (ENP / 4 + 255) / 256;
    float4 pre[NPRE];
    auto fetch = [&](u64 tile_idx) {
        const u64 i0f = base + tile_idx * T;
#pragma unroll
        for (int r = 0; r < NPRE; ++r) {
            const u32 m4 = 4 * (tid + 256 * r);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m4 < ENP && i0f < n) {
                const long long g = static_cast<long long>(i0f) - EOFF + m4;
                if (g >= 1 && static_cast<u64>(g) + 3 < n) {
                    v = __ldg(reinterpret_cast<const float4 *>(e + g));
                } else {
                    v.x = g >= 1 && static_cast<u64>(g) < n ? __ldg(e + g) : 0.f;
                    v.y = g + 1 >= 1 && static_cast<u64>(g + 1) < n ? __ldg(e + g + 1) : 0.f;
                    v.z = g + 2 >= 1 && static_cast<u64>(g + 2) < n ? __ldg(e + g + 2) : 0.f;
                    v.w = g + 3 >= 1 && static_cast<u64>(g + 3) < n ? __ldg(e + g + 3) : 0.f;
                }
            }
            pre[r] = v;
        }
    };
    fetch(blockIdx.x);
    for (u64 tile = blockIdx.x; base + tile * T < n; tile += gridDim.x) {
        const u64 i0 = base + tile * T;
        // ---- e tile: s_e[skew(m)] = e[i0 - EOFF + m] ----
#pragma unroll
        for (int r = 0; r < NPRE; ++r) {
            const u32 m4 = 4 * (tid + 256 * r);
            if (m4 < ENP) *reinterpret_cast<float4 *>(s_e + skew(m4)) = pre[r];
        }
        fetch(tile + gridDim.x);
        __syncthreads();
        // ---- low-pass: warp pair (2h, 2h+1) owns blocks 32h .. 32h+31 of 16 positions; even warp = the first 8 ----
        {
            const u32 blk = (warp >> 1) * 32 + lane;
            if (blk < FNP / 16) {
                if (warp & 1) lp_outputs<NT, 1>(taps, s_e, s_f, blk);
                else lp_outputs<NT, 0>(taps, s_e, s_f, blk);
            }
        }
        if (tid < BOX + 16) s_f[skew(FNP + tid)] = 0.f;   // tail read by the last box sums, never used
        __syncthreads();
        // ---- the tile's own f values go to HBM (f_out is 16-byte aligned, T a multiple of 4) ----
        for (u32 i4 = tid; (!BASED || f_out != nullptr) && i4 < T / 4; i4 += 256) {
            const u64 gi = i0 + 4 * i4;
            if (gi >= n) break;
            const float4 v = *reinterpret_cast<const float4 *>(s_f + skew(4 * i4));
            if (gi + 3 < n) {
                *reinterpret_cast<float4 *>(f_out + gi) = v;
            } else {
                f_out[gi] = v.x;
                if (gi + 1 < n) f_out[gi + 1] = v.y;
                if (gi + 2 < n) f_out[gi + 2] = v.z;
            }
        }
        if (corr_out == nullptr) {
            __syncthreads();
            continue;
        }
        // ---- box sums B[m] = f[m] + ... + f[m+BOX-1], 8 per thread-item, through the pair sums P[k] = f[2k] + f[2k+1]:
        //      B[2u] = P[u] + S_u,  B[2u+1] = f[2u+1] + S_u + f[2u+2PW],  S_u = P[u+1] + ... + P[u+PW-1] ----
        for (u32 item = tid; item < (BN + 7) / 8; item += 256) {
            const u32 o = item * 8;
            constexpr int WB = (8 + BOX - 1 + 3) / 4 * 4;
            float w[WB];
#pragma unroll
            for (int k = 0; k < WB / 4; ++k) {
                const float4 v = *reinterpret_cast<const float4 *>(s_f + skew(o + 4 * k));
                w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
            }
            float pr[WB / 2];
#pragma unroll
            for (int k = 0; k < WB / 2; ++k) pr[k] = w[2 * k] + w[2 * k + 1];
            float b[8];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float s = pr[u + 1];
#pragma unroll
                for (int k = 2; k < PW; ++k) s += pr[u + k];
                b[2 * u] = pr[u] + s;
                b[2 * u + 1] = (w[2 * u + 1] + s) + w[2 * u + BOX];
            }
            *reinterpret_cast<float4 *>(s_b + skew(o)) = make_float4(b[0], b[1], b[2], b[3]);
            *reinterpret_cast<float4 *>(s_b + skew(o + 4)) = make_float4(b[4], b[5], b[6], b[7]);
        }
        __syncthreads();
        // ---- correlation: 16 outputs = 8 packed pairs per thread-item; box pair m (even) belongs to output pairs m - BOX*b ----
        for (u32 item = tid; item < T / 16; item += 256) {
            const u32 o = item * 16;
            if (i0 + o >= ncorr) break;
            constexpr int NB = 16 + 18 * BOX;             // box values this item needs
            constexpr int NBP = (NB + 3) / 4 * 4;
            const f32x2 plus1 = pack2(1.f, 1.f), minus1 = pack2(-1.f, -1.f);
            f32x2 acc[8];
#pragma unroll
            for (int v = 0; v < 8; ++v) acc[v] = 0ull;
#pragma unroll
            for (int k = 0; k < NBP / 4; ++k) {
                const float4 q = *reinterpret_cast<const float4 *>(s_b + skew(o + 4 * k));
                const f32x2 val[2] = {pack2(q.x, q.y), pack2(q.z, q.w)};
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int m = 4 * k + 2 * c;          // box index relative to o (compile time, even)
#pragma unroll
                    for (int b = 0; b < 19; ++b) {
                        const int v = m - BOX * b;        // first output of the pair it contributes to with run b
                        if (v >= 0 && v < 16) {
                            // runs: b = 0 '-', then (-,+) x 7 for b = 1..14, then '-' x 4 (decode.rs:188-198)
                            const bool plus = b >= 1 && b <= 14 && (b % 2 == 0);
                            acc[v / 2] = fma2(val[c], plus ? plus1 : minus1, acc[v / 2]);
                        }
                    }
                }
            }
            float r[16];
#pragma unroll
            for (int v = 0; v < 8; ++v) unpack2(acc[v], r[2 * v], r[2 * v + 1]);
            const u64 gi = i0 + o;
            if (gi + 15 < ncorr) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    *reinterpret_cast<float4 *>(corr_out + gi + 4 * k) = make_float4(r[4 * k], r[4 * k + 1], r[4 * k + 2], r[4 * k + 3]);
            } else {
#pragma unroll
                for (int v = 0; v < 16; ++v)
                    if (gi + v < ncorr) corr_out[gi + v] = r[v];
            }
        }
        __syncthreads();
    }
}

}  // namespace aptb200
