// Polyphase resampler + envelope for LARGE interpolation factors (11025 / 22050 / 44100 Hz -> 12 480 Hz: L = 832 / 416 /
// 208, M = 735; fast_resampling dsp.rs:186-289 + demodulate dsp.rs:350-383), where the 14 057-tap filter gives every
// output only J = 17 / 34 / 68 taps but each of the L outputs of a period has its own tap set.
//
// Formulation (the same rows-by-phases view as kernels_ut.cuh, just with many phases and few taps):
//     y[L*q + r] = sum_{j < J} T[r][j] * X[M*q + xs[r] + j],   xs[r] = ceil(r*M / L),  T[r][j] = h[xs[r]*L - r*M + L*j]
// A warp's 32 lanes are 32 consecutive periods q, so the phase r and with it the tap set and the window start xs[r] are
// WARP-UNIFORM.  Four consecutive phases (a group) read nearly the same samples, so a group shares ONE 16-byte aligned
// window of WIN samples per lane (every period's input span sits in its own shared-memory row, pitch = 4 mod 32 floats:
// the 32 lanes' LDS.128 are conflict-free) and the table stores the group's taps laid out AGAINST that window (zero where
// a phase does not reach): element i of the window meets the four phases' taps as one broadcast LDS.128 and two pair
// FMAs, with compile-time register indices -- no shift variants, a quarter of the shared-memory window traffic of a
// per-phase formulation (which is shared-memory-bandwidth bound).  Ascending window index is
// ascending tap index for every phase: the reference's summation order.  PCM16 input is converted while the rows are
// staged (wav.rs:37 fused into the load).
//
// A warp owns a range of phases for the CTA's 32 periods; consecutive phases of a lane are consecutive outputs, so the
// envelope's predecessor is the previous loop iteration (one extra output per warp for the range start).  Outputs are
// transposed through a small per-warp stage so that every store is 32 consecutive floats of one period.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "kernels_fast.cuh"
#include "kernels_generic.cuh"
#include "launch.hpp"

namespace aptb200 {

constexpr int kPhPeriods = static_cast<int>(kPhTilePeriods);   // periods per tile = lanes
constexpr int kPhWarps = 8;

struct PhGeom {
    u32 l, m;
    u32 j;             // taps per output
    u32 pitch;         // floats per input row (16-byte aligned rows; pitch % 32 == 4)
    u32 row_len;       // staged samples per row: m + jpad + 8 rounded up to 4
    u32 smem_bytes;
};

__device__ __forceinline__ void ph_cp_async4(float *dst, const float *src, bool valid) {
    const u32 bytes = valid ? 4u : 0u;            // src-size 0: nothing is read, the destination is zero-filled
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(static_cast<u32>(__cvta_generic_to_shared(dst))), "l"(src),
                 "r"(bytes) : "memory");
}

// rows of a tile: f32 samples by 4-byte cp.async (a row starts at an arbitrary sample; all copies of a tile are in flight
// together), PCM16 samples through registers, eight loads at a time, converted on the way (wav.rs:37)
__device__ __forceinline__ void ph_stage_row(const float *signal, u64 len, long long gx0, u32 row_len, float *row, u32 lane) {
    // (aligned 16-byte loads through registers + scalar stores at the shifted positions measured slower)
    if (gx0 >= 0 && static_cast<u64>(gx0) + row_len <= len) {
        const float *src = signal + gx0;
        for (u32 i = lane; i < row_len; i += 32) ph_cp_async4(row + i, src + i, true);
    } else {
        for (u32 i = lane; i < row_len; i += 32) {
            const long long gx = gx0 + i;
            const bool ok = gx >= 0 && static_cast<u64>(gx) < len;
            ph_cp_async4(row + i, ok ? signal + gx : signal, ok);
        }
    }
}
__device__ __forceinline__ void ph_stage_row(const int16_t *signal, u64 len, long long gx0, u32 row_len, float *row, u32 lane) {
    for (u32 i0 = lane; i0 < row_len; i0 += 32 * 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const long long gx = gx0 + i0 + 32 * u;
            v[u] = (i0 + 32 * u < row_len && gx >= 0 && static_cast<u64>(gx) < len) ? load_sample(signal, static_cast<u64>(gx)) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (i0 + 32 * u < row_len) row[i0 + 32 * u] = v[u];
    }
}

// Four consecutive phases (one group) of this lane's period from ONE aligned window of WIN samples: window element i
// meets the four taps tg[i] = (T'[4g][i], .., T'[4g+3][i]) -- the group's taps laid out against the common window, zero
// where a phase does not reach -- as two pair FMAs (sample broadcast x tap pair).  Ascending i = ascending tap index
// for every phase: the reference's summation order.
template <int WIN>
__device__ __forceinline__ void ph_group(const float *row, u32 xa, const float4 *tg, float (&y)[4]) {
    float w[WIN];
#pragma unroll
    for (int k = 0; k < WIN / 4; ++k) {
        const float4 q = *reinterpret_cast<const float4 *>(row + xa + 4 * k);
        w[4 * k] = q.x; w[4 * k + 1] = q.y; w[4 * k + 2] = q.z; w[4 * k + 3] = q.w;
    }
    f32x2 a01 = 0ull, a23 = 0ull;
    const ulonglong2 *tp = reinterpret_cast<const ulonglong2 *>(tg);   // the tap pairs as the 64-bit operands they are
#pragma unroll
    for (int i = 0; i < WIN; ++i) {
        const ulonglong2 t = tp[i];                          // warp-uniform address: one broadcast wavefront
        const f32x2 s2 = pack2(w[i], w[i]);
        a01 = fma2(t.x, s2, a01);
        a23 = fma2(t.y, s2, a23);
    }
    unpack2(a01, y[0], y[1]);
    unpack2(a23, y[2], y[3]);
}

// two consecutive groups at once (their tables are adjacent): twice the independent chains in flight
template <int WIN>
__device__ __forceinline__ void ph_group2(const float *row, u32 xa0, u32 xa1, const float4 *tg, float (&y)[8]) {
    float w0[WIN], w1[WIN];
#pragma unroll
    for (int k = 0; k < WIN / 4; ++k) {
        const float4 q = *reinterpret_cast<const float4 *>(row + xa0 + 4 * k);
        w0[4 * k] = q.x; w0[4 * k + 1] = q.y; w0[4 * k + 2] = q.z; w0[4 * k + 3] = q.w;
        const float4 p = *reinterpret_cast<const float4 *>(row + xa1 + 4 * k);
        w1[4 * k] = p.x; w1[4 * k + 1] = p.y; w1[4 * k + 2] = p.z; w1[4 * k + 3] = p.w;
    }
    f32x2 a01 = 0ull, a23 = 0ull, b01 = 0ull, b23 = 0ull;
    const ulonglong2 *tp = reinterpret_cast<const ulonglong2 *>(tg);
#pragma unroll
    for (int i = 0; i < WIN; ++i) {
        const ulonglong2 t = tp[i], u = tp[WIN + i];
        const f32x2 s0 = pack2(w0[i], w0[i]), s1 = pack2(w1[i], w1[i]);
        a01 = fma2(t.x, s0, a01);
        a23 = fma2(t.y, s0, a23);
        b01 = fma2(u.x, s1, b01);
        b23 = fma2(u.y, s1, b23);
    }
    unpack2(a01, y[0], y[1]);
    unpack2(a23, y[2], y[3]);
    unpack2(b01, y[4], y[5]);
    unpack2(b23, y[6], y[7]);
}

template <typename InT, int WIN>
__global__ void __launch_bounds__(32 * kPhWarps, 1)
k_polyphase_ph(const InT *__restrict__ signal, u64 len, const float *__restrict__ table_g, const unsigned short *__restrict__ xa_g,
               const PhGeom g, u64 nout, u64 tile_begin, u64 tile_end, int envelope, float cosphi2, float inv_sinphi,
               float *__restrict__ out) {
    extern __shared__ __align__(16) float ph_smem[];
    const u32 ngroups = g.l / 4;
    float *s_table = ph_smem;                                        // [l/4][WIN][4]
    float *s_rows = s_table + static_cast<size_t>(ngroups) * WIN * 4;   // [33][pitch]: row 0 = the period before the tile
    float *s_stage = s_rows + static_cast<size_t>(kPhPeriods + 1) * g.pitch;   // [warps][32][33]
    unsigned short *s_xa = reinterpret_cast<unsigned short *>(s_stage + kPhWarps * 32 * 33);   // [l/4] window starts (row index)

    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // the 80-KB table by 16-byte cp.async: every copy in flight at once (a load-then-store loop costs one L2 round trip per
    // iteration, 20 of them); completion is awaited with the first tile's rows
    for (u32 i = tid; i < ngroups * WIN; i += blockDim.x)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<u32>(__cvta_generic_to_shared(s_table + 4 * i))),
                     "l"(table_g + 4 * i) : "memory");
    for (u32 i = tid; i < ngroups; i += blockDim.x) s_xa[i] = xa_g[i];

    // groups of this warp (8 groups = 32 phases per staging block)
    const u32 per = (ngroups + kPhWarps - 1) / kPhWarps;
    const u32 ga = min(warp * per, ngroups), gb = min(ga + per, ngroups);
    float *stage = s_stage + warp * (32 * 33);

    for (u64 tile = tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x) {
        const u64 q0 = tile * kPhPeriods;
        __syncthreads();                                             // the rows of the previous tile are no longer read
        // ---- stage the 33 rows: row p holds X[M*(q0 + p - 1) - 4 + i], zero outside [0, len) ----
        for (u32 p = warp; p <= kPhPeriods; p += kPhWarps) {
            const long long gx0 = static_cast<long long>(q0 + p) * g.m - static_cast<long long>(g.m) - 4;
            ph_stage_row(signal, len, gx0, g.row_len, s_rows + p * g.pitch, lane);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        if (ga >= gb) continue;
        const float *row = s_rows + (lane + 1) * g.pitch;            // this lane's period q0 + lane
        const u64 kq = (q0 + lane) * g.l;                            // first output of the period
        float prev = 0.f;
        if (envelope) {
            // r[k-1] of the range's first output: the last phase of the group before, or of the period before
            float y[4];
            if (ga > 0) ph_group<WIN>(row, s_xa[ga - 1], reinterpret_cast<const float4 *>(s_table) + static_cast<size_t>(ga - 1) * WIN, y);
            else ph_group<WIN>(row - g.pitch, s_xa[ngroups - 1], reinterpret_cast<const float4 *>(s_table) + static_cast<size_t>(ngroups - 1) * WIN, y);
            prev = y[3];
        }
        for (u32 g0 = ga; g0 < gb; g0 += 8) {
            const u32 ng = min(8u, gb - g0);
            u32 s = 0;
            for (; s + 1 < ng; s += 2) {                             // two groups per iteration: four independent packed chains
                const u32 gi = g0 + s;
                float y[8];
                ph_group2<WIN>(row, s_xa[gi], s_xa[gi + 1], reinterpret_cast<const float4 *>(s_table) + static_cast<size_t>(gi) * WIN, y);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float o = y[i];
                    if (envelope) {
                        o = (kq + 4 * gi + i == 0) ? 0.f : envelope2_fast(prev, y[i], cosphi2, inv_sinphi);   // dsp.rs:364: e[0] = 0
                        prev = y[i];
                    }
                    stage[lane * 33 + 4 * s + i] = o;
                }
            }
            if (s < ng) {
                const u32 gi = g0 + s;
                float y[4];
                ph_group<WIN>(row, s_xa[gi], reinterpret_cast<const float4 *>(s_table) + static_cast<size_t>(gi) * WIN, y);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float o = y[i];
                    if (envelope) {
                        o = (kq + 4 * gi + i == 0) ? 0.f : envelope2_fast(prev, y[i], cosphi2, inv_sinphi);
                        prev = y[i];
                    }
                    stage[lane * 33 + 4 * s + i] = o;
                }
            }
            __syncwarp();
            // 32 consecutive phases of one period per store
            const u32 nr = 4 * ng;
            for (u32 p = 0; p < kPhPeriods; ++p) {
                const u64 k = (q0 + p) * g.l + 4 * g0 + lane;
                if (lane < nr && k < nout) out[k] = stage[p * 33 + lane];
            }
            __syncwarp();
        }
    }
}

}  // namespace aptb200
