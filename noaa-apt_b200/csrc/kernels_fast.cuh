// Tiled polyphase resampler fused with the envelope demodulator (fast_resampling dsp.rs:186-289 + demodulate
// dsp.rs:350-383).  It served L = 13 until kernels_ut.cuh replaced it there and still serves other small
// interpolation factors (L <= 13 groups, e.g. L = 26); the mbarrier / TMA / fp32-pair helpers below are shared by both.
//
// Formulation.  y[k] = sum_x h[x*L - k*M] * X[x].  Outputs k and k + P_out (P_out = lcm(8, L)) use the
// same taps on inputs shifted by P_in = P_out*M/L, so per "group" g (outputs 8g..8g+7 of a super-period)
//     acc[r][q] += T_g[u][r] * X[tile_x0 + q*P_in + w0_g + u]        r < 8, q < QT
// with w0_g the first input sample the group touches (rounded down to a multiple of 4 for 16-byte loads)
// and T_g the zero-padded slice of h its outputs see.  The group's two halves (outputs 0..3 / 4..7) have
// windows offset by `shift` samples, so the first shift/16 loop iterations skip half B and the last skip A.
//
// Structure.  One persistent, warp-specialised CTA per SM:
//   producer warp  : 1-D TMA bulk copies (cp.async.bulk -> UBLKCP) of the next tiles' 32 input rows + one
//                    halo row into the free row stages (3 where shared memory allows, else 2: up to stages-1
//                    tiles in flight while one is computed), completion on an mbarrier;
//   compute warps  : one per group, except that with G = 13 there are 12 and warps 0..3 also compute 8 rows each
//                    of group 12 (see the warp roles below).  A warp's 32 lanes are KS=4 interleaved slices of the sample axis x 8 row
//                    lanes; a thread owns 8 outputs x 4 rows as 16 fp32 accumulator pairs.  Per loop
//                    iteration: 4 LDS.128 of samples (the 8 row lanes of a quarter-warp hit 8 distinct 16-byte
//                    bank groups because the row pitch/4 is odd), 8 warp-broadcast LDS.128 of taps (4 distinct
//                    addresses skewed across bank groups) and 64 pair FMAs (tap pair x broadcast sample).  For
//                    the loop shapes of the plans in use the loop is fully unrolled (tile_main_fixed), with the
//                    next iteration's sample loads in flight during the current one's FMAs.
//                    After the loop the four slices' partial sums are reduced by two shuffle rounds, and each
//                    lane turns 4 consecutive outputs of 2 rows into the envelope (dsp.rs:373) and stores them
//                    as float4.  The resampled signal itself never reaches HBM.  The output before a group's
//                    first one belongs to the previous warp: warps publish their last output per row in a small
//                    exchange array (one named barrier among the compute warps per tile); r[K0-1] comes from the
//                    halo row (window of the last group of the previous super-period), computed by one compute warp.
// Stages are handed over with full/empty mbarriers; the tap table is bulk-copied once per CTA.
#pragma once

#include <cstdint>
#include <type_traits>
#include <cuda_runtime.h>

#include "kernels_generic.cuh"
#include "launch.hpp"

namespace aptb200 {

// ---- mbarrier / TMA bulk-copy wrappers (PTX ISA: cp.async.bulk, mbarrier) -------------------------
__device__ __forceinline__ u32 smem_u32(const void *p) { return static_cast<u32>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(void *bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void *bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(void *bar, u32 parity) {
    u32 ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"   // suspend-time hint: sleep, don't spin
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(void *bar, u32 parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// global -> shared bulk copy, `bytes` a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, u32 bytes, void *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// warm L2 with a span of global memory (no shared-memory destination, no completion tracking)
__device__ __forceinline__ void tma_prefetch_l2(const void *src, u32 bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

constexpr int kTileR = 8, kTileH = 4, kTileQ = 4, kTileKS = 4;
constexpr int kTileRowLanes = 32 / kTileKS;           // 8
constexpr int kTileQT = kTileRowLanes * kTileQ;       // 32 rows per tile

// ---- fp32 pair helpers: a register pair holding two independent accumulators.  sm_90 has no packed fp32 FMA,
// so fma2 is two FFMAs, each half rounded on its own (the pack / unpack moves are register-pair aliases in SASS) ----
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pack2(float lo, float hi) {
    f32x2 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void unpack2(f32x2 v, float &lo, float &hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
    float a0, a1, b0, b1, c0, c1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    unpack2(c, c0, c1);
    return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ float4 lds128(u32 addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}

// One half (4 outputs, as two packed pairs) x Q rows x the 4 consecutive samples of one 16-byte chunk.
// acc[p][j] packs outputs (2p, 2p+1) of row j; the tap pair comes straight out of the LDS.128 register quad,
// the sample is duplicated into both lanes of the packed operand.
template <int Q>
__device__ __forceinline__ void half_fma2(f32x2 (&acc)[2][Q], u32 tap_addr, const float4 (&s)[Q]) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const float4 tp = lds128(tap_addr + 16 * u);  // taps of outputs r = 0..3 for sample u of the chunk
        const f32x2 t01 = pack2(tp.x, tp.y), t23 = pack2(tp.z, tp.w);
#pragma unroll
        for (int j = 0; j < Q; ++j) {
            const float sv = u == 0 ? s[j].x : u == 1 ? s[j].y : u == 2 ? s[j].z : s[j].w;
            const f32x2 sv2 = pack2(sv, sv);
            acc[0][j] = fma2(t01, sv2, acc[0][j]);
            acc[1][j] = fma2(t23, sv2, acc[1][j]);
        }
    }
}

// The main loop of one group over Q rows of a tile (row j at row_addr[j]): iterations [0, it_b_begin) run half A only,
// [it_b_begin, it_a_end) both halves, [it_a_end, iters) half B only.  Any plan shape.
template <int Q>
__device__ __forceinline__ void tile_main_runtime(f32x2 (&acc_a)[2][Q], f32x2 (&acc_b)[2][Q], u32 tap_addr,
                                                  const u32 (&row_addr)[Q], u32 it_b_begin, u32 it_a_end, u32 iters,
                                                  u32 rec_bytes) {
    u32 row_off = 0, it = 0;
    for (; it < it_b_begin; ++it) {                        // half A only
        float4 s[Q];
#pragma unroll
        for (int j = 0; j < Q; ++j) s[j] = lds128(row_addr[j] + row_off);
        half_fma2(acc_a, tap_addr, s);
        row_off += kTileKS * 16;
        tap_addr += rec_bytes;
    }
    for (; it < it_a_end; ++it) {                          // both halves
        float4 s[Q];
#pragma unroll
        for (int j = 0; j < Q; ++j) s[j] = lds128(row_addr[j] + row_off);
        half_fma2(acc_a, tap_addr, s);
        half_fma2(acc_b, tap_addr + 64, s);
        row_off += kTileKS * 16;
        tap_addr += rec_bytes;
    }
    for (; it < iters; ++it) {                             // half B only
        float4 s[Q];
#pragma unroll
        for (int j = 0; j < Q; ++j) s[j] = lds128(row_addr[j] + row_off);
        half_fma2(acc_b, tap_addr + 64, s);
        row_off += kTileKS * 16;
        tap_addr += rec_bytes;
    }
}

// The same loop for a plan shape known at compile time: ITERS iterations, half B active from BB on, half A up to AE,
// HALVES tap records per (iteration, slice lane).  Fully unrolled, every shared-memory address is a register plus an
// immediate, so there is no loop-carried register renaming.  The Q sample quads are double-buffered in registers and
// those of iteration it+1 are requested before the FMAs of iteration it, which hides the LDS latency behind them.  The
// tap quads are loaded in source order next to the FMAs that use them; how far ahead of those FMAs they are issued is
// left to ptxas's scheduling of the unrolled body.  Each accumulator sees the same FMAs in the same order as in
// tile_main_runtime, so the results are bit-identical.
template <int Q, int ITERS, int BB, int AE, int HALVES>
__device__ __forceinline__ void tile_main_fixed(f32x2 (&acc_a)[2][Q], f32x2 (&acc_b)[2][Q], u32 tap_addr,
                                                const u32 (&row_addr)[Q]) {
    constexpr u32 rec_bytes = HALVES * 64;
    float4 s[2][Q];
#pragma unroll
    for (int j = 0; j < Q; ++j) s[0][j] = lds128(row_addr[j]);
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        if (it + 1 < ITERS) {
#pragma unroll
            for (int j = 0; j < Q; ++j) s[(it + 1) & 1][j] = lds128(row_addr[j] + (it + 1) * kTileKS * 16);
        }
        if (it < AE) half_fma2(acc_a, tap_addr + it * rec_bytes, s[it & 1]);
        if (it >= BB) half_fma2(acc_b, tap_addr + it * rec_bytes + 64, s[it & 1]);
    }
}

__device__ __forceinline__ void mbar_arrive(void *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// barrier `id` among the first `nthreads` threads (a multiple of 32) of the CTA; orders their shared-memory accesses
__device__ __forceinline__ void named_bar_sync(u32 id, u32 nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// group_xs[g] = w0_g, the (4-aligned) first input sample of group g relative to its row.  ITERS > 0: the plan's loop
// shape (tp.iters, first iteration of half B, end of half A, halves) is <ITERS, BB, AE, HALVES> and the main loop is
// tile_main_fixed; ITERS == 0: any shape, runtime loop bounds.  The block is tp.compute_warps + 1 warps, at most 13.
template <bool ENVELOPE, int ITERS, int BB, int AE, int HALVES>
__global__ void __launch_bounds__(32 * (kTileMaxComputeWarps + 1), 1)
k_polyphase_ws(const float *__restrict__ signal, u64 len, const float *__restrict__ tile_taps,
               const u32 *__restrict__ group_xs, TilePlan tp, u64 nout, u64 tile_begin, u64 ntiles, float cosphi2,
               float sinphi, float *__restrict__ out, unsigned long long *__restrict__ prof) {
    // tiles [tile_begin, ntiles) are computed; `signal` may be a biased pointer into a chunk buffer (signal + x is
    // valid for every sample x those tiles touch), `len` is always the length of the whole signal
    constexpr int Q = kTileQ, KS = kTileKS, QT = kTileQT;
    // optional phase timing (APTB200_TILE_PROFILE): cycles summed over the tiles of CTA 0, lane 0 of one warp per role
    const bool profiling = prof != nullptr && blockIdx.x == 0 && (threadIdx.x & 31) == 0;
    const long long t_kernel0 = clock64();
    long long pt[3] = {0, 0, 0}, t_mark = 0;
#define PROF_MARK() do { if (profiling) t_mark = clock64(); } while (0)
#define PROF_ADD(i) do { if (profiling) { const long long now__ = clock64(); pt[i] += now__ - t_mark; t_mark = now__; } } while (0)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // layout: [7 mbarriers, 128 B][taps][stage 0: rows, halo row]...[stage S-1][exchange: 2 x G x (1 + QT)]
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(smem_raw);
    unsigned long long *bar_taps = bars + 0;
    unsigned long long *full_rows = bars + 1;     // [stages] TMA -> compute
    unsigned long long *empty_rows = bars + 4;    // [stages] compute -> producer
    float *s_taps = reinterpret_cast<float *>(smem_raw + 128);
    float *s_stage0 = s_taps + tp.groups * tp.group_stride;
    float *s_xch = s_stage0 + tp.stages * tp.stage_floats;

    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 G = tp.groups, CW = tp.compute_warps;
    const u32 tile_out = QT * tp.p_out;

    if (tid == 0) {
        mbar_init(bar_taps, 1);
        for (u32 s = 0; s < tp.stages; ++s) {
            mbar_init(full_rows + s, 1);
            mbar_init(empty_rows + s, CW);
        }
        fence_mbar_init();
    }
    __syncthreads();

    // Warp roles: compute warps 0..CW-1, then the producer.  Warps are spread over the 4 SM sub-partitions round-robin
    // (warp % 4).  With G <= 12 groups compute warp g owns group g.  With G = 13 there are 12 compute warps, 3 per
    // sub-partition: warp g owns group g < 12, and the 32 rows of group 12 are split over warps 0..3, one on each
    // sub-partition, 8 rows each (one per row lane).  Each sub-partition then carries 3.25 groups per tile instead of 4
    // on one and 3 on the others.  The producer (warp 12) lands on sub-partition 0, the halo dot product on warp 6
    // (sub-partition 2); both are light next to a group.
    const bool is_producer = warp == CW;
    if (is_producer) {
        // ======================================= producer =======================================
        const bool aligned16 = (reinterpret_cast<uintptr_t>(signal) & 15) == 0;
        const u32 w0_last = group_xs[G - 1];
        if (lane == 0) {
            fence_proxy_async();
            const u32 total = G * tp.group_stride * 4;
            mbar_expect_tx(bar_taps, total);
            for (u32 done = 0; done < total; done += 32768u)
                tma_bulk_g2s(reinterpret_cast<unsigned char *>(s_taps) + done,
                             reinterpret_cast<const unsigned char *>(tile_taps) + done, min(total - done, 32768u), bar_taps);
        }
        u32 st = 0, ph = 0;                                                  // stage and its phase parity
        for (u64 tile = tile_begin + blockIdx.x; tile < ntiles; tile += gridDim.x) {
            float *rows = s_stage0 + st * tp.stage_floats;
            float *vrow = rows + tp.rows_floats;
            const u64 x_base = tile * static_cast<u64>(QT) * tp.p_in;       // first input sample of row 0
            const u64 x_end = x_base + static_cast<u64>(QT - 1) * tp.p_in + tp.row_len;
            const bool want_halo = ENVELOPE && tile > 0;
            const u64 x_halo = x_base - tp.p_in + w0_last;                   // meaningful only when tile > 0
            PROF_MARK();
            mbar_wait(empty_rows + st, ph ^ 1);                              // stage free (first use passes)
            PROF_ADD(0);
            if (tp.debug == 2) {
                if (lane == 0) mbar_arrive(full_rows + st);
            } else if (aligned16) {
                // One bulk copy per row pair (rows 2i, 2i+1 overlap in the signal).  The part of a pair that
                // exists (a multiple of 4 floats) comes by TMA; the rest -- the last <4 samples and everything
                // past the end of the signal, which reads as zero (signal.get(x) == None, dsp.rs:257) -- by this
                // warp's own stores.  Interior tiles are pure TMA.
                const u32 rpc = tp.rows_per_copy, ncopies = QT / rpc;
                const u32 pair_len = (rpc - 1) * tp.p_in + tp.row_len;
                const u64 halo_end = x_halo + tp.usteps;
                const bool edge = x_end > len || (want_halo && halo_end > len);
                auto valid_of = [&](u64 x0, u32 nfl) -> u32 {
                    return x0 >= len ? 0u : static_cast<u32>(min(static_cast<u64>(nfl), len - x0));
                };
                if (edge) {
                    for (u32 i = 0; i < ncopies; ++i) {
                        const u64 xr = x_base + static_cast<u64>(rpc * i) * tp.p_in;
                        const u32 valid = valid_of(xr, pair_len);
                        for (u32 c = (valid & ~3u) + lane; c < pair_len; c += 32)
                            rows[i * tp.pair_pitch + c] = c < valid ? __ldg(signal + xr + c) : 0.f;
                    }
                    if (want_halo) {
                        const u32 valid = valid_of(x_halo, tp.usteps);
                        for (u32 c = (valid & ~3u) + lane; c < tp.usteps; c += 32)
                            vrow[c] = c < valid ? __ldg(signal + x_halo + c) : 0.f;
                    }
                    __syncwarp();                 // the warp's stores are ordered before lane 0's release-arrive
                }
                if (lane == 0) {
                    fence_proxy_async();          // the stage was last read through the generic proxy
                    if (!edge) {
                        mbar_expect_tx(full_rows + st, (ncopies * pair_len + (want_halo ? tp.usteps : 0)) * 4);
                        for (u32 i = 0; i < ncopies; ++i)
                            tma_bulk_g2s(rows + i * tp.pair_pitch, signal + x_base + static_cast<u64>(rpc * i) * tp.p_in,
                                         pair_len * 4, full_rows + st);
                        if (want_halo) tma_bulk_g2s(vrow, signal + x_halo, tp.usteps * 4, full_rows + st);
                    } else {
                        u32 tx_floats = want_halo ? (valid_of(x_halo, tp.usteps) & ~3u) : 0u;
                        for (u32 i = 0; i < ncopies; ++i)
                            tx_floats += valid_of(x_base + static_cast<u64>(rpc * i) * tp.p_in, pair_len) & ~3u;
                        mbar_expect_tx(full_rows + st, tx_floats * 4);
                        for (u32 i = 0; i < ncopies; ++i) {
                            const u64 xr = x_base + static_cast<u64>(rpc * i) * tp.p_in;
                            const u32 nfl = valid_of(xr, pair_len) & ~3u;
                            if (nfl) tma_bulk_g2s(rows + i * tp.pair_pitch, signal + xr, nfl * 4, full_rows + st);
                        }
                        if (want_halo) {
                            const u32 nfl = valid_of(x_halo, tp.usteps) & ~3u;
                            if (nfl) tma_bulk_g2s(vrow, signal + x_halo, nfl * 4, full_rows + st);
                        }
                    }
                }
            } else {
                // unaligned signal pointer: the warp fills the whole stage itself (slow, correct)
                const u32 rpc = tp.rows_per_copy;
                const u32 pair_len = (rpc - 1) * tp.p_in + tp.row_len;
                for (u32 i = 0; i < QT / rpc; ++i)
                    for (u32 c = lane; c < pair_len; c += 32) {
                        const u64 x = x_base + static_cast<u64>(rpc * i) * tp.p_in + c;
                        rows[i * tp.pair_pitch + c] = x < len ? __ldg(signal + x) : 0.f;
                    }
                if (want_halo)
                    for (u32 i = lane; i < tp.usteps; i += 32) vrow[i] = x_halo + i < len ? __ldg(signal + x_halo + i) : 0.f;
                __syncwarp();
                if (lane == 0) mbar_arrive(full_rows + st);
            }
            PROF_ADD(1);
            if (++st == tp.stages) { st = 0; ph ^= 1; }
        }
        if (profiling) { prof[0] = pt[0]; prof[1] = pt[1]; }
    } else {
        // ======================================= compute ========================================
        const u32 ks = lane >> 3, ql = lane & 7;
        const u32 it_a_end = tp.half_taps / 16;       // half A is active for iterations [0, it_a_end)
        const u32 it_b_begin = tp.halves == 2 ? tp.shift / 16 : tp.iters;   // half B for [it_b_begin, iters)
        const u32 rec_bytes = tp.halves * 64;         // one (iteration, slice lane) tap record
        const u32 R = 4 * tp.halves;
        const u32 row_step8 = (8 / tp.rows_per_copy) * tp.pair_pitch * 4;
        // row r lives at pair r/2, half r%2; this thread reads rows ql, ql+8, ql+16, ql+24 of its group
        const u32 lane_row = (tp.rows_per_copy == 2 ? (ql >> 1) * tp.pair_pitch + (ql & 1) * tp.p_in : ql * tp.pair_pitch) * 4;
        const u32 row_off = lane_row + (group_xs[warp] + ks * 4) * 4;
        const u32 tap_base = smem_u32(s_taps) + (warp * tp.group_stride + ks * tp.slice_stride) * 4;
        // G > CW: warps 0..3 also compute group G-1 in row qx = ql + 8*warp (one row per row lane)
        const bool split = G > CW && warp < 4;
        const u32 gx = G - 1, qx = ql + 8 * warp;
        const u32 row_off_x = lane_row + (group_xs[gx] + ks * 4) * 4 + warp * row_step8;
        const u32 tap_base_x = smem_u32(s_taps) + (gx * tp.group_stride + ks * tp.slice_stride) * 4;
        // after the reduction this lane holds outputs 4*hsel..4*hsel+3 of the group in rows q0 and q0 + 8
        const u32 hsel = ks & 1, rsel = ks >> 1, q0 = ql + 16 * rsel;
        const u32 halo_warp = G > CW ? 6 : G > 2 ? 2 : G - 1;
        const float inv_sinphi = 1.f / sinphi;
        const bool out_aligned = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
        // one group's main loop over the Q rows at row_addr
        auto main_loop = [&](auto &acc_a, auto &acc_b, u32 tap_addr, const auto &row_addr) {
            constexpr int NQ = static_cast<int>(std::extent_v<std::remove_reference_t<decltype(row_addr)>>);
            if constexpr (ITERS > 0) tile_main_fixed<NQ, ITERS, BB, AE, HALVES>(acc_a, acc_b, tap_addr, row_addr);
            else tile_main_runtime<NQ>(acc_a, acc_b, tap_addr, row_addr, it_b_begin, it_a_end, tp.iters, rec_bytes);
        };
        mbar_wait(bar_taps, 0);
        u32 n = 0, st = 0, ph = 0;
        for (u64 tile = tile_begin + blockIdx.x; tile < ntiles; tile += gridDim.x, ++n) {
            const float *rows = s_stage0 + st * tp.stage_floats;
            PROF_MARK();
            mbar_wait(full_rows + st, ph);
            PROF_ADD(0);
            f32x2 acc_a[2][Q], acc_b[2][Q], xa[2][1], xb[2][1];
#pragma unroll
            for (int p = 0; p < 2; ++p) {
#pragma unroll
                for (int j = 0; j < Q; ++j) acc_a[p][j] = acc_b[p][j] = 0ull;
                xa[p][0] = xb[p][0] = 0ull;
            }
            if (tp.debug != 1 && tp.debug < 5) {
                const u32 rbase = smem_u32(rows) + row_off;
                const u32 row_addr[Q] = {rbase, rbase + row_step8, rbase + 2 * row_step8, rbase + 3 * row_step8};
                main_loop(acc_a, acc_b, tap_base, row_addr);
                if (split) {
                    const u32 row_addr_x[1] = {smem_u32(rows) + row_off_x};
                    main_loop(xa, xb, tap_base_x, row_addr_x);
                }
            }
            // r[K0 - 1]: the last output of the last group, applied to the halo row -- by a warp that owns no rows of
            // group G-1 and shares its sub-partition only with other compute warps
            float halo = 0.f;
            if (ENVELOPE && warp == halo_warp && tile > 0) {
                const float *vrow = rows + tp.rows_floats;
                const float *tg = s_taps + static_cast<size_t>(G - 1) * tp.group_stride;
                // the group's last output: r = 3 of half B (two halves) or of half A (one)
                const u32 rec = 16 * tp.halves, off = tp.halves == 2 ? 16 + 3 : 3;
                const u32 ubeg = tp.halves == 2 ? tp.shift : 0, uend = tp.halves == 2 ? tp.usteps : tp.half_taps;
                for (u32 u = ubeg + lane; u < uend; u += 32) {
                    const u32 chunk = u >> 2, uu = u & 3;            // chunk = it*KS + ks
                    halo = fmaf(tg[(chunk & 3) * tp.slice_stride + (chunk >> 2) * rec + off + uu * 4], vrow[u], halo);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) halo += __shfl_xor_sync(0xffffffffu, halo, o);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_rows + st);           // this warp is done with the stage
            if (++st == tp.stages) { st = 0; ph ^= 1; }
            PROF_ADD(1);
            // Reduce the four slice lanes' partial sums: the xor-8 round keeps half `hsel`, the xor-16 round rows q0 and
            // q0 + 8.  Every sum is (ks0 + ks1) + (ks2 + ks3) up to the order of the operands of one addition.
            float v[2][Q][4];                                       // [half][row j: ql + 8j][output]
#pragma unroll
            for (int j = 0; j < Q; ++j) {
                unpack2(acc_a[0][j], v[0][j][0], v[0][j][1]);
                unpack2(acc_a[1][j], v[0][j][2], v[0][j][3]);
                unpack2(acc_b[0][j], v[1][j][0], v[1][j][1]);
                unpack2(acc_b[1][j], v[1][j][2], v[1][j][3]);
            }
            float w[Q][4], r[2][4];
#pragma unroll
            for (int j = 0; j < Q; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float send = hsel ? v[0][j][e] : v[1][j][e];
                    w[j][e] = (hsel ? v[1][j][e] : v[0][j][e]) + __shfl_xor_sync(0xffffffffu, send, 8);
                }
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float send = rsel ? w[jj][e] : w[2 + jj][e];
                    r[jj][e] = (rsel ? w[2 + jj][e] : w[jj][e]) + __shfl_xor_sync(0xffffffffu, send, 16);
                }
            // the same for the row of group G-1: lanes with rsel == 0 hold its outputs 4*hsel..4*hsel+3
            float rx[4] = {0.f, 0.f, 0.f, 0.f};
            if (split) {
                float vx[2][4];
                unpack2(xa[0][0], vx[0][0], vx[0][1]);
                unpack2(xa[1][0], vx[0][2], vx[0][3]);
                unpack2(xb[0][0], vx[1][0], vx[1][1]);
                unpack2(xb[1][0], vx[1][2], vx[1][3]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float send = hsel ? vx[0][e] : vx[1][e];
                    const float wx = (hsel ? vx[1][e] : vx[0][e]) + __shfl_xor_sync(0xffffffffu, send, 8);
                    rx[e] = wx + __shfl_xor_sync(0xffffffffu, wx, 16);
                }
            }
            float prev[2] = {0.f, 0.f}, prev_x = 0.f;
            if (ENVELOPE) {
                // Previous output of each lane's first one: output 3 of half A in the neighbouring lane (half B), else the
                // last output of the previous group in the same row, of the last group in the previous row, or the halo.
                // The exchange array [tile parity][group][1 + row] holds each group's last output per row (row -1: halo).
                float *xch = s_xch + (n & 1) * G * (QT + 1);
                if (hsel == tp.halves - 1) {
                    xch[warp * (QT + 1) + 1 + q0] = r[0][3];
                    xch[warp * (QT + 1) + 9 + q0] = r[1][3];
                    if (split && rsel == 0) xch[gx * (QT + 1) + 1 + qx] = rx[3];
                }
                if (warp == halo_warp && lane == 0) xch[(G - 1) * (QT + 1)] = halo;
                named_bar_sync(1, 32 * CW);
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const float left = __shfl_xor_sync(0xffffffffu, r[jj][3], 8);
                    const u32 q = q0 + 8 * jj;
                    prev[jj] = hsel ? left : warp > 0 ? xch[(warp - 1) * (QT + 1) + 1 + q] : xch[(G - 1) * (QT + 1) + q];
                }
                if (split) {
                    const float left = __shfl_xor_sync(0xffffffffu, rx[3], 8);
                    prev_x = hsel ? left : xch[(gx - 1) * (QT + 1) + 1 + qx];
                }
            }
            // envelope and store of outputs 4*hsel..4*hsel+3 of group g in row q (one half only: lanes of half B store
            // nothing)
            const u64 k_base = tile * tile_out;
            const bool full_tile = k_base + tile_out <= nout && out_aligned;
            auto finish = [&](u32 g, u32 q, const float (&y)[4], float before) {
                const u32 kl = q * tp.p_out + g * R + 4 * hsel;   // output index inside the tile
                float4 res = make_float4(y[0], y[1], y[2], y[3]);
                if (ENVELOPE) {
                    res.x = envelope2_fast(before, y[0], cosphi2, inv_sinphi);
                    res.y = envelope2_fast(y[0], y[1], cosphi2, inv_sinphi);
                    res.z = envelope2_fast(y[1], y[2], cosphi2, inv_sinphi);
                    res.w = envelope2_fast(y[2], y[3], cosphi2, inv_sinphi);
                    if (kl == 0 && k_base == 0) res.x = 0.f;     // output[0] = 0 (dsp.rs:357)
                }
                if (full_tile) {
                    *reinterpret_cast<float4 *>(out + k_base + kl) = res;
                } else {
                    const u64 k = k_base + kl;
                    if (k < nout) out[k] = res.x;
                    if (k + 1 < nout) out[k + 1] = res.y;
                    if (k + 2 < nout) out[k + 2] = res.z;
                    if (k + 3 < nout) out[k + 3] = res.w;
                }
            };
            if (hsel < tp.halves) {
                finish(warp, q0, r[0], prev[0]);
                finish(warp, q0 + 8, r[1], prev[1]);
                if (split && rsel == 0) finish(gx, qx, rx, prev_x);
            }
            PROF_ADD(2);
        }
        if (profiling && warp == 0) { prof[2] = pt[0]; prof[3] = pt[1]; prof[4] = pt[2]; prof[8] = n; }
        if (profiling && warp < 4) prof[9 + warp] = pt[1];   // main loops of warps 0..3, one per SM sub-partition
        if (prof != nullptr && warp == 0 && lane == 0) {   // per-CTA wall time of the whole kernel body + SM id
            u32 smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            prof[16 + 2 * blockIdx.x] = clock64() - t_kernel0;
            prof[17 + 2 * blockIdx.x] = smid;
        }
    }
#undef PROF_MARK
#undef PROF_ADD
}

}  // namespace aptb200
