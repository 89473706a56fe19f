// Averaged power spectrum of I/Q segments (DESIGN.md §10, "Finding carriers"): load + convert (as k_fm_demod), periodic
// Hann window, an nfft-point DFT by a Stockham FFT in shared memory, |X|^2 summed over the segments.
//
// A CTA transforms whole segments.  Segment k adds its |X|^2 into partial spectrum slot k mod kSpecSlots; the CTA of a
// slot takes that slot's segments of the launch in ascending k and starts from the slot's stored sums, so every slot
// holds ((0 + P_s) + P_{s+G}) + ... in the same order however the segments are split into launches.  k_spectrum_finish
// then adds the slots in slot order.  No atomics: the result is the same bits on every run and for every chunk size.
//
// FFT: nfft = 2^L, one radix-2 stage first when L is odd (its twiddles are all 1), then radix-4 stages.  A stage with
// sub-transform size Ns and radix R takes butterfly j's inputs x[j + r N/R], multiplies input r by
// tw[r (j mod Ns) N / (Ns R)] (tw[t] = exp(-2 pi i t / N), a table), transforms them and writes output r to
// y[(j - j mod Ns) R + j mod Ns + r Ns] (Stockham autosort: natural order in, natural order out).  Every thread reads its
// butterflies' inputs into registers before a barrier and writes after it, so x and y share one buffer.  The first stage
// reads the windowed samples from global memory; the last stage adds |y|^2 into the CTA's running sums, which each thread
// owns at bins tid + m * blockDim (the same bins for every segment, so they need no barrier).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "kernels_iq.cuh"

namespace aptb200 {

constexpr u32 kSpecSlots = 256;        // partial spectra (G)
constexpr u32 kSpecMinN = 256, kSpecMaxN = 16384;

struct SpecArgs {
    const void *in;               // segment k of the launch starts at sample (k - k0) * nfft of `in` (packed)
    u32 nfft, log2n;
    const float2 *tw;             // nfft twiddles exp(-2 pi i t / nfft)
    const float *win;             // nfft periodic Hann taps
    u64 k0, k1;                   // segments [k0, k1)
    float *partial;               // kSpecSlots x nfft running sums
};

__device__ __forceinline__ float2 cadd_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 csub_rn(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float power_rn(float2 a) { return __fadd_rn(__fmul_rn(a.x, a.x), __fmul_rn(a.y, a.y)); }

// threads per CTA for an nfft-point transform: one radix-4 butterfly per thread up to 512 threads (at most 8 radix-4 or
// 8 radix-2 butterflies per thread, whose inputs stay in registers across the stage's barrier)
constexpr u32 kSpecThreads = 512;
__host__ __device__ constexpr u32 spec_threads(u32 nfft) { return nfft / 4 < kSpecThreads ? nfft / 4 : kSpecThreads; }

// B4: radix-4 butterflies per thread (nfft / 4 / blockDim.x: 1, 2, 4 or 8); the radix-2 stage has 2 B4
template <int FMT, int B4>
__global__ void __launch_bounds__(kSpecThreads) k_spectrum(const SpecArgs a) {
    extern __shared__ float2 sx[];
    float *acc = reinterpret_cast<float *>(sx + a.nfft);
    const u32 N = a.nfft, T = blockDim.x, tid = threadIdx.x;
    const u32 q4 = N / 4;
    const u64 first = a.k0 + blockIdx.x;
    float *part = a.partial + static_cast<size_t>(first % kSpecSlots) * N;
    for (u32 b = tid; b < N; b += T) acc[b] = part[b];

    for (u64 k = first; k < a.k1; k += kSpecSlots) {
        const u64 base = (k - a.k0) * N;
        auto load = [&](u32 t) {
            const float2 x = iq_load<FMT>(a.in, base + t);
            const float w = __ldg(a.win + t);
            return make_float2(__fmul_rn(x.x, w), __fmul_rn(x.y, w));
        };
        u32 Ns = 1;
        if (B4 < 8 && (a.log2n & 1)) {   // B4 == 8 only at nfft 16384, an even power: no radix-2 stage to compile
            float2 v[2 * B4][2];
#pragma unroll
            for (int i = 0; i < 2 * B4; ++i) {
                const u32 j = tid + i * T;
                v[i][0] = load(j);
                v[i][1] = load(j + N / 2);
            }
            __syncthreads();   // the previous segment's last stage has read the buffer
#pragma unroll
            for (int i = 0; i < 2 * B4; ++i) {
                    const u32 j = tid + i * T;
                    sx[2 * j] = cadd_rn(v[i][0], v[i][1]);
                    sx[2 * j + 1] = csub_rn(v[i][0], v[i][1]);
                }
            __syncthreads();
            Ns = 2;
        }
        for (; Ns < N; Ns *= 4) {
            float2 v[B4][4];
#pragma unroll
            for (int i = 0; i < B4; ++i) {
                const u32 j = tid + i * T;
#pragma unroll
                for (int r = 0; r < 4; ++r) v[i][r] = Ns == 1 ? load(j + r * q4) : sx[j + r * q4];
            }
            __syncthreads();
            const u32 stride = N / (Ns * 4);
            const bool last = Ns * 4 == N;
#pragma unroll
            for (int i = 0; i < B4; ++i) {
                    const u32 j = tid + i * T, kk = j & (Ns - 1);
                    if (Ns > 1) {
#pragma unroll
                        for (int r = 1; r < 4; ++r) v[i][r] = cmul_rn(v[i][r], __ldg(a.tw + r * kk * stride));
                    }
                    const float2 a0 = cadd_rn(v[i][0], v[i][2]), a1 = csub_rn(v[i][0], v[i][2]);
                    const float2 a2 = cadd_rn(v[i][1], v[i][3]), d = csub_rn(v[i][1], v[i][3]);
                    const float2 a3 = make_float2(d.y, -d.x);   // -i (v1 - v3)
                    const float2 y[4] = {cadd_rn(a0, a2), cadd_rn(a1, a3), csub_rn(a0, a2), csub_rn(a1, a3)};
                    if (last) {
#pragma unroll
                        for (int r = 0; r < 4; ++r) acc[j + r * q4] = __fadd_rn(acc[j + r * q4], power_rn(y[r]));
                    } else {
                        const u32 o = (j - kk) * 4 + kk;
#pragma unroll
                        for (int r = 0; r < 4; ++r) sx[o + r * Ns] = y[r];
                    }
                }
            if (!last) __syncthreads();
        }
    }
    for (u32 b = tid; b < N; b += T) part[b] = acc[b];
}

// psd[b] = (sum over slots s < nslots, ascending, of partial[s][(b + nfft/2) mod nfft]) / K: the fftshifted average.
__global__ void __launch_bounds__(256) k_spectrum_finish(const float *__restrict__ partial, u32 nslots, u32 nfft, float K,
                                                         float *__restrict__ psd) {
    const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nfft) return;
    const u32 src = (b + nfft / 2) & (nfft - 1);
    float s = partial[src];
    for (u32 k = 1; k < nslots; ++k) s = __fadd_rn(s, partial[static_cast<size_t>(k) * nfft + src]);
    psd[b] = __fdiv_rn(s, K);
}

}  // namespace aptb200
