// Generic (any L/M/tap-count) kernels of the decode path.  One thread per output,
// summation in the reference's order with one FMA per tap.  They are the
// correctness baseline for every configuration; the tiled sm_90a fast paths in
// kernels_fast.cuh take over for the shapes the standard profiles produce.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "launch.hpp"

namespace aptb200 {


// wav.rs:37 -- the `as f32` cast of load_wav, fused into the sample load.
__device__ __forceinline__ float load_sample(const float *p, u64 i) { return __ldg(p + i); }
__device__ __forceinline__ float load_sample(const int16_t *p, u64 i) {
    return static_cast<float>(static_cast<int>(__ldg(p + i)));
}

// dsp.rs:373 with every operation rounded on its own (no FMA contraction): given the same two
// resampled samples this is bit-identical to the reference.
__device__ __forceinline__ float envelope2(float prev, float curr, float cosphi2, float sinphi) {
    const float sq = __fadd_rn(__fmul_rn(prev, prev), __fmul_rn(curr, curr));
    const float cross = __fmul_rn(__fmul_rn(prev, curr), cosphi2);
    return __fdiv_rn(__fsqrt_rn(__fsub_rn(sq, cross)), sinphi);
}

// Same formula with the hardware square root (sqrt.approx, <= 1 ulp) and a multiply by 1/sin(phi):
// 3 instructions instead of ~25.  Used by the fused kernel, whose FIR sums already differ from the
// reference by FMA rounding; error ~2e-7 relative, far inside the 1e-5 budget.
__device__ __forceinline__ float envelope2_fast(float prev, float curr, float cosphi2, float inv_sinphi) {
    const float sq = fmaf(prev, prev, curr * curr);
    const float arg = fmaf(-(prev * curr), cosphi2, sq);
    float root;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(root) : "f"(arg));   // one MUFU.SQRT; denormal arguments (|x| < 1e-19) flush to 0
    return root * inv_sinphi;
}

// One output of fast_resampling (dsp.rs:234-263):
//   y[k] = sum over x with 0 <= x*L - k*M <= 2*off, x < len of  h[x*L - k*M] * signal[x]
// accumulated in ascending x like the reference (sum += coeff * sample), one FMA per tap.
template <typename InT>
__device__ __forceinline__ float polyphase_dot(const InT *__restrict__ signal, u64 len,
                                               const float *__restrict__ h, u32 l, u32 m, u64 off2,
                                               u64 k) {
    const u64 t0 = k * m;                    // n at the start of the window (= t - offset)
    u64 x = (t0 + l - 1) / l;                // first input sample inside the window
    u64 xe = (t0 + off2) / l;                // last one (n <= t + offset)
    if (xe >= len) xe = len - 1;             // signal.get(x) == None beyond the end (dsp.rs:257)
    u64 j = x * l - t0;                      // tap index n + offset - t
    float sum = 0.f;
    for (; x <= xe; ++x, j += l) sum = fmaf(__ldg(h + j), load_sample(signal, x), sum);
    return sum;
}

// fast_resampling, optionally fused with demodulate (dsp.rs:350-383): with ENVELOPE the kernel
// writes e[k] = envelope(r[k-1], r[k]), e[0] = 0, and never materialises r.
template <typename InT, bool ENVELOPE>
__global__ void __launch_bounds__(256)
k_polyphase_generic(const InT *__restrict__ signal, u64 len, const float *__restrict__ h, u32 l, u32 m,
                    u64 off2, u64 k_begin, u64 nout, float cosphi2, float sinphi, float *__restrict__ out) {
    // outputs [k_begin, nout); `signal` may be a biased pointer into a chunk buffer, `len` is the whole signal's length
    __shared__ float r[257];
    for (u64 k0 = k_begin + static_cast<u64>(blockIdx.x) * 256; k0 < nout; k0 += static_cast<u64>(gridDim.x) * 256) {
        const u64 k = k0 + threadIdx.x;
        float v = 0.f;
        if (k < nout) v = polyphase_dot(signal, len, h, l, m, off2, k);
        if (!ENVELOPE) {
            if (k < nout) out[k] = v;
            continue;
        }
        r[threadIdx.x + 1] = v;
        if (threadIdx.x == 0) r[0] = k0 > 0 ? polyphase_dot(signal, len, h, l, m, off2, k0 - 1) : 0.f;
        __syncthreads();
        if (k < nout) out[k] = k == 0 ? 0.f : envelope2(r[threadIdx.x], r[threadIdx.x + 1], cosphi2, sinphi);
        __syncthreads();
    }
}

// wav.rs:37 as a kernel: PCM16 -> f32 (`as f32`), 8 samples per thread (16-byte load, two 16-byte stores).
// Feeds the tiled resampler when the caller hands over the WAV's int16 samples (halves the PCIe bytes).
__global__ void __launch_bounds__(256)
k_pcm16_to_f32(const int16_t *__restrict__ in, u64 n, float *__restrict__ out) {
    const u64 n8 = n / 8;
    for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += static_cast<u64>(gridDim.x) * blockDim.x) {
        const int4 v = __ldg(reinterpret_cast<const int4 *>(in) + i);
        float4 a, b;
        a.x = static_cast<float>(static_cast<short>(v.x & 0xffff)); a.y = static_cast<float>(v.x >> 16);
        a.z = static_cast<float>(static_cast<short>(v.y & 0xffff)); a.w = static_cast<float>(v.y >> 16);
        b.x = static_cast<float>(static_cast<short>(v.z & 0xffff)); b.y = static_cast<float>(v.z >> 16);
        b.z = static_cast<float>(static_cast<short>(v.w & 0xffff)); b.w = static_cast<float>(v.w >> 16);
        reinterpret_cast<float4 *>(out)[2 * i] = a;
        reinterpret_cast<float4 *>(out)[2 * i + 1] = b;
    }
    if (blockIdx.x == 0 && threadIdx.x < n - n8 * 8) out[n8 * 8 + threadIdx.x] = static_cast<float>(in[n8 * 8 + threadIdx.x]);
}

// demodulate alone (stage entry point, and the L == 1 decode path): outputs [begin, n), indices absolute.
__global__ void __launch_bounds__(256)
k_envelope(const float *__restrict__ x, u64 begin, u64 n, float cosphi2, float sinphi, float *__restrict__ out) {
    for (u64 i = begin + static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<u64>(gridDim.x) * blockDim.x)
        out[i] = i == 0 ? 0.f : envelope2(__ldg(x + i - 1), __ldg(x + i), cosphi2, sinphi);
}

// dsp::filter (dsp.rs:396-404) followed by decimate (dsp.rs:299-303):
//   out[i] = sum_{j < ntaps, j < i*m} x[i*m - j] * c[j],  begin <= i < nout  (m == 1: plain filter)
// ZERO_FIRST reproduces what NoFilter does to element 0 in the final stage of decode().
template <typename InT>
__global__ void __launch_bounds__(256)
k_fir_decimate_generic(const InT *__restrict__ x, const float *__restrict__ c, u32 ntaps, u32 m, u64 begin, u64 nout,
                       float *__restrict__ out) {
    for (u64 i = begin + static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < nout;
         i += static_cast<u64>(gridDim.x) * blockDim.x) {
        const u64 pos = i * m;
        const u32 jn = pos < ntaps ? static_cast<u32>(pos) : ntaps;   // strict i > j
        float sum = 0.f;
        for (u32 j = 0; j < jn; ++j) sum = fmaf(load_sample(x, pos - j), __ldg(c + j), sum);
        out[i] = sum;
    }
}

// Cross-correlation with the +-1 sync template (decode.rs:225-233), sequential in j like the
// reference: given the same signal the result is bit-identical (adds only).
__global__ void __launch_bounds__(256)
k_corr_generic(const float *__restrict__ f, u64 ncorr, const int8_t *__restrict__ guard, u32 glen,
               float *__restrict__ corr) {
    for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < ncorr;
         i += static_cast<u64>(gridDim.x) * blockDim.x) {
        float acc = 0.f;
        for (u32 j = 0; j < glen; ++j) {
            const float v = __ldg(f + i + j);
            acc = guard[j] > 0 ? __fadd_rn(acc, v) : __fsub_rn(acc, v);
        }
        corr[i] = acc;
    }
}

}  // namespace aptb200
