// Pass search (DESIGN.md §12): the quality of each envelope window, the Pearson correlation of image row w with row w + 1.
#pragma once

#include <cstdint>

namespace aptb200 {

constexpr int kPassQualityThreads = 256;

// q[w] for windows [w0, w1): one CTA per window, rows a = e[wR ..), b = e[(w+1)R ..) of R samples each.  `e` is the
// address envelope sample 0 would have (only the two rows of each window are read).
//
// Precision: each thread accumulates, in f64, the sums of (a - a0), (b - b0), their squares and their product, where a0
// and b0 are the first samples of the two rows.  Shifting by a0 / b0 is exact (f32 differences are exact in f64) and
// removes the row means' size from the sums, so the one-pass combination S_ab - S_a S_b / R loses no precision to
// cancellation even where the envelope's mean is large next to its spread; a constant row gives S_aa = 0 exactly.
// Determinism: the per-thread order is fixed (stride kPassQualityThreads) and the block reduction is a fixed shuffle tree
// followed by a fixed-order sum over warps, so q[w] depends only on the 2R samples of its window: the same bits on every
// run and for every split of the envelope into chunks.
// q[w] = 0 when the denominator is 0 or not finite (silence), a centred sum of squares that rounding left at or below 0
// included.
__global__ void __launch_bounds__(kPassQualityThreads)
k_pass_quality(const float *__restrict__ e, uint64_t w0, uint32_t R, float *__restrict__ q) {
    const uint64_t w = w0 + blockIdx.x;
    const float *a = e + w * R;
    const float *b = a + R;
    const double a0 = static_cast<double>(__ldg(a)), b0 = static_cast<double>(__ldg(b));
    double sa = 0.0, sb = 0.0, saa = 0.0, sbb = 0.0, sab = 0.0;
    for (uint32_t i = threadIdx.x; i < R; i += kPassQualityThreads) {
        const double x = static_cast<double>(__ldg(a + i)) - a0;
        const double y = static_cast<double>(__ldg(b + i)) - b0;
        sa += x;
        sb += y;
        saa = fma(x, x, saa);
        sbb = fma(y, y, sbb);
        sab = fma(x, y, sab);
    }
    for (int off = 16; off > 0; off >>= 1) {
        sa += __shfl_down_sync(0xffffffffu, sa, off);
        sb += __shfl_down_sync(0xffffffffu, sb, off);
        saa += __shfl_down_sync(0xffffffffu, saa, off);
        sbb += __shfl_down_sync(0xffffffffu, sbb, off);
        sab += __shfl_down_sync(0xffffffffu, sab, off);
    }
    constexpr int kWarps = kPassQualityThreads / 32;
    __shared__ double part[5][kWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        part[0][warp] = sa;
        part[1][warp] = sb;
        part[2][warp] = saa;
        part[3][warp] = sbb;
        part[4][warp] = sab;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    double s[5];
    for (int k = 0; k < 5; ++k) {
        s[k] = part[k][0];
        for (int j = 1; j < kWarps; ++j) s[k] += part[k][j];
    }
    const double r = static_cast<double>(R);
    const double caa = s[2] - s[0] * s[0] / r;
    const double cbb = s[3] - s[1] * s[1] / r;
    const double cab = s[4] - s[0] * s[1] / r;
    const double den = sqrt(caa * cbb);
    q[w] = caa > 0.0 && cbb > 0.0 && isfinite(den) ? static_cast<float>(cab / den) : 0.f;
}

}  // namespace aptb200
