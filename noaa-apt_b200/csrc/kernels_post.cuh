// After the hot path, still on the device: contrast bounds, telemetry statistics and the u8 image (SURVEY.md §8 f3), so
// that the decoded rows leave the GPU 4x smaller.  Restates, operation by operation (every f32 op rounded on its own,
// no FMA contraction, the reference's summation order):
//   dsp::get_min / get_max                      dsp.rs:20-54
//   misc::percent (1000-bucket histogram)       misc.rs:119-175
//   telemetry::read_telemetry / from_bands      telemetry.rs:125-243, :30-66
//   noaa_apt::map_signal_u8                     noaa_apt.rs:249-259
//   grey histogram equalisation                 processing.rs:87-103, imageext.rs:23-46, :95-119
//   processing::false_color                     processing.rs:108-157
//   processing::rotate (Rotate::Yes)            processing.rs:21-37
// Given the same f32 rows these kernels reproduce the reference's u8 / RGBA image and contrast bounds bit for bit,
// non-finite pixels and signed zeros included.  Min / max follow dsp::get_min / get_max, a walk from pixel 0 with strict
// `<` / `>`: if pixel 0 is NaN both are pixel 0; otherwise the minimum is the pixel of lowest index among the non-NaN
// pixels that compare == to the smallest value (-0.0 == +0.0), with its own bits, and the maximum likewise.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "launch.hpp"

namespace aptb200 {

// telemetry.rs:129-133: contrast wedges 1-9, seven variable wedges, contrast wedges of the next frame
__device__ const float kTelemetryPattern[25] = {31.f, 63.f, 95.f, 127.f, 159.f, 191.f, 224.f, 255.f, 0.f,
                                                0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f,
                                                31.f, 63.f, 95.f, 127.f, 159.f, 191.f, 224.f, 255.f, 0.f};

// monotone map float -> u32 of the non-NaN floats, -0.0 folded onto +0.0 so that the two zeros tie
__device__ __forceinline__ u32 float_key(float v) {
    const u32 b = __float_as_uint(v == 0.f ? 0.f : v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ u32 post_rows(const PostCtl *ctl, const SyncResult *result, u32 fixed_rows) {
    (void)ctl;
    return result ? (result->status == 0 ? result->n_rows : 0u) : fixed_rows;
}

// (min, max) of the n pixels from what k_post_stats left in ctl: pixel 0 when it is NaN, else the winning pixels' values
__device__ __forceinline__ float2 post_minmax(const float *rows, u64 n, const PostCtl *ctl) {
    if (n == 0) return make_float2(0.f, 0.f);
    const float x0 = rows[0];
    if (x0 != x0) return make_float2(x0, x0);
    return make_float2(rows[static_cast<u32>(~ctl->nmin_at)], rows[~static_cast<u32>(ctl->max_at)]);
}

// min / max of the image as the pixel index that wins them (first wins among ties: the thread's pixels come in
// ascending index, the cross-thread reduction takes the lower index on equal keys; NaN pixels take no part) and, per
// row, the telemetry band means and their pooled variance in the reference's sequential order (telemetry.rs:147-170):
// bands at pixels 994..1037 and 2034..2077.  Pixel indices fit in u32 (post_launch checks).
__global__ void __launch_bounds__(256)
k_post_stats(const float *__restrict__ rows, const SyncResult *__restrict__ result, u32 fixed_rows, u32 px, PostCtl *__restrict__ ctl,
             float *__restrict__ mean_a, float *__restrict__ mean_b, float *__restrict__ variance) {
    __shared__ u64 s_min[8], s_max[8];
    const u32 n_rows = post_rows(ctl, result, fixed_rows);
    u32 kmin = 0xFFFFFFFFu, imin = 0xFFFFFFFFu, kmax = 0u, imax = 0xFFFFFFFFu;   // no key of a non-NaN float is 0 or ~0
    for (u32 r = blockIdx.x; r < n_rows; r += gridDim.x) {
        const float *line = rows + static_cast<u64>(r) * px;
        for (u32 c = threadIdx.x; c < px; c += blockDim.x) {
            const float v = line[c];
            if (v != v) continue;
            const u32 k = float_key(v);
            if (k < kmin) { kmin = k; imin = r * px + c; }
            if (k > kmax) { kmax = k; imax = r * px + c; }
        }
        if (threadIdx.x < 2 && px >= 2078 && mean_a != nullptr) {
            const float *band = line + (threadIdx.x == 0 ? 994 : 2034);
            float sum = 0.f;
            for (int i = 0; i < 44; ++i) sum = __fadd_rn(sum, band[i]);
            const float mean = __fdiv_rn(sum, 44.f);
            float var = 0.f;
            for (int i = 0; i < 44; ++i) {
                const float d = __fsub_rn(band[i], mean);
                var = __fadd_rn(var, __fmul_rn(d, d));
            }
            (threadIdx.x == 0 ? mean_a : mean_b)[r] = mean;
            const float other = __shfl_xor_sync(0x3u, var, 1);
            if (threadIdx.x == 0) variance[r] = __fdiv_rn(__fadd_rn(var, other), 88.f);
        }
    }
    // key << 32 | index ordered by min, key << 32 | ~index by max: equal keys go to the lower index either way
    u64 cmin = (static_cast<u64>(kmin) << 32) | imin, cmax = (static_cast<u64>(kmax) << 32) | ~imax;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        cmin = min(cmin, __shfl_xor_sync(0xffffffffu, cmin, o));
        cmax = max(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
    }
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = cmin; s_max[threadIdx.x >> 5] = cmax; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) { cmin = min(cmin, s_min[w]); cmax = max(cmax, s_max[w]); }
        atomicMax(&ctl->nmin_at, ~cmin);                           // zero-initialised control block: keep ~min as a maximum
        atomicMax(&ctl->max_at, cmax);
    }
}

// misc.rs:139-154: bucket = trunc((x - min) / total_range * 1000) clamped to [0, 999]
__global__ void __launch_bounds__(256)
k_post_histogram(const float *__restrict__ rows, const SyncResult *__restrict__ result, u32 fixed_rows, u32 px, PostCtl *__restrict__ ctl) {
    __shared__ u32 s_b[1000];
    for (u32 i = threadIdx.x; i < 1000; i += blockDim.x) s_b[i] = 0;
    __syncthreads();
    const u64 n = static_cast<u64>(post_rows(ctl, result, fixed_rows)) * px;
    const float2 m = post_minmax(rows, n, ctl);
    const float mn = m.x, mx = m.y;
    const float range = __fsub_rn(mx, mn);
    for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x) {
        const float t = truncf(__fmul_rn(__fdiv_rn(__fsub_rn(rows[i], mn), range), 1000.f));
        const u32 b = !(t >= 0.f) ? 0u : (t >= 999.f ? 999u : static_cast<u32>(t));   // `as usize` saturates, NaN -> 0
        atomicAdd(&s_b[b], 1u);
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < 1000; i += blockDim.x)
        if (s_b[i]) atomicAdd(&ctl->buckets[i], s_b[i]);
}

// One CTA: the contrast bounds (low, high) from what the two kernels above left in ctl.
//   mode 0  MinMax     noaa_apt.rs:157-163
//   mode 1  Percent    misc.rs:156-174 (the scan over the buckets, `else if` included)
//   mode 2  Telemetry  telemetry.rs:172-228 frame search (first-wins strict maximum of the quality), :30-66 wedge values,
//                      low = wedge 9, high = wedge 8 averaged over both channels (noaa_apt.rs:143-149)
__global__ void __launch_bounds__(1024)
k_post_bounds(int mode, float percent, const float *__restrict__ rows, const SyncResult *__restrict__ result, u32 fixed_rows, u32 px,
              PostCtl *__restrict__ ctl, const float *__restrict__ mean_a, const float *__restrict__ mean_b,
              const float *__restrict__ variance) {
    __shared__ u32 s_scan[1024];
    __shared__ float s_q[1024];
    __shared__ u32 s_i[1024];
    const u32 tid = threadIdx.x;
    const u32 n_rows = post_rows(ctl, result, fixed_rows);
    const float2 m = post_minmax(rows, static_cast<u64>(n_rows) * px, ctl);
    const float mn = m.x, mx = m.y;
    if (tid == 0) {
        ctl->rows = n_rows;
        ctl->low = mn;
        ctl->high = mx;
        ctl->status = n_rows == 0 ? 1u : 0u;
    }
    if (n_rows == 0) return;
    if (mode == 1) {
        // inclusive prefix sums of the 1000 bucket counts (u32 like the reference's accum)
        s_scan[tid] = tid < 1000 ? ctl->buckets[tid] : 0u;
        __syncthreads();
        for (u32 o = 1; o < 1024; o <<= 1) {
            const u32 v = tid >= o ? s_scan[tid - o] : 0u;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        const float total = static_cast<float>(static_cast<u64>(n_rows) * px);     // signal.len() as f32
        const float remainder = __fdiv_rn(__fsub_rn(1.f, percent), 2.f);
        const float frac = __fdiv_rn(static_cast<float>(s_scan[tid]), total);
        const bool over_low = tid < 1000 && frac > remainder;
        const bool over_high = tid < 1000 && frac > __fsub_rn(1.f, remainder);
        // low = first bucket over the remainder; high = first bucket over 1 - remainder that is not the iteration that set low
        s_i[tid] = over_low ? tid : 0xFFFFFFFFu;
        __syncthreads();
        for (u32 o = 512; o > 0; o >>= 1) {
            if (tid < o) s_i[tid] = min(s_i[tid], s_i[tid + o]);
            __syncthreads();
        }
        const u32 low_b = s_i[0];
        __syncthreads();
        s_i[tid] = (over_high && tid != low_b) ? tid : 0xFFFFFFFFu;
        __syncthreads();
        for (u32 o = 512; o > 0; o >>= 1) {
            if (tid < o) s_i[tid] = min(s_i[tid], s_i[tid + o]);
            __syncthreads();
        }
        if (tid == 0) {
            u32 high_b = s_i[0];
            if (high_b == 0xFFFFFFFFu) high_b = 999;
            const float range = __fsub_rn(mx, mn);
            if (low_b == 0xFFFFFFFFu) {
                ctl->status = 2u;                                   // low_bucket.unwrap() panics in the reference
            } else {
                ctl->low = __fadd_rn(__fmul_rn(__fdiv_rn(static_cast<float>(low_b), 1000.f), range), mn);
                ctl->high = __fadd_rn(__fmul_rn(__fdiv_rn(static_cast<float>(high_b), 1000.f), range), mn);
            }
        }
        return;
    }
    if (mode != 2) return;
    // ---- telemetry frame search ----
    if (n_rows < 200) {                                             // "Recording too short for telemetry decoding"
        if (tid == 0) ctl->status = 3u;
        return;
    }
    float best_q = 0.f;
    u32 best_i = 0;
    for (u32 i = tid; i + 200 < n_rows; i += blockDim.x) {
        float sum = 0.f, dev = 0.f;
        for (int j = 0; j < 200; ++j) {
            const float smp = kTelemetryPattern[j >> 3];             // each wedge value repeated 8 times (telemetry.rs:129-136)
            sum = __fadd_rn(sum, __fmul_rn(smp, mean_a[i + j]));
            sum = __fadd_rn(sum, __fmul_rn(smp, mean_b[i + j]));
        }
        for (int j = 0; j < 200; ++j) dev = __fadd_rn(dev, __fsqrt_rn(variance[i + j]));
        const float q = __fdiv_rn(sum, dev);
        if (q > best_q) { best_q = q; best_i = i; }                 // ascending i within the thread: first wins
    }
    s_q[tid] = best_q;
    s_i[tid] = best_i;
    __syncthreads();
    for (u32 o = 512; o > 0; o >>= 1) {
        if (tid < o) {
            const float q2 = s_q[tid + o];
            const u32 i2 = s_i[tid + o];
            if (q2 > s_q[tid] || (q2 == s_q[tid] && q2 > 0.f && i2 < s_i[tid])) { s_q[tid] = q2; s_i[tid] = i2; }
        }
        __syncthreads();
    }
    const u32 best = s_q[0] > 0.f ? s_i[0] : 0u;                    // best = (0, 0.) unless some quality exceeds 0
    // from_bands: means of 8 contiguous rows from `best`, 16 + 9 wedges
    __shared__ float s_w[2][25];
    if (tid < 50) {
        const u32 w = tid % 25;
        const float *m = tid < 25 ? mean_a : mean_b;
        float v = 0.f;
        if (best + 8u * (w + 1) <= n_rows) {
            for (int k = 0; k < 8; ++k) v = __fadd_rn(v, m[best + 8 * w + k]);
            v = __fdiv_rn(v, 8.f);
        } else if (tid == 0) {
            ctl->status = 4u;                                       // not enough rows after the frame start (index panic)
        }
        s_w[tid / 25][w] = v;
    }
    __syncthreads();
    if (tid < 32) {
        const u32 ch = tid / 16, w = tid % 16;                      // wedge w + 1
        const float v = w < 9 ? __fdiv_rn(__fadd_rn(s_w[ch][w], s_w[ch][w + 16]), 2.f) : s_w[ch][w];
        (ch == 0 ? ctl->wedges_a : ctl->wedges_b)[w] = v;
    }
    __syncthreads();
    if (tid == 0) {
        ctl->telemetry_row = best;
        if (best + 200 > n_rows) ctl->status = 4u;
        ctl->low = __fdiv_rn(__fadd_rn(ctl->wedges_a[8], ctl->wedges_b[8]), 2.f);    // wedge 9
        ctl->high = __fdiv_rn(__fadd_rn(ctl->wedges_a[7], ctl->wedges_b[7]), 2.f);   // wedge 8
    }
}

// noaa_apt.rs:249-259: ((x - low) / range * 255).max(0).min(255).round() as u8
__device__ __forceinline__ unsigned char map_u8(float x, float low, float range) {
    float v = __fmul_rn(__fdiv_rn(__fsub_rn(x, low), range), 255.f);
    v = fminf(fmaxf(v, 0.f), 255.f);                                // f32::max / min return the non-NaN operand
    return static_cast<unsigned char>(roundf(v));                   // round half away from zero, like f32::round
}

__global__ void __launch_bounds__(256)
k_post_map_u8(const float *__restrict__ rows, const SyncResult *__restrict__ result, u32 fixed_rows, u32 px,
              const PostCtl *__restrict__ ctl, const float *bounds /* nullptr: ctl's */, unsigned char *__restrict__ out) {
    const u64 n = static_cast<u64>(post_rows(ctl, result, fixed_rows)) * px;
    const float low = bounds ? bounds[0] : ctl->low, high = bounds ? bounds[1] : ctl->high;
    const float range = __fsub_rn(high, low);
    const u64 n4 = n / 4;
    const bool vec = ((reinterpret_cast<uintptr_t>(rows) & 15) | (reinterpret_cast<uintptr_t>(out) & 3)) == 0;
    if (vec) {
        for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<u64>(gridDim.x) * blockDim.x) {
            const float4 v = reinterpret_cast<const float4 *>(rows)[i];
            uchar4 o;
            o.x = map_u8(v.x, low, range); o.y = map_u8(v.y, low, range); o.z = map_u8(v.z, low, range); o.w = map_u8(v.w, low, range);
            reinterpret_cast<uchar4 *>(out)[i] = o;
        }
        for (u64 i = n4 * 4 + static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x)
            out[i] = map_u8(rows[i], low, range);
    } else {
        for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x)
            out[i] = map_u8(rows[i], low, range);
    }
}

// ------------------------------------------------ the rest of noaa_apt::process (noaa_apt.rs:140-240), map overlay excepted
// Column layout, decode.rs:16-35: channel A is x in [0, 1040), B is x in [1040, 2080); the image data of a channel is its
// columns [86, 995) (sync 39 px + space 47 px in front, telemetry 45 px behind).
constexpr u32 kProcRowPx = 2080, kProcChannelPx = 1040, kProcImageX0 = 86, kProcImageEnd = 995;

// map_signal_u8 (as k_post_map_u8) and, in the same pass, the grey-value histogram of each channel half for
// Contrast::Histogram (imageext.rs:95-119).  Counts are privatised per warp in shared memory.  APT images have long runs
// of one value (sync bars, the space band, telemetry wedges, pixels clipped at 0 / 255), so lanes holding the same
// (channel, value) are first merged with __match_any_sync: a run costs one shared atomic per warp, not one per lane.
// Rows of 2080 px and 16-byte aligned rows / 4-byte aligned output (the launcher checks): every float4 lies in one channel.
__global__ void __launch_bounds__(256)
k_post_map_u8_hist(const float *__restrict__ rows, const SyncResult *__restrict__ result, u32 fixed_rows,
                   const PostCtl *__restrict__ ctl, unsigned char *__restrict__ out, ProcCtl *__restrict__ proc) {
    __shared__ u32 s_h[8][512];
    for (u32 i = threadIdx.x; i < 8 * 512; i += blockDim.x) (&s_h[0][0])[i] = 0u;
    __syncthreads();
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 *h = s_h[warp];
    const u64 n4 = static_cast<u64>(post_rows(ctl, result, fixed_rows)) * (kProcRowPx / 4);
    const float low = ctl->low, range = __fsub_rn(ctl->high, low);
    const u64 stride = static_cast<u64>(gridDim.x) * blockDim.x;
    // the loop bound is per warp, so that every lane reaches the __match_any_sync calls
    for (u64 base = static_cast<u64>(blockIdx.x) * blockDim.x + (warp << 5); base < n4; base += stride) {
        const u64 i = base + lane;
        u32 key[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
        if (i < n4) {
            const float4 v = reinterpret_cast<const float4 *>(rows)[i];
            uchar4 o;
            o.x = map_u8(v.x, low, range); o.y = map_u8(v.y, low, range); o.z = map_u8(v.z, low, range); o.w = map_u8(v.w, low, range);
            reinterpret_cast<uchar4 *>(out)[i] = o;
            const u32 ch = static_cast<u32>(i % (kProcRowPx / 4)) >= kProcChannelPx / 4 ? 256u : 0u;
            key[0] = ch + o.x; key[1] = ch + o.y; key[2] = ch + o.z; key[3] = ch + o.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const u32 peers = __match_any_sync(0xffffffffu, key[j]);
            if (key[j] != 0xFFFFFFFFu && lane == static_cast<u32>(__ffs(peers) - 1)) atomicAdd(&h[key[j]], static_cast<u32>(__popc(peers)));
        }
    }
    __syncthreads();
    for (u32 b = threadIdx.x; b < 512; b += blockDim.x) {
        u32 s = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += s_h[w][b];
        if (s) atomicAdd(&proc->hist[0][0] + b, s);
    }
}

// imageext.rs:23-46, :95-119 for both channel halves: cumulative u32 histogram, total = hist[255] as f32, and
// v -> (255.0 * (hist[v] as f32 / total)) as u8.  The u32 -> f32 conversions round to nearest (they are inexact above 2^24
// pixels per half, about 16 000 rows); `as u8` truncates and saturates (NaN -> 0).  One CTA, one thread per (channel, value).
__global__ void __launch_bounds__(512)
k_post_eq_lut(ProcCtl *__restrict__ proc) {
    __shared__ u32 s[512];
    const u32 t = threadIdx.x, bin = t & 255u;
    s[t] = (&proc->hist[0][0])[t];
    __syncthreads();
    for (u32 o = 1; o < 256; o <<= 1) {
        const u32 v = bin >= o ? s[t - o] : 0u;
        __syncthreads();
        s[t] += v;
        __syncthreads();
    }
    const float total = __uint2float_rn(s[t | 255u]);
    const float v = __fmul_rn(255.f, __fdiv_rn(__uint2float_rn(s[t]), total));
    (&proc->lut[0][0])[t] = !(v >= 0.f) ? 0 : (v >= 255.f ? 255 : static_cast<unsigned char>(static_cast<u32>(v)));
}

// processing.rs:125-140 tune_input_values for one channel: (in * ((1 + e) - s) - s * 255).clamp(0, 255) as u32 with
// s = start * 0.3, e = end * 0.3, every f32 operation rounded on its own (no FMA).
__device__ __forceinline__ unsigned char tune_value(u32 in, float start, float end) {
    const float s = __fmul_rn(start, 0.3f), e = __fmul_rn(end, 0.3f);
    const float o = __fsub_rn(__fmul_rn(static_cast<float>(in), __fsub_rn(__fadd_rn(1.f, e), s)), __fmul_rn(s, 255.f));
    return !(o >= 0.f) ? 0 : (o >= 255.f ? 255 : static_cast<unsigned char>(static_cast<u32>(o)));   // f32::clamp keeps NaN; `as u32` -> 0
}

// The finishing pass over the grey plane: rotation (processing.rs:21-37, Rotate::Yes) as a gather of source coordinates
// -- (x0 + i, y) <- (x0 + 908 - i, rows - 1 - y) inside the two 909-px image rectangles -- then
//   mode 0  the grey value
//   mode 1  the equalisation table of the pixel's channel half (Contrast::Histogram)
//   mode 2  false colour (processing.rs:108-157): in channel A's image columns palette[val_b][val_a] with the tuned values
//           of a = grey(x, y) and b = grey(x + 1040, y); everywhere else the grey value
// and writes grey (1 B/px, 4-byte stores) or RGBA (R = G = B = grey, A = 255 outside the colour region; 16-byte stores).
// One thread per 4 consecutive output pixels of a row.  Both per-value tables (equalisation, or the two tune maps) sit in
// shared memory; the palette, 256 KB packed as u32, is read through the read-only path (__ldg, L1 / L2).
template <bool RGBA>
__global__ void __launch_bounds__(256)
k_post_finish(const unsigned char *__restrict__ grey, const PostCtl *__restrict__ ctl, const ProcCtl *__restrict__ proc, int mode,
              int rotate, const u32 *__restrict__ palette, float4 tune, void *__restrict__ out) {
    __shared__ unsigned char s_tab[2][256];
    for (u32 i = threadIdx.x; i < 512; i += blockDim.x) {
        const u32 ch = i >> 8, v = i & 255u;
        unsigned char t = static_cast<unsigned char>(v);
        if (mode == 1) t = proc->lut[ch][v];
        else if (mode == 2) t = ch == 0 ? tune_value(v, tune.x, tune.y) : tune_value(v, tune.z, tune.w);
        s_tab[ch][v] = t;
    }
    __syncthreads();
    const u32 rows = ctl->rows;
    const u64 nq = static_cast<u64>(rows) * (kProcRowPx / 4);
    for (u64 q = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; q < nq; q += static_cast<u64>(gridDim.x) * blockDim.x) {
        const u32 y = static_cast<u32>(q / (kProcRowPx / 4));
        const u32 x0 = static_cast<u32>(q % (kProcRowPx / 4)) * 4;
        u32 px[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const u32 x = x0 + k;
            const u32 chb = x >= kProcChannelPx ? 1u : 0u;
            const u32 xc = x - chb * kProcChannelPx;                          // column within the channel
            const bool img = xc >= kProcImageX0 && xc < kProcImageEnd;
            u32 sx = x, sy = y;
            if (rotate && img) {
                sx = x - xc + (kProcImageX0 + kProcImageEnd - 1) - xc;        // x0 + 908 - i
                sy = rows - 1 - y;
            }
            const unsigned char *line = grey + static_cast<u64>(sy) * kProcRowPx;
            const u32 g = line[sx];
            if (RGBA && mode == 2 && img && !chb) {
                const u32 b = line[sx + kProcChannelPx];
                px[k] = __ldg(palette + (static_cast<u32>(s_tab[1][b]) << 8) + s_tab[0][g]);
            } else {
                const u32 v = mode == 1 ? s_tab[chb][g] : g;
                px[k] = RGBA ? (v * 0x010101u) | 0xFF000000u : v;
            }
        }
        if (RGBA) reinterpret_cast<uint4 *>(out)[q] = make_uint4(px[0], px[1], px[2], px[3]);
        else reinterpret_cast<u32 *>(out)[q] = px[0] | (px[1] << 8) | (px[2] << 16) | (px[3] << 24);
    }
}

// wav.rs:71-85 for 16-bit files: (sample / max * 32767.0) as i16 -- `as` truncates toward zero, saturates, NaN -> 0.
// The maximum is dsp::get_max as k_post_stats leaves it in ctl (post_minmax).
__global__ void __launch_bounds__(256)
k_quantize_i16(const float *__restrict__ x, u64 n, const PostCtl *__restrict__ ctl, short *__restrict__ out) {
    const float mx = post_minmax(x, n, ctl).y;
    for (u64 i = static_cast<u64>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<u64>(gridDim.x) * blockDim.x) {
        const float v = __fmul_rn(__fdiv_rn(x[i], mx), 32767.f);
        short q;
        if (v != v) q = 0;
        else if (v >= 32767.f) q = 32767;
        else if (v <= -32768.f) q = -32768;
        else q = static_cast<short>(static_cast<int>(v));           // cvt.rzi
        out[i] = q;
    }
}

}  // namespace aptb200
