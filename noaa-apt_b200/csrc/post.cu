// Image stage: settings, buffers, launch sequence and result (post.hpp).
#include "post.hpp"

#include <algorithm>
#include <cstddef>
#include <cstring>
#include <vector>

#include "common.hpp"
#include "kernels_post.cuh"

namespace aptb200 {

int make_post(const apt_process_settings &ps, PostPlan &plan) {
    if (ps.contrast < 0 || ps.contrast > APT_CONTRAST_HISTOGRAM) return fail(APT_ERR_BAD_ARG, "unknown contrast mode %d", ps.contrast);
    if (ps.contrast == APT_CONTRAST_PERCENT && !(ps.percent >= 0.f && ps.percent <= 1.f))
        return fail(APT_ERR_BAD_ARG, "Percent given should be between 0 and 1");      // misc.rs:120-124
    if (ps.palette && !ps.rgba) return fail(APT_ERR_BAD_ARG, "false colour needs RGBA output");
    if (ps.palette && ps.contrast == APT_CONTRAST_HISTOGRAM)
        return fail(APT_ERR_BAD_ARG, "colour histogram equalisation is not available");
    plan = PostPlan{};
    plan.s = ps;
    plan.s.palette = nullptr;
    plan.palette = ps.palette != nullptr;
    plan.hist = ps.contrast == APT_CONTRAST_HISTOGRAM;
    plan.finish = plan.hist || ps.rotate || ps.rgba || plan.palette;
    plan.bpp = ps.rgba ? 4 : 1;
    return APT_OK;
}

int PostBuffers::alloc(const PostPlan &p, u32 max_rows) {
    const size_t rows = std::max<u32>(max_rows, 1);
    if (!ctl) {
        APT_CUDA(cudaMalloc(&ctl, sizeof(PostCtl)));
        APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&head), sizeof(PostCtl), cudaHostAllocDefault));
        APT_CUDA(cudaMalloc(&tel, 3 * rows * sizeof(float)));
    }
    if (p.hist && !proc) APT_CUDA(cudaMalloc(&proc, sizeof(ProcCtl)));
    if (p.finish && !grey) APT_CUDA(cudaMalloc(&grey, rows * kProcRowPx));
    return APT_OK;
}

int PostBuffers::upload_palette(const uint8_t *rgb, cudaStream_t stream) {
    // 256*256*3 RGB -> 256*256 u32 with R in the low byte and alpha 255 (Rgb::to_rgba), one 4-byte load per coloured pixel
    std::vector<u32> packed(256 * 256);
    for (size_t i = 0; i < packed.size(); ++i)
        packed[i] = static_cast<u32>(rgb[3 * i]) | (static_cast<u32>(rgb[3 * i + 1]) << 8) | (static_cast<u32>(rgb[3 * i + 2]) << 16) |
                    0xFF000000u;
    if (!palette) APT_CUDA(cudaMalloc(&palette, packed.size() * sizeof(u32)));
    APT_CUDA(cudaMemcpyAsync(palette, packed.data(), packed.size() * sizeof(u32), cudaMemcpyHostToDevice, stream));
    APT_CUDA(cudaStreamSynchronize(stream));
    return APT_OK;
}

void PostBuffers::release() {
    for (void *q : {(void *)ctl, (void *)tel, (void *)proc, (void *)grey, (void *)palette})
        if (q) cudaFree(q);
    if (head) cudaFreeHost(head);
    ctl = head = nullptr;
    tel = nullptr;
    proc = nullptr;
    grey = nullptr;
    palette = nullptr;
}

int post_launch(const LaunchCtx &c, const PostPlan &p, PostBuffers &b, const float *rows, const SyncResult *result,
                u32 fixed_rows, u32 max_rows, u32 px, const float *bounds_dev, void *out, KernelHook *hook) {
    if (max_rows == 0) return APT_OK;
    if ((p.hist || p.finish) && px != kProcRowPx) return fail(APT_ERR_BAD_ARG, "image stage: rows of %u pixels", px);
    // the vectorised kernels: k_post_map_u8_hist reads float4 rows, k_post_finish writes 4 or 16 bytes per thread
    if ((p.hist && (reinterpret_cast<uintptr_t>(rows) & 15)) || (p.finish && (reinterpret_cast<uintptr_t>(out) & 15)))
        return fail(APT_ERR_BAD_ARG, "image stage: buffers must be 16-byte aligned");
    const unsigned wide = static_cast<unsigned>(c.sm_count) * 8;
    float *tel_a = b.tel, *tel_b = b.tel + max_rows, *tel_v = b.tel + 2 * static_cast<size_t>(max_rows);
    if (!bounds_dev) {
        // k_post_stats names the min / max pixels by u32 index: the decoder's rows stay below 2^32 work-rate samples, a
        // stream's or watch's max_rows below 2^32 / 2080, apt_process and apt_quantize_i16 refuse larger inputs
        if (static_cast<u64>(max_rows) * px >= (1ull << 32))
            return fail(APT_ERR_BAD_ARG, "image stage: %u rows of %u pixels reach 2^32 pixels", max_rows, px);
        const int bounds_mode = p.hist ? APT_CONTRAST_MINMAX : p.s.contrast;   // Contrast::Histogram takes the MinMax bounds,
                                                                                // noaa_apt.rs:158-163
        APT_CUDA(cudaMemsetAsync(b.ctl, 0, sizeof(PostCtl), c.stream));
        if (p.hist) APT_CUDA(cudaMemsetAsync(b.proc->hist, 0, sizeof(b.proc->hist), c.stream));
        {
            KernelSlot s(hook, "post_stats");
            k_post_stats<<<std::min<unsigned>(max_rows, wide), 256, 0, c.stream>>>(rows, result, fixed_rows, px, b.ctl, tel_a, tel_b,
                                                                                   tel_v);
        }
        if (bounds_mode == APT_CONTRAST_PERCENT) {
            KernelSlot s(hook, "post_histogram");
            k_post_histogram<<<wide / 2, 256, 0, c.stream>>>(rows, result, fixed_rows, px, b.ctl);
        }
        {
            KernelSlot s(hook, "post_bounds");
            k_post_bounds<<<1, 1024, 0, c.stream>>>(bounds_mode, p.s.percent, rows, result, fixed_rows, px, b.ctl, tel_a, tel_b,
                                                   tel_v);
        }
    }
    if (out) {
        // the grey image is the output when nothing follows the map
        unsigned char *grey = p.finish ? b.grey : static_cast<unsigned char *>(out);
        if (p.hist) {
            {
                // two CTAs per SM: every CTA adds its 512 counts to the same 512 global words at the end
                KernelSlot s(hook, "post_map_u8_hist");
                k_post_map_u8_hist<<<static_cast<unsigned>(c.sm_count) * 2, 256, 0, c.stream>>>(rows, result, fixed_rows, b.ctl, grey,
                                                                                                  b.proc);
            }
            KernelSlot s(hook, "post_eq_lut");
            k_post_eq_lut<<<1, 512, 0, c.stream>>>(b.proc);
        } else {
            KernelSlot s(hook, "post_map_u8");
            k_post_map_u8<<<wide, 256, 0, c.stream>>>(rows, result, fixed_rows, px, b.ctl, bounds_dev, grey);
        }
        if (p.finish) {
            KernelSlot s(hook, "post_finish");
            const int mode = p.palette ? 2 : (p.hist ? 1 : 0);
            const float4 tune = make_float4(p.s.tune[0], p.s.tune[1], p.s.tune[2], p.s.tune[3]);
            if (p.s.rgba)
                k_post_finish<true><<<wide, 256, 0, c.stream>>>(grey, b.ctl, b.proc, mode, p.s.rotate ? 1 : 0,
                                                                p.palette ? b.palette : nullptr, tune, out);
            else k_post_finish<false><<<wide, 256, 0, c.stream>>>(grey, b.ctl, b.proc, mode, p.s.rotate ? 1 : 0, nullptr, tune, out);
        }
    }
    APT_CUDA(cudaGetLastError());
    if (!bounds_dev) APT_CUDA(cudaMemcpyAsync(b.head, b.ctl, offsetof(PostCtl, buckets), cudaMemcpyDeviceToHost, c.stream));
    return APT_OK;
}

int post_result(const PostCtl &h, apt_image_info *info) {
    if (info) {
        info->low = h.low;
        info->high = h.high;
        info->rows = h.rows;
        info->telemetry_row = h.telemetry_row;
        memcpy(info->wedges_a, h.wedges_a, sizeof(info->wedges_a));
        memcpy(info->wedges_b, h.wedges_b, sizeof(info->wedges_b));
    }
    switch (h.status) {
    case 0: return APT_OK;
    case 3: return fail(APT_ERR_TOO_SHORT, "Recording too short for telemetry decoding");
    default:
        return fail(APT_ERR_BAD_ARG, "image stage: %s", h.status == 1 ? "empty image" : h.status == 2 ? "no contrast bucket found"
                                                                                                    : "telemetry frame runs off the image");
    }
}

int launch_quantize_i16(const LaunchCtx &c, const float *x, u64 n, PostCtl *ctl, short *out) {
    if (n == 0) return APT_OK;
    if (n >= (1ull << 32)) return fail(APT_ERR_BAD_ARG, "signal too long");
    APT_CUDA(cudaMemsetAsync(ctl, 0, sizeof(PostCtl), c.stream));
    const unsigned wide = static_cast<unsigned>(c.sm_count) * 8;
    // the signal as one "row" of n pixels: only the maximum is used
    k_post_stats<<<1, 256, 0, c.stream>>>(x, nullptr, 1, static_cast<u32>(n), ctl, nullptr, nullptr, nullptr);
    k_quantize_i16<<<wide, 256, 0, c.stream>>>(x, n, ctl, out);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

}  // namespace aptb200
