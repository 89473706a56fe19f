// The image stage (DESIGN.md §3.5): contrast bounds, telemetry, the u8 map, histogram equalisation, false colour and
// rotation of rows of 2080 pixels.  This module alone reads apt_process_settings: it validates them, decides which
// kernels and buffers a job needs, launches the kernel sequence and turns the device's result into a status and an
// apt_image_info.  Image mode is process mode with the settings of image_settings().
#pragma once

#include <cstdint>

#include "aptb200.h"
#include "launch.hpp"

namespace aptb200 {

struct PostPlan {
    apt_process_settings s{};      // palette NULL: the packed copy is PostBuffers::palette
    bool palette = false;          // false colour
    bool hist = false;             // Contrast::Histogram: MinMax bounds, k_post_map_u8_hist and k_post_eq_lut
    bool finish = false;           // k_post_finish follows the map (histogram, rotation, RGBA or palette): the map writes
                                   // the grey plane; otherwise it writes the output
    int bpp = 1;                   // output bytes per pixel: 4 RGBA, 1 grey (also the channels of a PNG of the image)
};

// The argument rules (host only, APT_ERR_BAD_ARG) and the plan.
int make_post(const apt_process_settings &ps, PostPlan &plan);

// Image mode (apt_decoder_set_image_mode, apt_decode_image_u8 and the stage entry points): contrast bounds and the u8 map.
inline apt_process_settings image_settings(int contrast, float percent) {
    return apt_process_settings{contrast, percent, 0, nullptr, {0.f, 0.f, 0.f, 0.f}, 0};
}

// Device buffers of the stage for images of up to max_rows rows.
struct PostBuffers {
    PostCtl *ctl = nullptr;
    PostCtl *head = nullptr;       // pinned copy of ctl up to `buckets`, written by every post_launch that computes bounds
    float *tel = nullptr;          // 3 * max_rows floats: telemetry band means and variance per row
    ProcCtl *proc = nullptr;       // histogram plans
    unsigned char *grey = nullptr; // max_rows * 2080 B, plans with a finishing pass
    u32 *palette = nullptr;        // 256*256 packed RGBA (upload_palette)

    PostBuffers() = default;
    PostBuffers(const PostBuffers &) = delete;
    ~PostBuffers() { release(); }
    int alloc(const PostPlan &p, u32 max_rows);   // what the plan needs and is not there yet (max_rows stays the same)
    // A 256*256*3 RGB palette, packed and uploaded; returns when the copy is done.
    int upload_palette(const uint8_t *rgb, cudaStream_t stream);
    void release();
};

// Enqueues the stage on rows of px pixels (device), counted by `result` (sync decode) or fixed_rows; b was allocated for
// max_rows.  bounds_dev != nullptr: map with the two floats there (no statistics, no head); out == nullptr: statistics
// and bounds only; px other than 2080: a signal that is not rows, for plans without histogram or finishing pass.  The head
// of the control block reaches b.head once the stream gets there.  hook (or nullptr) brackets each kernel with a slot.
int post_launch(const LaunchCtx &c, const PostPlan &p, PostBuffers &b, const float *rows, const SyncResult *result,
                u32 fixed_rows, u32 max_rows, u32 px, const float *bounds_dev, void *out, KernelHook *hook);

// The status of a finished stage (the reference's error for each device status) and the fill of *info (may be nullptr).
int post_result(const PostCtl &head, apt_image_info *info);

// wav.rs:71-85: normalise by the maximum and quantise to i16 (x, out: device; ctl: scratch control block).
int launch_quantize_i16(const LaunchCtx &c, const float *x, u64 n, PostCtl *ctl, short *out);

}  // namespace aptb200
