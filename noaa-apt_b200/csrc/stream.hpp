// What the streaming decoder (stream.cu) shares with the watcher (watch.cu): the f32 input window, its compaction and the
// streamed first stage, and a push of samples that are already on the device.
#pragma once

#include <cstdint>

#include <cuda_runtime.h>

#include "aptb200.h"
#include "decoder.hpp"
#include "front.hpp"
#include "launch.hpp"
#include "png.hpp"

namespace aptb200 {

// Moves the tail [keep, end) of a window based at `base` to its front when that does not overlap (keep is floored to a
// multiple of 16, so the window keeps its alignment).
int window_compact(cudaStream_t s, float *buf, uint64_t &base, uint64_t keep, uint64_t end);
// n samples into the f32 window at dst: f32 from the host or, with on_device, from the device; PCM16 from the host through
// d_pcm (uploaded) and d_conv (cast), so that pushes may mix formats.
int window_upload(const LaunchCtx &c, const void *src, bool on_device, int format, uint64_t n, int16_t *d_pcm, float *d_conv,
                  float *dst);
// The first stage over the units whose input is complete after N samples (all of them at finish): `in` is the address input
// sample 0 would have, d_e (and d_r, the decimating kind's scratch) hold the envelope from work sample e_base on.
int front_advance(const LaunchCtx &c, const Plan &p, const FrontTables &t, const float *in, uint64_t N, bool finish,
                  uint64_t cap_e, float *d_r, float *d_e, uint64_t e_base, uint64_t &units_done, uint64_t &work_final);

// apt_stream_push of n f32 samples at d_src on the device (a copy on the stream's CUDA stream, no H2D).
int stream_push_device(apt_stream *st, const float *d_src, uint64_t n, float *rows, uint64_t cap, uint64_t *nout);
cudaStream_t stream_cuda(const apt_stream *st);
uint64_t stream_rows_out(const apt_stream *st);
// Device bytes apt_stream_set_process_mode (and apt_stream_set_png_mode, plan.png) allocate for max_rows rows: the pass's
// rows and the ImageOut.
uint64_t stream_image_bytes(const OutPlan &plan, uint64_t max_rows);

}  // namespace aptb200
