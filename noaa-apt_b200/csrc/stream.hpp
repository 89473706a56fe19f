// What the watcher (watch.cu) uses of the streaming decoder (stream.cu) beyond the C ABI: a push of samples that are
// already on the device, the stream's CUDA stream and rows, and the device bytes of its image output.
#pragma once

#include <cstdint>

#include <cuda_runtime.h>

#include "aptb200.h"
#include "png.hpp"

namespace aptb200 {

// apt_stream_push of n f32 samples at d_src on the device (a copy on the stream's CUDA stream, no H2D).
int stream_push_device(apt_stream *st, const float *d_src, uint64_t n, float *rows, uint64_t cap, uint64_t *nout);
cudaStream_t stream_cuda(const apt_stream *st);
uint64_t stream_rows_out(const apt_stream *st);
// Device bytes apt_stream_set_process_mode (and apt_stream_set_png_mode, plan.png) allocate for max_rows rows: the pass's
// rows and the ImageOut.
uint64_t stream_image_bytes(const OutPlan &plan, uint64_t max_rows);

}  // namespace aptb200
