// Finding the satellite passes in a long recording (DESIGN.md §12): the recording kept in device memory, the quality of
// each envelope window (kernels_passes.cuh) and the pass rule on the host.
#pragma once

#include <cstdint>
#include <vector>

#include <cuda_runtime.h>

#include "aptb200.h"
#include "decoder.hpp"

namespace aptb200 {

// apt_pass_search with its defaults filled in and the seconds turned into windows.
struct PassRule {
    float enter = 0.30f, exit = 0.15f;
    uint64_t max_gap = 60, min_length = 120;
};
int make_pass_rule(const apt_pass_search *ps, PassRule &r);

// One chunk of apt_recording_quality: the first stage's units [u0, u1) written to the envelope buffer from work sample e0
// on (e0 a multiple of 4, so the buffer keeps 16-byte alignment), then the windows [w0, w1), whose two rows lie inside.
struct PassChunk {
    uint64_t u0, u1, e0, w0, w1;
};

}  // namespace aptb200

struct apt_recording {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    aptb200::Plan plan;
    int format = APT_F32;
    uint64_t n = 0, nwork = 0, windows = 0;
    uint32_t row = 0;                          // R: work samples per image row
    void *d_sig = nullptr;                     // the n samples, in their own format
    aptb200::FrontTables front;
    std::vector<aptb200::PassChunk> chunks;    // the fixed chunk geometry of apt_recording_quality
    float *d_e = nullptr;                      // envelope of one chunk
    float *d_conv = nullptr;                   // f32 copy of one chunk's PCM16 span (a first stage that wants f32 only)
    float *d_scratch = nullptr;                // resampled signal of the decimating first stage
    float *d_q = nullptr;                      // q, W floats
    uint64_t device_bytes = 0;
};
