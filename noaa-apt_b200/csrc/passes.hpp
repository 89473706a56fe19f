// Finding the satellite passes in a long recording (DESIGN.md §12): the recording kept in device memory, the quality of
// each envelope window (kernels_passes.cuh) and the pass rule on the host.
#pragma once

#include <algorithm>
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

// k_pass_quality (kernels_passes.cuh) over windows [w0, w0 + count): e and q are the addresses envelope sample 0 and q[0]
// would have.
int launch_pass_quality(cudaStream_t s, const float *e, uint64_t w0, uint64_t count, uint32_t R, float *q);

// The pass rule fed one window at a time (DESIGN.md §13).  apt_find_passes_quality is "feed every window, then finish",
// so the rule exists once.  A group is the run of windows with q >= exit that starts at `first`; a window joins it while it
// lies at most max_gap windows after the group's last window (`last`).  The group's AOS event fires at the first window
// that joins it once it has reached enter and spans min_length windows; its LOS event fires at the evaluation of window
// last + max_gap (no later window can join), or at finish.  The mean is summed in double in window order, gap windows
// included, so the q of the current gap (fewer than max_gap floats) is held until a later window joins or the group ends.
class PassTracker {
public:
    // Allocates nothing: the gap grows with the windows fed, never past max_gap - 1 floats.
    PassTracker(const PassRule &rule, uint32_t input_rate) : rule_(rule), rate_(input_rate) {}

    // Window next() with quality q.  emit(const apt_pass_event &) receives at most two events: an AOS, then a LOS.
    template <typename Emit>
    void feed(float q, Emit &&emit) {
        const uint64_t w = next_++;
        if (q >= rule_.exit) {
            if (open_) {   // w <= last + max_gap: the group closes at last + max_gap otherwise
                for (float g : gap_) add(g);
                gap_.clear();
            } else {
                open_ = true;
                entered_ = aos_ = false;
                first_ = w;
                sum_ = 0.0;
                peak_ = q;
            }
            last_ = w;
            add(q);
            entered_ = entered_ || q >= rule_.enter;
            if (!aos_ && entered_ && w - first_ + 1 >= rule_.min_length) {
                aos_ = true;
                emit(event(APT_PASS_AOS, w, ~0ull, false));
            }
        } else if (open_) {
            gap_.push_back(q);
        }
        if (open_ && w - last_ == rule_.max_gap) close(w, ~0ull, emit);   // w >= last_: no overflow for any max_gap
    }
    // The end of a recording of n input samples: the open group, if any, closes.  The tracker starts over at window 0.
    template <typename Emit>
    void finish(uint64_t n, Emit &&emit) {
        if (open_) close(next_, n, emit);
        next_ = 0;
    }

    bool open() const { return open_; }
    uint64_t first() const { return first_; }
    uint64_t last() const { return last_; }
    uint64_t next() const { return next_; }
    // Input samples of group [a, b] of a recording of n samples (apt_find_passes_quality's ranges).
    uint64_t start_of(uint64_t a) const { return a * rate_ / 2; }
    uint64_t end_of(uint64_t b, uint64_t n) const { return std::min<uint64_t>(n, ((b + 2) * rate_ + 1) / 2); }

private:
    void add(float q) {
        sum_ += static_cast<double>(q);
        peak_ = std::max(peak_, q);
    }
    apt_pass_event event(int kind, uint64_t w, uint64_t n, bool closed) const {
        apt_pass_event e{};
        e.kind = kind;
        e.window = w;
        e.pass.start = start_of(first_);
        e.pass.end = closed ? end_of(last_, n) : 0;
        e.pass.first_window = first_;
        e.pass.windows = last_ - first_ + 1;
        e.pass.mean_quality = static_cast<float>(sum_ / static_cast<double>(e.pass.windows));
        e.pass.peak_quality = peak_;
        return e;
    }
    template <typename Emit>
    void close(uint64_t w, uint64_t n, Emit &&emit) {
        if (entered_ && last_ - first_ + 1 >= rule_.min_length) emit(event(APT_PASS_LOS, w, n, true));
        open_ = false;
        gap_.clear();
    }

    PassRule rule_;
    uint64_t rate_;
    uint64_t next_ = 0, first_ = 0, last_ = 0;
    bool open_ = false, entered_ = false, aos_ = false;
    double sum_ = 0.0;
    float peak_ = 0.f;
    std::vector<float> gap_;
};

// One chunk of apt_recording_quality: the first stage's units [u0, u1) written to the envelope buffer from work sample e0
// on (e0 a multiple of 4, so the buffer keeps 16-byte alignment), then the windows [w0, w1), whose two rows lie inside.
struct PassChunk {
    uint64_t u0, u1, e0, w0, w1;
};

}  // namespace aptb200

struct apt_pass_tracker {
    aptb200::PassTracker t;
};

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
