// The decoder object behind the C ABI: plan (filters, rates, sizes), device workspaces, one
// stream, and the kernel sequence of decode::decode (decode.rs:43-162).
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "aptb200.h"
#include <memory>

#include "back.hpp"
#include "filters_host.hpp"
#include "front.hpp"
#include "hostpool.hpp"
#include "iq.hpp"
#include "launch.hpp"
#include "png.hpp"
#include "post.hpp"

namespace aptb200 {

// decode.rs:14-38
constexpr uint32_t kFinalRate = 4160;
constexpr uint32_t kPxPerRow = 2080;
constexpr uint32_t kCarrierHz = 2400;

// Everything decode() derives from (input_rate, settings) before touching a sample.
struct Plan {
    uint32_t input_rate = 0;
    apt_settings st{};
    FrontPlan front;               // input_rate -> work_rate with the LowpassDcRemoval filter (decode.rs:65-89)
    std::vector<float> lp;         // demodulation low-pass taps (Lowpass, decode.rs:95-100)
    float cosphi2 = 0.f, sinphi = 1.f;   // dsp.rs:360-363
    uint32_t row = 0;              // samples_per_work_row (decode.rs:55)
    uint32_t dist = 0;             // min_distance (decode.rs:216)
    bool work_multiple = false;    // work_rate % 4160 == 0
    uint32_t dec = 0;              // work_rate / 4160 when work_multiple
    Ratio last{};                  // work_rate -> 4160 for the final NoFilter resample
    std::vector<int8_t> guard;     // sync template (empty unless work_multiple)
};

int make_plan(uint32_t input_rate, const apt_settings &s, Plan &plan);
// decode() output length for no-sync / upper bound for sync.
uint64_t plan_out_bound(const Plan &p, uint64_t n);

// Uploads the plan's filter taps and resampler tables (apt_decoder_create and apt_stream_create); plan_table_bytes is
// the device memory that takes.
int upload_plan(apt_decoder *d);
uint64_t plan_table_bytes(const Plan &p);
// Frees every buffer, event and stream the decoder owns (the object itself stays).
int free_decoder_buffers(apt_decoder *d);
// Grows the f32 copy of a PCM16 input to `alloc` samples when it holds fewer than `need`.
int ensure_conv(apt_decoder *d, uint64_t need, uint64_t alloc);
// The decoders the convenience entry points park between calls (APTB200_NO_CACHE: none are parked).  take_decoder hands
// out a parked decoder for (device, rate, settings) of at least n samples, else creates one of n samples, with head-room
// for a slightly longer next recording when `headroom` and the cache is on.  park_decoder drains the decoder's stream, clears the state of
// the call (image, process and PNG mode, img.keep, the status callback, a borrowed stager) and parks the decoder
// under its own key, or destroys it.  `several`: keep it beside others of its key (a batch's decoders), else it
// replaces a smaller one of the same key.
int take_decoder(int device, uint32_t rate, const apt_settings &st, uint64_t n, bool headroom, apt_decoder **d);
void park_decoder(apt_decoder *d, bool several);

// Kernel accounting of a decoder: counts the launch and, when profiling, records the begin event of slot `name`;
// returns the slot to close with prof_end (-1: none).
int prof_begin(apt_decoder *d, const char *name);
void prof_end(apt_decoder *d, int slot);
struct DecoderHook : KernelHook {
    apt_decoder *d;
    int slot = -1;
    explicit DecoderHook(apt_decoder *dec) : d(dec) {}
    void begin(const char *name) override { slot = prof_begin(d, name); }
    void end() override { prof_end(d, slot); }
    void extra(int kernels) override;
};

}  // namespace aptb200

struct apt_decoder {
    int device = 0;
    int sm_count = 0;              // of `device`, set by apt_decoder_create
    cudaStream_t stream = nullptr;
    aptb200::Plan plan;

    uint64_t max_samples = 0, max_work = 0, max_out = 0;

    aptb200::FrontTables front;    // the first stage's taps and tables
    float *d_lp = nullptr, *d_one = nullptr;
    int8_t *d_guard = nullptr;
    void *d_in = nullptr;          // staging for submit_host (f32 sized)
    float *d_conv = nullptr;       // f32 copy of a PCM16 input for a first stage that wants one (allocated on first use)
    // chunked upload of long host recordings (BASELINE configs[2]): two staging buffers of chunk_samples each,
    // a copy stream and events so that the H2D of chunk c+1 overlaps the resampling of chunk c
    uint64_t chunk_samples = 0;    // 0: the whole recording is staged at once
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
    uint64_t job_chunks = 0;
    uint64_t conv_cap = 0;         // samples d_conv holds
    float *d_r = nullptr;          // resampled signal, only for a first stage that needs the scratch
    float *d_e = nullptr;          // envelope           ("demodulation_result")
    uint64_t l2_window_bytes = 0;  // bytes of d_e covered by a persisting L2 access-policy window on `stream` (0: none)
    aptb200::BackPlan back_plan;   // the back half's kind and buffer sizes
    aptb200::BackBuffers back;     // its buffers
    aptb200::BackKind last_back = aptb200::BackKind::Generic;   // the kind that ran the last job: where its roots and
                                                                  // records are, and whether it wrote f / corr
    bool stages_materialised = false;  // f / corr of a Records job computed since by apt_decoder_read_stage
    float *d_out = nullptr;        // rows for submit_host
    // pageable host buffers (what the reference-facing apt_decode receives) go through a pinned ring + copy threads
    aptb200::HostStager *stager = nullptr;                 // the one in use (own_stager, or the batch feeder's)
    std::unique_ptr<aptb200::HostStager> own_stager;
    float *h_out = nullptr;        // pinned landing buffer for the rows when the caller's buffer is pageable
    bool job_in_pageable = false, job_out_pageable = false;
    uint64_t job_d2h_floats = 0;   // rows copied back by the job (an upper bound when syncing: n_rows is not known yet)
    aptb200::SyncResult *h_res = nullptr;   // pinned

    // image / process mode and PNG mode (png.hpp): img.plan.image, the job's output is the image of the plan, else f32
    // rows.  The pixels grow on first use; in PNG mode the image is encoded at wait() and only the file is copied out.
    aptb200::ImageOut img;

    // apt_decode_iq (allocated on first use): the I/Q stage's tables for iq_settings, one chunk's I/Q window and the
    // audio the FM kernel writes, which is the input of the decode job
    apt_iq_settings iq_settings{};
    bool iq_tables_valid = false;
    aptb200::IqTables iq_tables;
    aptb200::IqWindow iq_win;
    float *d_audio = nullptr;
    uint64_t audio_cap = 0;        // floats d_audio holds

    // job in flight
    bool in_flight = false;
    bool job_host = false, job_sync = false;
    int job_status = APT_OK;
    uint64_t job_n = 0, job_work = 0, job_fixed_out = 0;
    float *job_out = nullptr;      // caller's buffer (host or device)
    uint64_t job_cap = 0;
    const float *job_rows_src = nullptr;
    uint64_t last_work = 0, last_rows = 0, last_peaks = 0, last_out = 0;

    // profiling
    bool profiling = false;
    std::vector<std::string> kernel_names;
    std::vector<cudaEvent_t> ev_begin, ev_end;
    std::vector<float> kernel_ms;
    int ev_used = 0;
    uint64_t launches = 0;

    apt_status_cb cb = nullptr;
    void *cb_user = nullptr;
};
