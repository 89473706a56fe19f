// The first stage of decode() (decode.rs:65-89): resampling to the work rate, fused with or followed by the envelope.
// This module alone knows which kernel serves a (ratio, taps) pair, which device tables it reads, what one unit of its
// work is and how to launch it; the decoder, the chunked upload, the stream and apt_resample_with_filter see a FrontPlan.
#pragma once

#include <cstdint>
#include <vector>

#include "filters_host.hpp"
#include "launch.hpp"

namespace aptb200 {

enum class FrontKind {
    Tiled,        // k_polyphase_ws (kernels_fast.cuh): the shapes make_tile_plan fits (48 / 96 kHz)
    UniformTap,   // k_polyphase_ut (kernels_ut.cuh): L = 13 shapes the tiled kernel does not fit (192 kHz)
    PhaseMajor,   // k_polyphase_ph (kernels_ph.cuh): large L (11025 / 22050 / 44100 Hz)
    Generic,      // k_polyphase_generic: any L > 1, one thread per output
    Decimate,     // L = 1: k_fir_decimate_generic into a scratch signal, then k_envelope
};

// Profiling slot of a polyphase kind (the decimate kind reports filter_decimate + envelope).
constexpr const char *kFrontSlot = "resample_envelope";

// Work is counted in units (a tile / block of a tiled kernel, else one output): a unit makes unit_out outputs from unit_in
// new samples, plus `before` samples in front of the first unit of a run and `after` beyond the start of the last one.
struct FrontPlan {
    FrontKind kind = FrontKind::Generic;
    Ratio r{};
    std::vector<float> h;        // filter taps
    uint64_t off2 = 0;           // 2 * ((N-1)/2): highest tap index fast_resampling touches
    uint64_t unit_in = 0, unit_out = 1, before = 0, after = 0;
    // geometry and host tables of the chosen kind (the others stay empty)
    TilePlan tile{};
    std::vector<float> tile_taps;
    std::vector<u32> tile_xs;
    UtPlan ut{};
    std::vector<float> ut_stream;
    PhPlan ph{};
    std::vector<float> ph_table;
    std::vector<unsigned short> ph_xs;

    uint64_t work_len(uint64_t n) const {   // outputs of n input samples: fast_resampling, or filter + decimate (L = 1)
        return kind == FrontKind::Decimate ? n / r.m : polyphase_len(n, r.l, r.m, h.size());
    }
    uint64_t units(uint64_t nwork) const { return (nwork + unit_out - 1) / unit_out; }
    // Input samples [xa, xb) that units [u0, u1) read from a recording of n samples.
    void span(uint64_t u0, uint64_t u1, uint64_t n, uint64_t &xa, uint64_t &xb) const;
    // Units whose input is complete after n samples (nwork outputs in all); at the end of the recording, all of them.
    uint64_t complete(uint64_t n, uint64_t nwork, bool finish) const;
    // Input samples a stream keeps beyond the first sample of its next unit (less than one unit span).
    uint64_t tail() const;
    // Units one chunk of `cap` staged samples serves in the chunked upload (polyphase kinds only: chunkable()).
    int chunk_units(uint64_t cap, uint64_t &per_chunk) const;
    bool chunkable() const { return kind != FrontKind::Decimate; }
    bool needs_scratch() const { return kind == FrontKind::Decimate; }   // front_launch needs nwork floats of scratch
    // The kernel reads f32 only: PCM16 input wants a 16-byte aligned f32 copy to run on it.
    bool wants_f32() const { return kind == FrontKind::Tiled || kind == FrontKind::UniformTap; }
    bool tiles() const { return unit_in != 0; }                              // a unit is more than one output
};

// The kernel for (r, taps): tiled, then uniform-tap, then phase-major, then generic; L = 1 is the decimate kind.
// APTB200_GENERIC_RESAMPLER=1 puts every L > 1 on the generic kernel.
FrontPlan make_front(Ratio r, std::vector<float> taps);

// Device copies of a FrontPlan's taps and of its kind's tables.
struct FrontTables {
    float *h = nullptr;
    float *table = nullptr;      // tiled: tap table; phase-major: phase table
    void *xs = nullptr;          // tiled: u32 window starts; phase-major: u16 window starts
    FrontTables() = default;
    FrontTables(const FrontTables &) = delete;
    ~FrontTables() { release(); }
    int upload(const FrontPlan &f);
    void release();
    static uint64_t bytes(const FrontPlan &f);   // device memory upload() takes
};

// Resampling (+ envelope) of units [u0, u1) of n samples (nwork outputs).  in (APT_F32 / APT_PCM16), conv (an f32 copy of
// PCM16 input, or nullptr), scratch and out are the addresses sample / output 0 would have.  When the chosen kernel cannot
// take the input as given (PCM16 without a copy, f32 that is not 16-byte aligned for the uniform-tap kernel), the generic
// kernel computes exactly the outputs of [u0, u1).  hook (or nullptr) brackets each kernel with a profiling slot.
int front_launch(const LaunchCtx &c, const FrontPlan &f, const FrontTables &t, const void *in, int format, const float *conv,
                 uint64_t n, uint64_t nwork, uint64_t u0, uint64_t u1, bool envelope, float cosphi2, float sinphi,
                 float *scratch, float *out, KernelHook *hook);

// Moves the tail [keep, end) of a window based at `base` to its front when that does not overlap (keep is floored to a
// multiple of 16, so the window keeps its alignment).
int window_compact(cudaStream_t s, float *buf, uint64_t &base, uint64_t keep, uint64_t end);

struct Plan;   // decoder.hpp

// The streamed first stage of the stream and the watcher: the f32 input window ([in_base, samples_in)), the envelope
// window ([e_base, work_final), with the decimating kind's scratch d_r) and the units done; the caller sizes and trims both.
struct FrontWindow {
    float *d_in = nullptr, *d_conv = nullptr, *d_e = nullptr, *d_r = nullptr;   // d_conv: a PCM16 push (d_pcm) as f32
    int16_t *d_pcm = nullptr;
    uint64_t cap_in = 0, cap_e = 0, max_push = 0;
    uint64_t samples_in = 0, in_base = 0, units_done = 0, work_final = 0, e_base = 0;
    FrontWindow() = default;
    FrontWindow(const FrontWindow &) = delete;
    ~FrontWindow() { release(); }
    // envelope outputs one step of max_push samples can finalise (finish: the units the input tail still held)
    static uint64_t step_outputs(const FrontPlan &f, uint64_t max_push) {
        return (max_push + f.tail()) * f.r.l / f.r.m + 2 * f.unit_out + 64;
    }
    static uint64_t bytes(const FrontPlan &f, uint64_t cap_in, uint64_t cap_e, uint64_t max_push) {   // what alloc() takes
        return cap_in * 4 + max_push * (2 + 4) + cap_e * 4 * (f.needs_scratch() ? 2 : 1);
    }
    int alloc(const FrontPlan &f, uint64_t cap_in, uint64_t cap_e, uint64_t max_push);
    void release();
    void clear() { samples_in = in_base = units_done = work_final = e_base = 0; }
    int zero_input(cudaStream_t s) const;   // at create and reset, not at a watcher's segment roll
    // input from min(keep_in, the next unit's first sample), envelope from keep_e (d_r follows only when d_e moves)
    int compact(cudaStream_t s, const FrontPlan &f, uint64_t keep_in, uint64_t keep_e);
    // n host samples (f32, or PCM16 cast through d_pcm and d_conv, so pushes may mix formats) or n f32 device samples
    int push(const LaunchCtx &c, const void *src, bool on_device, int format, uint64_t n);
    // audio written into the window on the device: room(n) checks that n samples fit, commit(n) counts them
    float *in_origin() const { return d_in - in_base; }   // the address input sample 0 would have
    int room(uint64_t n) const;
    void commit(uint64_t n) { samples_in += n; }
    int advance(const LaunchCtx &c, const Plan &p, const FrontTables &t, bool finish);   // the units now complete (all at finish)
    const float *e_origin() const { return d_e - e_base; }   // the address envelope sample 0 would have
};

}  // namespace aptb200
