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

}  // namespace aptb200
