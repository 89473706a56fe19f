// The I/Q stage (DESIGN.md §10): FM demodulation of complex samples to audio at audio_rate.  This module alone reads
// apt_iq_settings: it validates them, designs the channel filter, lays out the polyphase taps and the phasor table, owns
// their device copies and launches k_fm_demod and k_fm_demod_channels.
#pragma once

#include <cstdint>
#include <vector>

#include "aptb200.h"
#include "launch.hpp"

namespace aptb200 {

struct IqPlan {
    apt_iq_settings s{};
    u32 D = 1;                    // iq_rate / audio_rate
    std::vector<float> h;         // channel Lowpass, N taps
    u32 qpad = 0;                 // taps per polyphase plane, rounded up to 16
    std::vector<float> hp;        // D x qpad: hp[r][q] = h[q*D + r], 0 past N
    std::vector<float> W;         // kIqBlock interleaved phasors W[t] = exp(-2 pi j ((t f) mod fs) / fs)
    uint64_t f = 0;               // offset_hz mod iq_rate, in [0, iq_rate)
    float scale = 0.f;            // (float)(audio_rate / 2pi)
    u32 tz = 0, lp16 = 0, ps = 0; // tile geometry of k_fm_demod
    size_t smem = 0;              // its dynamic shared memory

    uint64_t out_len(uint64_t n) const { return (n + D - 1) / D; }
    // I/Q samples [xa, xb) that audio outputs [m0, m1) read (z[m0 - 1] included), clipped to a recording of n samples.
    void span(uint64_t m0, uint64_t m1, uint64_t n, uint64_t &xa, uint64_t &xb) const;
};

// Validation (host only, APT_ERR_BAD_ARG on failure), D, the taps, W and the tile geometry.
int make_iq(const apt_iq_settings &s, IqPlan &plan);
int iq_default_settings(uint32_t iq_rate, int32_t offset_hz, apt_iq_settings &s);
// bytes per complex sample of an I/Q format, 0 for any other format
size_t iq_sample_bytes(int format);

// Device copies of the taps and the phasor table.
struct IqTables {
    float *hp = nullptr;
    float *W = nullptr;
    IqTables() = default;
    IqTables(const IqTables &) = delete;
    ~IqTables() { release(); }
    int upload(const IqPlan &p, bool taps = true);   // taps = false: the phasors alone (channels that share hp)
    void release();
};

// Audio outputs [m0, m1) of a recording of n I/Q samples.  `window` holds the absolute samples [w_lo, w_hi), which must
// cover plan.span(m0, m1, n); in and out are the addresses sample / output 0 would have.
int iq_launch(const LaunchCtx &c, const IqPlan &plan, const IqTables &t, const void *in, uint64_t w_lo, uint64_t w_hi,
              int format, uint64_t m0, uint64_t m1, float *out);

// The same outputs for `count` (1..8) channels of one window in one launch of k_fm_demod_channels: plans that differ in
// offset_hz only, plans[k] with tables[k] into outs[k].  Channel k's audio is iq_launch's with plans[k], bit for bit.
int iq_launch_channels(const LaunchCtx &c, const IqPlan *const *plans, const IqTables *const *tables, int count,
                       const void *in, uint64_t w_lo, uint64_t w_hi, int format, uint64_t m0, uint64_t m1,
                       float *const *outs);

// n samples of an I/Q format, converted exactly to interleaved f32 at out (the streaming decoder's cf32 window).
int iq_to_cf32(const LaunchCtx &c, const void *in, int format, uint64_t n, float *out);

// I/Q samples per upload chunk: 32 Mi, or APTB200_IQ_CHUNK (diagnostic: puts chunk boundaries inside short inputs).
uint64_t iq_chunk_samples();

// Device buffer of one chunk's I/Q window (grows, never shrinks).
struct IqWindow {
    void *p = nullptr;
    uint64_t cap = 0;   // bytes
    IqWindow() = default;
    IqWindow(const IqWindow &) = delete;
    ~IqWindow() { release(); }
    int reserve(uint64_t bytes);
    void release();
};

// The cf32 window of a live I/Q feed (the I/Q stream's, and the one an I/Q watcher's channels share): each push is uploaded
// once, converted into it exactly, and it keeps the N - 1 + D samples the next audio output reads.  It holds one step, that
// halo and the same again, so that compaction never overlaps.
struct IqFeed {
    float *d_iq = nullptr;        // interleaved cf32, cap complex samples from absolute sample base
    void *d_raw = nullptr;        // one step's pushed samples as they came
    uint64_t cap = 0, in = 0, base = 0;
    IqFeed() = default;
    IqFeed(const IqFeed &) = delete;
    ~IqFeed() { release(); }
    static uint64_t window(const IqPlan &q, uint64_t max_push) { return 2 * (q.h.size() + 2ull * q.D) + max_push + 64; }
    static uint64_t bytes(const IqPlan &q, uint64_t max_push) { return window(q, max_push) * 8 + max_push * 8; }
    int alloc(const IqPlan &q, uint64_t max_push);
    void release();
    // n host samples (at most max_push) on c.stream, after moving to the front what audio output m_next still reads
    int push(const LaunchCtx &c, const IqPlan &q, uint64_t m_next, const void *host, int format, uint64_t n);
    const float *origin() const { return d_iq - 2 * base; }   // the address sample 0 would have
};

// All ceil(n / D) audio samples of the host I/Q `iq` into device d_audio, on c.stream: chunk by chunk, each chunk's window
// (its samples and the halo its first output reads) uploaded through `stager` (pageable input) or cudaMemcpyAsync
// (stager == nullptr), then one launch for the outputs the chunk completes.  The audio is the same for every chunk size.
class HostStager;
int iq_demod_host(const LaunchCtx &c, const IqPlan &p, const IqTables &t, const void *iq, int format, uint64_t n,
                  IqWindow &win, HostStager *stager, float *d_audio, KernelHook *hook);
// The same for `count` channels of one recording (plans that differ in offset_hz only): each chunk is uploaded once and
// demodulated by one iq_launch_channels per 8 channels, plans[k] with tables[k] into d_audio[k].  Channel k's audio is
// iq_demod_host's.
int iq_demod_host_multi(const LaunchCtx &c, const IqPlan *const *plans, const IqTables *const *tables,
                        float *const *d_audio, int count, const void *iq, int format, uint64_t n, IqWindow &win,
                        HostStager *stager, KernelHook *hook);

}  // namespace aptb200
