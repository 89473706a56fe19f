// noaa_apt.hpp -- C++ host-side mirror of the reference's module surface for the decode path, layered on
// the C ABI (aptb200.h).  Same names, argument meaning and error behaviour as the Rust crate:
//
//   noaa_apt::decode(ctx, settings, signal, input_rate, sync)        decode.rs:43-49  (re-exported noaa_apt.rs:5)
//   noaa_apt::dsp::{resample_with_filter, resample, demodulate, filter}   dsp.rs:62,132,350,386
//   noaa_apt::filters::{Filter, NoFilter, Lowpass, LowpassDcRemoval}      filters.rs:10-46
//   noaa_apt::{Freq, Rate}                                                frequency.rs:30-117
//   noaa_apt::Context (status callback)                                   context.rs:100-129
//   noaa_apt::config::Settings (DSP fields)                               config.rs:85-98
//   noaa_apt::err::Error                                                  err.rs:9-44  (err::Result<T> -> exceptions)
//
// Header only; link with libaptb200.so.  The Rust toolchain is not available in the build image, so this is
// the compiled host side above the ABI; rust/ holds the equivalent Rust shim as source.
#pragma once

#include <algorithm>
#include <cstdint>
#include <exception>
#include <functional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "aptb200.h"

namespace noaa_apt {

using Signal = std::vector<float>;   // dsp.rs:16

namespace err {
enum class Kind { Internal, RateOverflow, InvalidInput, Cuda };
struct Error : std::runtime_error {
    Kind kind;
    int status;
    Error(Kind k, int st, const std::string &msg) : std::runtime_error(msg), kind(k), status(st) {}
};
inline void check(int st) {
    if (st == APT_OK) return;
    std::string msg = apt_last_error();
    if (msg.empty()) msg = apt_strerror(st);
    switch (st) {
    case APT_ERR_RESAMPLE_TO_ZERO:
    case APT_ERR_TOO_SHORT:
    case APT_ERR_FEW_SYNC_FRAMES:
    case APT_ERR_WORK_RATE:
    case APT_ERR_EMPTY_RESULT: throw Error(Kind::Internal, st, msg);
    case APT_ERR_RATE_OVERFLOW: throw Error(Kind::RateOverflow, st, msg);
    case APT_ERR_CUDA:
    case APT_ERR_NOMEM: throw Error(Kind::Cuda, st, msg);
    default: throw Error(Kind::InvalidInput, st, msg);
    }
}
}  // namespace err

struct Rate {   // frequency.rs:98-117
    uint32_t value;
    static Rate hz(uint32_t r) { return Rate{r}; }
    uint32_t get_hz() const { return value; }
    bool operator==(Rate o) const { return value == o.value; }
};

struct Freq {   // frequency.rs:30-87 (held as a fraction of pi rad/sample)
    float value;
    static Freq pi_rad(float f) { return Freq{f}; }
    static Freq hz(float f, Rate rate) { return Freq{apt_freq_hz(f, rate.get_hz())}; }
    float get_pi_rad() const { return value; }
    Freq operator/(float d) const { return Freq{value / d}; }
    bool operator==(Freq o) const { return value == o.value; }
};

class Context {   // context.rs:100-129; the per-step WAV export is not part of the fast path
  public:
    using Callback = std::function<void(float, const std::string &)>;
    explicit Context(Callback cb = nullptr) : cb_(std::move(cb)) {}
    static Context decode(Callback cb = nullptr) { return Context(std::move(cb)); }
    static Context resample(Callback cb = nullptr) { return Context(std::move(cb)); }
    void status(float progress, const std::string &description) {
        if (cb_) cb_(progress, description);
    }
    static void trampoline(float progress, const char *description, void *user) {
        static_cast<Context *>(user)->status(progress, description ? description : "");
    }
    static constexpr bool export_steps = false, export_resample_filtered = false;

  private:
    Callback cb_;
};

namespace config {
struct Settings {   // config.rs:85-98, defaults = "standard" profile (default_settings.toml:108-116)
    uint32_t work_rate = 12480;
    float resample_atten = 30.f, resample_delta_freq = 1000.f, resample_cutout = 4800.f, demodulation_atten = 25.f;
    float wav_resample_atten = 40.f, wav_resample_delta_freq = 0.1f;
    apt_settings to_c() const {
        return apt_settings{work_rate, resample_atten, resample_delta_freq, resample_cutout, demodulation_atten};
    }
    static Settings profile(const std::string &name) {
        apt_settings c;
        err::check(apt_profile_settings(name.c_str(), &c));
        Settings s;
        s.work_rate = c.work_rate;
        s.resample_atten = c.resample_atten;
        s.resample_delta_freq = c.resample_delta_freq;
        s.resample_cutout = c.resample_cutout;
        s.demodulation_atten = c.demodulation_atten;
        return s;
    }
};
}  // namespace config

namespace filters {
struct Filter {   // filters.rs:10-16
    virtual ~Filter() = default;
    virtual apt_filter to_c() const = 0;
    virtual void resample(Rate /*input_rate*/, Rate /*output_rate*/) {}
    Signal design() const {
        const apt_filter f = to_c();
        size_t n = 0;
        err::check(apt_filter_design(&f, nullptr, 0, &n));
        Signal taps(n);
        err::check(apt_filter_design(&f, taps.data(), taps.size(), &n));
        return taps;
    }
};
struct NoFilter : Filter {   // filters.rs:48-54
    apt_filter to_c() const override { return apt_filter{APT_FILTER_NONE, 0.f, 0.f, 0.f}; }
};
struct Lowpass : Filter {   // filters.rs:56-95
    Freq cutout;
    float atten;
    Freq delta_w;
    Lowpass(Freq c, float a, Freq d) : cutout(c), atten(a), delta_w(d) {}
    apt_filter to_c() const override { return apt_filter{APT_FILTER_LOWPASS, cutout.value, atten, delta_w.value}; }
    void resample(Rate in, Rate out) override {
        apt_filter f = to_c();
        apt_filter_resample(&f, in.get_hz(), out.get_hz());
        cutout.value = f.cutout_pi;
        delta_w.value = f.delta_w_pi;
    }
};
struct LowpassDcRemoval : Lowpass {   // filters.rs:97-139
    using Lowpass::Lowpass;
    apt_filter to_c() const override { return apt_filter{APT_FILTER_LOWPASS_DC, cutout.value, atten, delta_w.value}; }
};
}  // namespace filters

namespace dsp {
using noaa_apt::Freq;
using noaa_apt::Rate;
using noaa_apt::Signal;

inline Signal resample_with_filter(Context &, const Signal &signal, Rate input_rate, Rate output_rate,
                                   const filters::Filter &filt) {   // dsp.rs:62-126
    const apt_filter f = filt.to_c();
    uint64_t n = 0;
    err::check(apt_resample_len(signal.size(), input_rate.get_hz(), output_rate.get_hz(), &f, &n));
    Signal out(n);
    err::check(apt_resample_with_filter(signal.data(), signal.size(), input_rate.get_hz(), output_rate.get_hz(), &f,
                                        out.data(), out.size(), &n));
    out.resize(n);
    return out;
}
inline Signal resample(Context &ctx, const Signal &signal, Rate input_rate, Rate output_rate, float atten,
                       Freq delta_w) {   // dsp.rs:132-162
    const float cut_hz = output_rate.get_hz() > input_rate.get_hz() ? static_cast<float>(input_rate.get_hz()) / 2.f
                                                                    : static_cast<float>(output_rate.get_hz()) / 2.f;
    return resample_with_filter(ctx, signal, input_rate, output_rate,
                                filters::Lowpass(Freq::hz(cut_hz, input_rate), atten, delta_w));
}
inline Signal demodulate(Context &, const Signal &signal, Freq carrier_freq) {   // dsp.rs:350-383
    Signal out(signal.size());
    err::check(apt_demodulate(signal.data(), signal.size(), carrier_freq.get_pi_rad(), out.data()));
    return out;
}
inline Signal filter(Context &, const Signal &signal, const filters::Filter &filt) {   // dsp.rs:386-410
    const apt_filter f = filt.to_c();
    Signal out(signal.size());
    err::check(apt_filter_signal(signal.data(), signal.size(), &f, out.data()));
    return out;
}
}  // namespace dsp

// noaa_apt::decode == decode::decode, decode.rs:43-162
inline Signal decode(Context &ctx, const config::Settings &settings, const Signal &signal, Rate input_rate, bool sync) {
    const apt_settings s = settings.to_c();
    uint64_t bound = 0, n = 0;
    err::check(apt_decode_len_bound(signal.size(), input_rate.get_hz(), &s, &bound));
    Signal out(bound ? bound : 1);
    err::check(apt_decode(signal.data(), signal.size(), input_rate.get_hz(), &s, sync ? 1 : 0, out.data(), out.size(),
                          &n, &Context::trampoline, &ctx));
    out.resize(n);
    return out;
}

// decode() with tracked sync (aptb200.h apt_decoder_set_sync_mode, DESIGN.md "Tracked sync") on a decoder of its own
// on device 0; track == nullptr takes the defaults (delta 2, lambda 0.25).
inline Signal decode_tracked(const config::Settings &settings, const Signal &signal, Rate input_rate,
                             const apt_track_settings *track = nullptr) {
    const apt_settings s = settings.to_c();
    uint64_t bound = 0, n = 0;
    err::check(apt_decode_len_bound(signal.size(), input_rate.get_hz(), &s, &bound));
    apt_decoder *dec = nullptr;
    err::check(apt_decoder_create(0, input_rate.get_hz(), &s, signal.size(), &dec));
    struct Guard {
        apt_decoder *d;
        ~Guard() { apt_decoder_destroy(d); }
    } guard{dec};
    Signal out(bound ? bound : 1);
    err::check(apt_decoder_set_sync_mode(dec, APT_SYNC_TRACK, track));
    err::check(apt_decoder_submit_host(dec, signal.data(), APT_F32, signal.size(), 1, out.data(), out.size()));
    err::check(apt_decoder_wait(dec, &n));
    out.resize(n);
    return out;
}

// decode::find_sync, decode.rs:204-263 (private in the crate; exposed for tests)
inline std::vector<uint64_t> find_sync(Context &, const Signal &signal, Rate work_rate) {
    std::vector<uint64_t> pos(signal.size() / 64 + 8);
    size_t n = 0;
    err::check(apt_find_sync(signal.data(), signal.size(), work_rate.get_hz(), pos.data(), pos.size(), &n, nullptr));
    pos.resize(n);
    return pos;
}

// Live decoding (apt_stream_*): push audio as it arrives, get the rows that became final.  The rows of all pushes plus
// finish() equal decode() on the whole recording bit for bit.  Owns the device memory from construction to destruction.
class Stream {
  public:
    Stream(Rate input_rate, const config::Settings &settings, bool sync = true, uint64_t max_push = 48000, int device = 0) {
        const apt_settings s = settings.to_c();
        err::check(apt_stream_create(device, input_rate.get_hz(), &s, sync ? 1 : 0, max_push, &st_));
    }
    // I/Q stream (apt_stream_create_iq): push_iq() takes APT_CU8 / APT_CS16 / APT_CF32 samples, max_push counts them.
    Stream(const apt_iq_settings &iq, const config::Settings &settings, bool sync = true, uint64_t max_push = 1200000,
           int device = 0) {
        const apt_settings s = settings.to_c();
        err::check(apt_stream_create_iq(device, &iq, &s, sync ? 1 : 0, max_push, &st_));
    }
    ~Stream() { apt_stream_destroy(st_); }
    Stream(const Stream &) = delete;
    Stream &operator=(const Stream &) = delete;

    Signal push(const float *samples, size_t n) { return rows(n, [&](float *o, uint64_t c, uint64_t *k) {
        return apt_stream_push(st_, samples, APT_F32, n, o, c, k); }); }
    Signal push(const int16_t *samples, size_t n) { return rows(n, [&](float *o, uint64_t c, uint64_t *k) {
        return apt_stream_push(st_, samples, APT_PCM16, n, o, c, k); }); }
    Signal push(const Signal &samples) { return push(samples.data(), samples.size()); }
    // n complex samples, interleaved I, Q
    Signal push_iq(const void *samples, int format, size_t n) { return rows(n, [&](float *o, uint64_t c, uint64_t *k) {
        return apt_stream_push(st_, samples, format, n, o, c, k); }); }
    Signal finish() { return rows(0, [&](float *o, uint64_t c, uint64_t *k) { return apt_stream_finish(st_, o, c, k); }); }
    void reset() { err::check(apt_stream_reset(st_)); }

    // Image output (before the first push of a pass): finish_image() also returns the image of process() (ps) for up to
    // max_rows rows, or with set_png_mode its PNG file.  set_process_mode(nullptr) switches both off.
    void set_process_mode(const apt_process_settings *ps, uint64_t max_rows = 2400) {
        err::check(apt_stream_set_process_mode(st_, ps, max_rows));
        max_rows_ = ps ? max_rows : 0;
        bpp_ = ps && ps->rgba ? 4 : 1;
        png_ = false;
    }
    void set_png_mode(const apt_png_settings *png) {
        err::check(apt_stream_set_png_mode(st_, png));
        png_ = png != nullptr;
        if (png) png_settings_ = *png;
    }
    struct Image {
        Signal rows;                  // the rows finish() would return
        std::vector<uint8_t> bytes;   // rows * 2080 * (1 grey | 4 RGBA) pixel bytes, or the PNG file
        apt_image_info info{};
    };
    Image finish_image() {
        Image im;
        uint64_t cap = max_rows_ * 2080 * bpp_, n = 0;
        if (png_) err::check(apt_png_bound(2080, static_cast<uint32_t>(max_rows_ ? max_rows_ : 1), bpp_, &png_settings_, &cap));
        im.bytes.resize(cap ? cap : 1);
        im.rows = rows(0, [&](float *o, uint64_t c, uint64_t *k) {
            return apt_stream_finish_image(st_, o, c, k, im.bytes.data(), im.bytes.size(), &n, &im.info);
        });
        im.bytes.resize(n);
        return im;
    }
    std::vector<uint64_t> positions() const {
        size_t n = 0;
        err::check(apt_stream_sync_positions(st_, nullptr, 0, &n));
        std::vector<uint64_t> pos(n);
        if (n) err::check(apt_stream_sync_positions(st_, pos.data(), pos.size(), &n));
        return pos;
    }
    apt_stream_info info() const {
        apt_stream_info i{};
        err::check(apt_stream_get_info(st_, &i));
        return i;
    }

  private:
    template <typename F>
    Signal rows(uint64_t n, F call) {
        uint64_t cap = 0, got = 0;
        err::check(apt_stream_push_bound(st_, n, &cap));
        Signal out(cap ? cap : 1);
        err::check(call(out.data(), out.size(), &got));
        out.resize(got);
        return out;
    }
    apt_stream *st_ = nullptr;
    uint64_t max_rows_ = 0;
    int bpp_ = 1;
    bool png_ = false;
    apt_png_settings png_settings_{};
};

// Decoding straight from SDR I/Q (DESIGN.md §10).  format: APT_CU8 / APT_CS16 / APT_CF32, n complex samples.
namespace iq {
inline apt_iq_settings default_settings(uint32_t iq_rate, int32_t offset_hz = 0) {
    apt_iq_settings s{};
    err::check(apt_iq_default_settings(iq_rate, offset_hz, &s));
    return s;
}
inline Signal fm_demod(const void *samples, int format, uint64_t n, const apt_iq_settings &s) {
    uint64_t len = 0, got = 0;
    err::check(apt_fm_demod_len(n, &s, &len));
    Signal out(len ? len : 1);
    err::check(apt_fm_demod(samples, format, n, &s, out.data(), out.size(), &got));
    out.resize(got);
    return out;
}
inline Signal decode_iq(Context &ctx, const config::Settings &settings, const void *samples, int format, uint64_t n,
                        const apt_iq_settings &s, bool sync) {
    const apt_settings st = settings.to_c();
    uint64_t len = 0, bound = 0, got = 0;
    err::check(apt_fm_demod_len(n, &s, &len));
    err::check(apt_decode_len_bound(len, s.audio_rate, &st, &bound));
    Signal out(bound ? bound : 1);
    err::check(apt_decode_iq(samples, format, n, &s, &st, sync ? 1 : 0, out.data(), out.size(), &got, &Context::trampoline, &ctx));
    out.resize(got);
    return out;
}
// Finding the carriers of a recording (DESIGN.md §10, "Finding carriers")
struct Spectrum {
    std::vector<float> psd;   // fftshifted: bin b is (b - nfft/2) iq_rate / nfft Hz
    uint32_t segments = 0;
};
inline Spectrum spectrum(const void *samples, int format, uint64_t n, uint32_t iq_rate, uint32_t nfft = 16384,
                         uint32_t max_segments = 2048) {
    const apt_spectrum_settings ss{nfft, max_segments};
    Spectrum out;
    out.psd.resize(nfft);
    err::check(apt_iq_spectrum(samples, format, n, iq_rate, &ss, out.psd.data(), out.psd.size(), &out.segments));
    return out;
}
inline std::vector<apt_carrier> find_carriers(const void *samples, int format, uint64_t n, const apt_iq_settings &s,
                                              const apt_carrier_search &cs = apt_carrier_search{}) {
    std::vector<apt_carrier> out(s.iq_rate / 40000 + 2);   // kept carriers are more than 40 kHz apart
    uint32_t count = 0;
    err::check(apt_iq_find_carriers(samples, format, n, &s, &cs, out.data(), static_cast<uint32_t>(out.size()), &count));
    out.resize(count);
    return out;
}
struct Channel {
    apt_carrier carrier;
    int status;               // APT_OK, or the failure of this channel's decode
    Signal rows;
};
// Every APT carrier decoded from one upload of the recording; a channel that fails keeps its status, the call throws
// only for errors every channel shares.
inline std::vector<Channel> decode_iq_auto(const config::Settings &settings, const void *samples, int format, uint64_t n,
                                           const apt_iq_settings &s, bool sync,
                                           const apt_carrier_search &cs = apt_carrier_search{}, uint32_t max_channels = 8) {
    const apt_settings st = settings.to_c();
    apt_iq_settings s0 = s;
    s0.offset_hz = 0;
    uint64_t len = 0, bound = 0;
    err::check(apt_fm_demod_len(n, &s0, &len));
    err::check(apt_decode_len_bound(len, s.audio_rate, &st, &bound));
    const uint32_t k = max_channels ? max_channels : 1;
    std::vector<Signal> bufs(k, Signal(bound ? bound : 1));
    std::vector<float *> outs(k);
    for (uint32_t i = 0; i < k; ++i) outs[i] = bufs[i].data();
    std::vector<uint64_t> caps(k, bound ? bound : 1), nouts(k, 0);
    std::vector<int> statuses(k, 0);
    std::vector<apt_carrier> found(k);
    uint32_t nfound = 0;
    const int rc = apt_decode_iq_auto(samples, format, n, &s, &cs, &st, sync ? 1 : 0, found.data(), k, &nfound, outs.data(),
                                      caps.data(), nouts.data(), statuses.data());
    bool shared = rc != APT_OK;
    for (uint32_t i = 0; i < nfound; ++i) shared = shared && statuses[i] == rc;
    if (rc != APT_OK && (nfound == 0 || shared)) err::check(rc);
    std::vector<Channel> out;
    for (uint32_t i = 0; i < nfound; ++i) {
        bufs[i].resize(statuses[i] == APT_OK ? nouts[i] : 0);
        out.push_back(Channel{found[i], statuses[i], std::move(bufs[i])});
    }
    return out;
}
}  // namespace iq

// PNG output encoded on the device (DESIGN.md §11): the file's bytes, ready to write.
namespace png {
inline apt_png_settings default_settings() {
    apt_png_settings s{};
    apt_png_default_settings(&s);
    return s;
}
// pixels: height rows of width * channels bytes (channels 1 grey, 3 RGB, 4 RGBA)
inline std::vector<uint8_t> encode(const uint8_t *pixels, uint32_t width, uint32_t height, int channels,
                                   const apt_png_settings &ps = default_settings()) {
    uint64_t cap = 0, got = 0;
    err::check(apt_png_bound(width, height, channels, &ps, &cap));
    std::vector<uint8_t> out(cap);
    err::check(apt_png_encode(pixels, width, height, channels, &ps, out.data(), out.size(), &got));
    out.resize(got);
    return out;
}
// decode() + process() (no map overlay) + PNG in one call; only the PNG bytes leave the GPU
inline std::vector<uint8_t> decode_png(Context &ctx, const config::Settings &settings, const Signal &signal, Rate input_rate,
                                       bool sync, const apt_process_settings &ps,
                                       const apt_png_settings &png = default_settings(), apt_image_info *info = nullptr) {
    const apt_settings s = settings.to_c();
    uint64_t bound = 0, cap = 0, got = 0;
    err::check(apt_decode_len_bound(signal.size(), input_rate.get_hz(), &s, &bound));
    const uint64_t rows = bound / 2080 ? bound / 2080 : 1;
    err::check(apt_png_bound(2080, static_cast<uint32_t>(rows), ps.rgba ? 4 : 1, &png, &cap));
    std::vector<uint8_t> out(cap);
    err::check(apt_decode_png(signal.data(), APT_F32, signal.size(), input_rate.get_hz(), &s, sync ? 1 : 0, &ps, &png,
                              out.data(), out.size(), &got, info, &Context::trampoline, &ctx));
    out.resize(got);
    return out;
}
// A batch of recordings, each ending in its PNG file (png != nullptr) or its processed image (png == nullptr), sharded
// over `devices` as apt_decode_batch does.  files[i] is empty where statuses[i] is not APT_OK; infos[i] is that
// recording's apt_image_info.  Returns the first failing status (0 when every recording succeeded).
struct BatchImages {
    std::vector<std::vector<uint8_t>> files;
    std::vector<apt_image_info> infos;
    std::vector<int> statuses;
};
inline int decode_batch_png(const std::vector<Signal> &signals, Rate input_rate, const config::Settings &settings, bool sync,
                            const apt_process_settings &ps, const apt_png_settings *png, BatchImages &res,
                            const std::vector<int> &devices = {}, int streams_per_device = 4) {
    const apt_settings s = settings.to_c();
    const size_t count = signals.size();
    std::vector<const void *> sigs(count);
    std::vector<uint64_t> lens(count), caps(count), nouts(count);
    std::vector<uint8_t *> outs(count);
    res.files.assign(count, {});
    res.infos.assign(count, apt_image_info{});
    res.statuses.assign(count, APT_ERR_CUDA);
    for (size_t i = 0; i < count; ++i) {
        uint64_t bound = 0;
        err::check(apt_decode_len_bound(signals[i].size(), input_rate.get_hz(), &s, &bound));
        const uint64_t rows = bound / 2080 ? bound / 2080 : 1;
        if (png) err::check(apt_png_bound(2080, static_cast<uint32_t>(rows), ps.rgba ? 4 : 1, png, &caps[i]));
        else caps[i] = (bound ? bound : 1) * (ps.rgba ? 4 : 1);
        res.files[i].resize(caps[i]);
        sigs[i] = signals[i].data();
        lens[i] = signals[i].size();
        outs[i] = res.files[i].data();
    }
    const int rc = apt_decode_batch_image(sigs.data(), APT_F32, lens.data(), static_cast<int>(count), input_rate.get_hz(), &s,
                                          sync ? 1 : 0, &ps, png, outs.data(), caps.data(), nouts.data(), res.infos.data(),
                                          res.statuses.data(), devices.empty() ? nullptr : devices.data(),
                                          static_cast<int>(devices.size()), streams_per_device);
    for (size_t i = 0; i < count; ++i) res.files[i].resize(res.statuses[i] == APT_OK ? nouts[i] : 0);
    return rc;
}
// The reference CLI's job: WAV in, PNG file out
inline void decode_wav_png(const std::string &input, const std::string &output, const config::Settings &settings, bool sync,
                           const apt_process_settings &ps, const apt_png_settings &png = default_settings()) {
    const apt_settings s = settings.to_c();
    err::check(apt_decode_wav_png(input.c_str(), output.c_str(), &s, sync ? 1 : 0, &ps, &png, nullptr));
}
}  // namespace png

// Finding the satellite passes in a long recording and decoding each one from one upload (DESIGN.md §12)
namespace passes {
inline std::vector<apt_pass> find_passes_quality(const std::vector<float> &q, uint64_t n, uint32_t input_rate,
                                                 const apt_pass_search &ps = apt_pass_search{}) {
    uint32_t count = 0;
    const int st = apt_find_passes_quality(q.data(), q.size(), n, input_rate, &ps, nullptr, 0, &count);
    if (st != APT_ERR_CAPACITY) err::check(st);
    std::vector<apt_pass> out(count);
    if (count) err::check(apt_find_passes_quality(q.data(), q.size(), n, input_rate, &ps, out.data(), count, &count));
    return out;
}
struct Image {
    int status;               // APT_OK, or the failure of this range alone
    std::vector<uint8_t> png;
    apt_image_info info;
};
// The samples (APT_F32 / APT_PCM16 host memory) uploaded once and kept on the device until the object goes away.
class Recording {
public:
    Recording(const void *samples, int format, uint64_t n, Rate input_rate, const config::Settings &settings = {},
              int device = 0)
        : n_(n), rate_(input_rate.get_hz()), settings_(settings) {
        const apt_settings st = settings.to_c();
        err::check(apt_recording_create(device, samples, format, n, rate_, &st, &h_));
    }
    ~Recording() { apt_recording_destroy(h_); }
    Recording(const Recording &) = delete;
    Recording &operator=(const Recording &) = delete;
    apt_recording_info info() const {
        apt_recording_info i{};
        err::check(apt_recording_get_info(h_, &i));
        return i;
    }
    std::vector<float> quality() const {
        uint64_t nq = 0;
        err::check(apt_recording_quality(h_, nullptr, 0, &nq));
        std::vector<float> q(nq);
        if (nq) err::check(apt_recording_quality(h_, q.data(), q.size(), &nq));
        return q;
    }
    std::vector<apt_pass> find_passes(const apt_pass_search &ps = apt_pass_search{}) const {
        return find_passes_quality(quality(), n_, rate_, ps);
    }
    // Each range as apt_decode_png of the host slice; throws only for errors every range shares.
    std::vector<Image> decode_png(const std::vector<apt_pass> &ranges, bool sync, const apt_process_settings &ps,
                                  const apt_png_settings &png = png::default_settings()) const {
        const uint32_t k = static_cast<uint32_t>(ranges.size());
        std::vector<Image> out(k);
        if (!k) return out;
        const apt_settings st = settings_.to_c();
        std::vector<void *> outs(k);
        std::vector<uint64_t> caps(k), nouts(k, 0);
        std::vector<apt_image_info> infos(k);
        std::vector<int> statuses(k, 0);
        for (uint32_t i = 0; i < k; ++i) {
            uint64_t bound = 0, bytes = 0;
            const uint64_t len = ranges[i].end > ranges[i].start ? ranges[i].end - ranges[i].start : 0;
            err::check(apt_decode_len_bound(len, rate_, &st, &bound));
            const uint32_t rows = static_cast<uint32_t>(std::max<uint64_t>(bound / 2080, 1));
            err::check(apt_png_bound(2080, rows, ps.rgba ? 4 : 1, &png, &bytes));
            out[i].png.resize(bytes ? bytes : 1);
            outs[i] = out[i].png.data();
            caps[i] = out[i].png.size();
        }
        const int rc = apt_recording_decode(h_, ranges.data(), k, sync ? 1 : 0, &ps, &png, outs.data(), caps.data(),
                                            nouts.data(), infos.data(), statuses.data());
        bool shared = rc != APT_OK;
        for (uint32_t i = 0; i < k; ++i) shared = shared && statuses[i] == rc;
        if (shared && rc == APT_ERR_BAD_ARG) err::check(rc);
        for (uint32_t i = 0; i < k; ++i) {
            out[i].status = statuses[i];
            out[i].info = infos[i];
            out[i].png.resize(statuses[i] == APT_OK ? nouts[i] : 0);
        }
        return out;
    }

private:
    apt_recording *h_ = nullptr;
    uint64_t n_;
    uint32_t rate_;
    config::Settings settings_;
};

// A continuous feed watched for satellite passes (apt_watch, DESIGN.md §13).  on_event receives every AOS, SEGMENT and
// LOS on the pushing thread; an LOS carries the pass's decode (ev.data valid during the call only).  An exception thrown
// by on_event is kept and rethrown when the push or finish returns; it never crosses the library.
class Watch {
public:
    using Callback = std::function<void(const apt_watch_event &)>;
    Watch(Rate input_rate, Callback on_event, const apt_watch_settings &ws = apt_watch_settings{},
          const config::Settings &settings = {}, int device = 0)
        : cb_(std::move(on_event)) {
        const apt_settings st = settings.to_c();
        err::check(apt_watch_create(device, input_rate.get_hz(), &st, &ws, &Watch::trampoline, this, &h_));
    }
    ~Watch() { apt_watch_destroy(h_); }
    Watch(const Watch &) = delete;
    Watch &operator=(const Watch &) = delete;
    // The quality of the windows that became final.
    std::vector<float> push(const float *samples, uint64_t n) { return push_format(samples, APT_F32, n); }
    std::vector<float> push(const int16_t *samples, uint64_t n) { return push_format(samples, APT_PCM16, n); }
    std::vector<float> finish() {
        std::vector<float> q(bound(0));
        uint64_t nq = 0;
        const int rc = apt_watch_finish(h_, q.data(), q.size(), &nq);
        rethrow();
        err::check(rc);
        q.resize(nq);
        return q;
    }
    void reset() { err::check(apt_watch_reset(h_)); }
    apt_watch_info info() const {
        apt_watch_info i{};
        err::check(apt_watch_get_info(h_, &i));
        return i;
    }

private:
    static void trampoline(const apt_watch_event *ev, void *user) {
        Watch *w = static_cast<Watch *>(user);
        if (!w->cb_ || w->error_) return;
        try {
            w->cb_(*ev);
        } catch (...) {
            w->error_ = std::current_exception();
        }
    }
    uint64_t bound(uint64_t n) {
        uint64_t cap = 0;
        err::check(apt_watch_push_bound(h_, n, &cap));
        return std::max<uint64_t>(cap, 1);
    }
    std::vector<float> push_format(const void *samples, int format, uint64_t n) {
        std::vector<float> q(bound(n));
        uint64_t nq = 0;
        const int rc = apt_watch_push(h_, samples, format, n, q.data(), q.size(), &nq);
        rethrow();
        err::check(rc);
        q.resize(nq);
        return q;
    }
    void rethrow() {
        if (!error_) return;
        std::exception_ptr e = error_;
        error_ = nullptr;
        std::rethrow_exception(e);
    }
    Callback cb_;
    std::exception_ptr error_;
    apt_watch *h_ = nullptr;
};

// apt_watch_iq (DESIGN.md §14): one SDR's I/Q feed watched on up to 8 channels (offsets in Hz from the tuned centre;
// iq.offset_hz is ignored).  Channel c behaves as a Watch on apt_fm_demod at offsets[c]; push / finish return each
// channel's new q.  Event positions are audio samples of the channel.
class IqWatch {
public:
    using Callback = std::function<void(int channel, const apt_watch_event &)>;
    IqWatch(const apt_iq_settings &iq, const std::vector<int32_t> &offsets, Callback on_event,
            const apt_watch_settings &ws = apt_watch_settings{}, const config::Settings &settings = {}, int device = 0)
        : cb_(std::move(on_event)), count_(static_cast<int>(offsets.size())) {
        const apt_settings st = settings.to_c();
        err::check(apt_watch_iq_create(device, &iq, offsets.data(), count_, &st, &ws, &IqWatch::trampoline, this, &h_));
    }
    ~IqWatch() { apt_watch_iq_destroy(h_); }
    IqWatch(const IqWatch &) = delete;
    IqWatch &operator=(const IqWatch &) = delete;
    // n complex samples of APT_CU8, APT_CS16 or APT_CF32 (interleaved I, Q): the q of each channel's windows that became final.
    std::vector<std::vector<float>> push(const void *iq, int format, uint64_t n) {
        const uint64_t cap = bound(n);
        std::vector<float> q(cap * count_);
        std::vector<uint64_t> nq(count_);
        const int rc = apt_watch_iq_push(h_, iq, format, n, q.data(), cap, nq.data());
        rethrow();
        err::check(rc);
        return split(q, cap, nq);
    }
    std::vector<std::vector<float>> finish() {
        const uint64_t cap = bound(0);
        std::vector<float> q(cap * count_);
        std::vector<uint64_t> nq(count_);
        const int rc = apt_watch_iq_finish(h_, q.data(), cap, nq.data());
        rethrow();
        err::check(rc);
        return split(q, cap, nq);
    }
    void reset() { err::check(apt_watch_iq_reset(h_)); }
    apt_watch_info info(int channel) const {
        apt_watch_info i{};
        err::check(apt_watch_iq_get_info(h_, channel, &i));
        return i;
    }

private:
    static void trampoline(int channel, const apt_watch_event *ev, void *user) {
        IqWatch *w = static_cast<IqWatch *>(user);
        if (!w->cb_ || w->error_) return;
        try {
            w->cb_(channel, *ev);
        } catch (...) {
            w->error_ = std::current_exception();
        }
    }
    uint64_t bound(uint64_t n) {
        uint64_t cap = 0;
        err::check(apt_watch_iq_push_bound(h_, n, &cap));
        return std::max<uint64_t>(cap, 1);
    }
    std::vector<std::vector<float>> split(const std::vector<float> &q, uint64_t cap, const std::vector<uint64_t> &nq) const {
        std::vector<std::vector<float>> out(count_);
        for (int c = 0; c < count_; ++c) out[c].assign(q.begin() + c * cap, q.begin() + c * cap + nq[c]);
        return out;
    }
    void rethrow() {
        if (!error_) return;
        std::exception_ptr e = error_;
        error_ = nullptr;
        std::rethrow_exception(e);
    }
    Callback cb_;
    std::exception_ptr error_;
    int count_ = 0;
    apt_watch_iq *h_ = nullptr;
};
}  // namespace passes

}  // namespace noaa_apt
