// Minimal RIFF/WAVE reader and writer for the two file formats the path touches (SURVEY.md §8 f1/f2):
//   wav::load_wav  (wav.rs:11-56): integer PCM (8/16/24/32 bit) or 32-bit float, any channel count, channel 0 kept,
//                  integer samples cast with `as f32` (raw values, not normalised);
//   wav::write_wav (wav.rs:62-98) as resample.rs:53-66 uses it: 16-bit mono PCM.
// Host code only; the reference gets both from the `hound` crate (3.5.1, not vendored).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "aptb200.h"
#include "common.hpp"

using namespace aptb200;

namespace {

struct WavFile {
    FILE *f = nullptr;
    apt_wav_info info{};
    long data_pos = 0;
    uint64_t data_bytes = 0;
    ~WavFile() {
        if (f) fclose(f);
    }
};

uint32_t rd32(const unsigned char *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24); }
uint16_t rd16(const unsigned char *p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }

int open_wav(const char *path, WavFile &w) {
    if (!path) return fail(APT_ERR_BAD_ARG, "null path");
    w.f = fopen(path, "rb");
    if (!w.f) return fail(APT_ERR_IO, "WavOpen: cannot open '%s'", path);
    unsigned char hdr[12];
    if (fread(hdr, 1, 12, w.f) != 12 || memcmp(hdr, "RIFF", 4) || memcmp(hdr + 8, "WAVE", 4))
        return fail(APT_ERR_IO, "WavOpen: '%s' is not a RIFF/WAVE file", path);
    bool have_fmt = false;
    for (;;) {
        unsigned char ch[8];
        if (fread(ch, 1, 8, w.f) != 8) break;
        const uint32_t size = rd32(ch + 4);
        if (!memcmp(ch, "fmt ", 4)) {
            unsigned char fmt[40] = {0};
            const size_t take = size < sizeof(fmt) ? size : sizeof(fmt);
            if (size < 16 || fread(fmt, 1, take, w.f) != take) return fail(APT_ERR_IO, "WavOpen: truncated fmt chunk");
            uint16_t tag = rd16(fmt);
            w.info.channels = rd16(fmt + 2);
            w.info.sample_rate = rd32(fmt + 4);
            w.info.bits_per_sample = rd16(fmt + 14);
            if (tag == 0xFFFE && size >= 26) tag = rd16(fmt + 24);          // WAVE_FORMAT_EXTENSIBLE: sub-format GUID
            if (tag == 1) w.info.is_float = 0;
            else if (tag == 3) w.info.is_float = 1;
            else return fail(APT_ERR_IO, "WavOpen: unsupported WAV format tag %u", tag);
            if (size > take) fseek(w.f, static_cast<long>(size - take), SEEK_CUR);
            if (size & 1) fseek(w.f, 1, SEEK_CUR);
            have_fmt = true;
        } else if (!memcmp(ch, "data", 4)) {
            if (!have_fmt) return fail(APT_ERR_IO, "WavOpen: data chunk before fmt chunk");
            w.data_pos = ftell(w.f);
            w.data_bytes = size;
            // a streamed file may carry 0 / 0xFFFFFFFF here: use what the file really holds
            fseek(w.f, 0, SEEK_END);
            const uint64_t rest = static_cast<uint64_t>(ftell(w.f) - w.data_pos);
            if (size == 0xFFFFFFFFu || size > rest) w.data_bytes = rest;
            break;
        } else {
            fseek(w.f, static_cast<long>(size + (size & 1)), SEEK_CUR);
        }
    }
    if (!have_fmt || w.data_pos == 0) return fail(APT_ERR_IO, "WavOpen: no fmt / data chunk in '%s'", path);
    const uint32_t bps = w.info.bits_per_sample;
    const bool ok = w.info.is_float ? bps == 32 : (bps == 8 || bps == 16 || bps == 24 || bps == 32);
    if (!ok || w.info.channels == 0) return fail(APT_ERR_IO, "WavOpen: unsupported sample size %u bit / %u channels", bps, w.info.channels);
    w.info.frames = w.data_bytes / (static_cast<uint64_t>(bps / 8) * w.info.channels);
    return APT_OK;
}

// channel 0 of the frames, converted by `conv(raw bytes of one sample)`
template <typename T, typename Conv>
int read_channel0(WavFile &w, T *out, uint64_t cap, uint64_t *n, Conv conv) {
    const uint64_t frames = w.info.frames;
    *n = frames;
    if (frames > cap || (!out && frames)) return fail(APT_ERR_CAPACITY, "output needs room for %llu samples", (unsigned long long)frames);
    const size_t bs = w.info.bits_per_sample / 8, fs = bs * w.info.channels;
    fseek(w.f, w.data_pos, SEEK_SET);
    std::vector<unsigned char> buf(fs * 65536);
    uint64_t done = 0;
    while (done < frames) {
        const size_t want = static_cast<size_t>(frames - done < 65536 ? frames - done : 65536);
        if (fread(buf.data(), fs, want, w.f) != want) return fail(APT_ERR_IO, "WavOpen: truncated data chunk");
        for (size_t i = 0; i < want; ++i) out[done + i] = conv(buf.data() + i * fs);
        done += want;
    }
    return APT_OK;
}

}  // namespace

extern "C" int apt_wav_info_read(const char *path, apt_wav_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    WavFile w;
    APT_TRY(open_wav(path, w));
    *info = w.info;
    return APT_OK;
}

extern "C" int apt_wav_load(const char *path, float *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate) {
    if (!n) return fail(APT_ERR_BAD_ARG, "null argument");
    WavFile w;
    APT_TRY(open_wav(path, w));
    if (sample_rate) *sample_rate = w.info.sample_rate;
    const uint32_t bps = w.info.bits_per_sample;
    if (w.info.is_float)
        return read_channel0(w, out, cap, n, [](const unsigned char *p) { float v; memcpy(&v, p, 4); return v; });
    // integer PCM -> i32 (hound: 8-bit is unsigned with an offset of 128, the rest signed little endian) -> `as f32` (wav.rs:37)
    switch (bps) {
    case 8: return read_channel0(w, out, cap, n, [](const unsigned char *p) { return static_cast<float>(static_cast<int>(p[0]) - 128); });
    case 16: return read_channel0(w, out, cap, n, [](const unsigned char *p) { return static_cast<float>(static_cast<int16_t>(rd16(p))); });
    case 24: return read_channel0(w, out, cap, n, [](const unsigned char *p) {
        int v = p[0] | (p[1] << 8) | (p[2] << 16);
        if (v & 0x800000) v -= 0x1000000;
        return static_cast<float>(v);
    });
    default: return read_channel0(w, out, cap, n, [](const unsigned char *p) { return static_cast<float>(static_cast<int32_t>(rd32(p))); });
    }
}

extern "C" int apt_wav_load_pcm16(const char *path, int16_t *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate) {
    if (!n) return fail(APT_ERR_BAD_ARG, "null argument");
    WavFile w;
    APT_TRY(open_wav(path, w));
    if (sample_rate) *sample_rate = w.info.sample_rate;
    if (w.info.is_float || w.info.bits_per_sample != 16)
        return fail(APT_ERR_BAD_ARG, "'%s' does not hold 16-bit integer samples (use apt_wav_load)", path);
    return read_channel0(w, out, cap, n, [](const unsigned char *p) { return static_cast<int16_t>(rd16(p)); });
}

extern "C" int apt_wav_load_iq16(const char *path, int16_t *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate) {
    if (!n) return fail(APT_ERR_BAD_ARG, "null argument");
    WavFile w;
    APT_TRY(open_wav(path, w));
    if (w.info.is_float || w.info.bits_per_sample != 16 || w.info.channels != 2)
        return fail(APT_ERR_IO, "'%s' is not a 2-channel 16-bit PCM WAV (I/Q baseband)", path);
    if (sample_rate) *sample_rate = w.info.sample_rate;
    const uint64_t frames = w.info.frames;
    *n = frames;
    if (2 * frames > cap || (!out && frames)) return fail(APT_ERR_CAPACITY, "output needs room for %llu int16", (unsigned long long)(2 * frames));
    fseek(w.f, w.data_pos, SEEK_SET);
    std::vector<unsigned char> buf(4 * 65536);
    for (uint64_t done = 0; done < frames;) {
        const size_t want = static_cast<size_t>(frames - done < 65536 ? frames - done : 65536);
        if (fread(buf.data(), 4, want, w.f) != want) return fail(APT_ERR_IO, "WavOpen: truncated data chunk");
        for (size_t i = 0; i < 2 * want; ++i) out[2 * done + i] = static_cast<int16_t>(rd16(buf.data() + 2 * i));
        done += want;
    }
    return APT_OK;
}

extern "C" int apt_wav_write_i16(const char *path, const int16_t *samples, uint64_t n, uint32_t sample_rate) {
    if (!path || (!samples && n)) return fail(APT_ERR_BAD_ARG, "null argument");
    if (n * 2 > 0xFFFFFFFFull - 36) return fail(APT_ERR_BAD_ARG, "too many samples for a RIFF file");
    FILE *f = fopen(path, "wb");
    if (!f) return fail(APT_ERR_IO, "Io: cannot create '%s'", path);
    const uint32_t data = static_cast<uint32_t>(n * 2), riff = 36 + data, byte_rate = sample_rate * 2;
    unsigned char h[44] = {'R', 'I', 'F', 'F', 0, 0, 0, 0, 'W', 'A', 'V', 'E', 'f', 'm', 't', ' ', 16, 0, 0, 0, 1, 0, 1, 0};
    auto put32 = [&](int at, uint32_t v) { h[at] = v & 255; h[at + 1] = (v >> 8) & 255; h[at + 2] = (v >> 16) & 255; h[at + 3] = v >> 24; };
    put32(4, riff);
    put32(24, sample_rate);
    put32(28, byte_rate);
    h[32] = 2; h[33] = 0;       // block align
    h[34] = 16; h[35] = 0;      // bits per sample
    memcpy(h + 36, "data", 4);
    put32(40, data);
    const bool ok = fwrite(h, 1, 44, f) == 44 && (n == 0 || fwrite(samples, 2, n, f) == n);
    fclose(f);
    if (!ok) return fail(APT_ERR_IO, "Io: short write to '%s'", path);
    return APT_OK;
}
