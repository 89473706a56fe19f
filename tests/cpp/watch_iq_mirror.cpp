// Compiled and run by tests/test_cpp_watch_iq.py: noaa_apt::passes::IqWatch (include/noaa_apt.hpp).  Without a GPU it checks
// that the calls compile and that argument and device errors come back as exceptions; with one it watches a synthetic
// two-carrier cu8 feed in 0.5 s pushes and compares each channel's q, events and PNG files with a noaa_apt::passes::Watch
// fed that channel's audio from apt_fm_demod_channels.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdio>
#include <string>
#include <vector>

#include "noaa_apt.hpp"

using namespace noaa_apt;

#define EXPECT(cond)                                                            \
    do {                                                                        \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #cond); return 1; } \
    } while (0)

struct Got {
    std::vector<int> kind;
    std::vector<apt_pass> pass;
    std::vector<std::vector<uint8_t>> files;
};

static void keep(Got &g, const apt_watch_event &e) {
    g.kind.push_back(e.ev.kind);
    g.pass.push_back(e.ev.pass);
    if (e.ev.kind == APT_PASS_LOS && e.status == APT_OK) {
        const uint8_t *d = static_cast<const uint8_t *>(e.data);
        g.files.emplace_back(d, d + e.bytes);
    }
}

int main(int argc, char **argv) {
    const bool gpu = argc > 1 && std::string(argv[1]) == "gpu";
    const apt_process_settings grey{APT_CONTRAST_MINMAX, 0.f, 1, nullptr, {0.f, 0.f, 0.f, 0.f}, 0};
    const apt_png_settings png = png::default_settings();
    apt_watch_settings ws{};
    ws.sync = 1;
    ws.search = apt_pass_search{0.f, 0.f, 5.f, 20.f};
    ws.ps = &grey;
    ws.png = &png;
    const uint32_t iq_rate = 250000;
    apt_iq_settings iq{};
    EXPECT(apt_iq_default_settings(iq_rate, 0, &iq) == APT_OK);
    const std::vector<int32_t> offsets{-60000, 60000};
    if (!gpu) {
        try {
            passes::IqWatch w(iq, {0, 0, 0, 0, 0, 0, 0, 0, 0}, nullptr, ws);   // nine channels
            EXPECT(false);
        } catch (const err::Error &e) { EXPECT(e.status == APT_ERR_BAD_ARG); }
        try {
            passes::IqWatch w(iq, {0, 110000}, nullptr, ws);                   // |offset| + cutout >= iq_rate / 2
            EXPECT(false);
        } catch (const err::Error &e) { EXPECT(e.status == APT_ERR_BAD_ARG); }
        if (apt_device_count() == 0) {
            try {
                passes::IqWatch w(iq, offsets, nullptr, ws);
                EXPECT(false);
            } catch (const err::Error &e) { EXPECT(e.kind == err::Kind::Cuda); }
        }
        std::printf("OK host\n");
        return 0;
    }
    // 61 s of cu8: channel 0 carries a pass from 8 to 53 s, channel 1 from 5 to 40 s
    const size_t n = size_t(iq_rate) * 61;
    std::vector<uint8_t> x(2 * n);
    uint32_t lcg = 12345;
    double ph[2] = {0.0, 0.0};
    const double on[2][2] = {{8.0, 53.0}, {5.0, 40.0}};
    for (size_t i = 0; i < n; ++i) {
        const double t = double(i) / iq_rate;
        double re = 0.0, im = 0.0;
        for (int c = 0; c < 2; ++c) {
            const double line = std::fmod(t + 0.1 * c, 0.5);
            const double px = line < 0.0094 ? (std::fmod(line * 4160.0, 4.0) < 2.0 ? 0.1 : 1.0) : 0.5 + 0.3 * std::sin(40.0 * line);
            const double audio = px * std::sin(2.0 * M_PI * 2400.0 * t);
            ph[c] += 2.0 * M_PI * (offsets[c] + 17000.0 * audio) / iq_rate;
            if (t >= on[c][0] && t < on[c][1]) {
                re += 0.5 * std::cos(ph[c]);
                im += 0.5 * std::sin(ph[c]);
            }
        }
        for (int k = 0; k < 2; ++k) {
            lcg = lcg * 1664525u + 1013904223u;
            const double noise = 0.03 * (double(lcg >> 8) / double(1u << 24) - 0.5);
            const double v = 100.0 * ((k == 0 ? re : im) + noise) + 127.5;
            x[2 * i + k] = uint8_t(std::lrint(std::max(0.0, std::min(255.0, v))));
        }
    }
    // each channel's audio, and an audio Watch on it
    uint64_t na = 0;
    EXPECT(apt_fm_demod_len(n, &iq, &na) == APT_OK);
    std::vector<std::vector<float>> audio(2, std::vector<float>(na));
    float *outs[2] = {audio[0].data(), audio[1].data()};
    uint64_t got = 0;
    EXPECT(apt_fm_demod_channels(x.data(), APT_CU8, n, &iq, offsets.data(), 2, outs, na, &got) == APT_OK && got == na);
    Got want[2], have[2];
    std::vector<float> want_q[2];
    for (int c = 0; c < 2; ++c) {
        passes::Watch w(Rate::hz(iq.audio_rate), [&](const apt_watch_event &e) { keep(want[c], e); }, ws);
        want_q[c] = w.push(audio[c].data(), audio[c].size());
        const std::vector<float> tail = w.finish();
        want_q[c].insert(want_q[c].end(), tail.begin(), tail.end());
    }
    passes::IqWatch w(iq, offsets, [&](int c, const apt_watch_event &e) { keep(have[c], e); }, ws);
    const uint64_t bytes = w.info(0).device_bytes;
    std::vector<float> q[2];
    for (size_t at = 0; at < n; at += iq_rate / 2) {
        const auto part = w.push(x.data() + 2 * at, APT_CU8, std::min<size_t>(iq_rate / 2, n - at));
        for (int c = 0; c < 2; ++c) q[c].insert(q[c].end(), part[c].begin(), part[c].end());
    }
    const auto tail = w.finish();
    EXPECT(w.info(1).device_bytes == bytes && w.info(1).samples_in == n);
    size_t files = 0;
    for (int c = 0; c < 2; ++c) {
        q[c].insert(q[c].end(), tail[c].begin(), tail[c].end());
        EXPECT(q[c].size() == want_q[c].size());
        for (size_t i = 0; i < q[c].size(); ++i) EXPECT(std::memcmp(&q[c][i], &want_q[c][i], sizeof(float)) == 0);
        EXPECT(have[c].kind == want[c].kind && have[c].kind.size() == 2 && have[c].kind[1] == APT_PASS_LOS);
        for (size_t k = 0; k < have[c].pass.size(); ++k)
            EXPECT(std::memcmp(&have[c].pass[k], &want[c].pass[k], sizeof(apt_pass)) == 0);
        EXPECT(have[c].files == want[c].files && have[c].files.size() == 1);
        files += have[c].files.size();
    }
    std::printf("OK gpu %zu + %zu windows, %zu PNG files\n", q[0].size(), q[1].size(), files);
    return 0;
}
