// Compiled and run by tests/test_cpp_watch.py: noaa_apt::passes::Watch (include/noaa_apt.hpp).  Without a GPU it checks
// that the calls compile and that argument and device errors come back as exceptions; with one it watches a synthetic feed
// in 1 s pushes and compares q, the passes and each pass's PNG file with noaa_apt::passes::Recording on the same samples.
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

int main(int argc, char **argv) {
    const bool gpu = argc > 1 && std::string(argv[1]) == "gpu";
    const apt_process_settings grey{APT_CONTRAST_MINMAX, 0.f, 1, nullptr, {0.f, 0.f, 0.f, 0.f}, 0};
    const apt_png_settings png = png::default_settings();
    apt_watch_settings ws{};
    ws.sync = 1;
    ws.search = apt_pass_search{0.f, 0.f, 5.f, 20.f};
    ws.ps = &grey;
    ws.png = &png;
    if (!gpu) {
        apt_watch_settings bad = ws;
        bad.ps = nullptr;   // PNG output without process settings
        try {
            passes::Watch w(Rate::hz(48000), nullptr, bad);
            EXPECT(false);
        } catch (const err::Error &e) { EXPECT(e.status == APT_ERR_BAD_ARG); }
        if (apt_device_count() == 0) {
            try {
                passes::Watch w(Rate::hz(48000), nullptr, ws);
                EXPECT(false);
            } catch (const err::Error &e) { EXPECT(e.kind == err::Kind::Cuda); }
        }
        std::printf("OK host\n");
        return 0;
    }
    // 8 s of noise, a 45 s pass, 8 s of noise
    const uint32_t rate = 48000;
    std::vector<int16_t> x(size_t(rate) * 61);
    uint32_t lcg = 12345;
    for (size_t i = 0; i < x.size(); ++i) {
        lcg = lcg * 1664525u + 1013904223u;
        const double noise = 2000.0 * (double(lcg >> 8) / double(1u << 24) - 0.5);
        const double t = double(i) / rate;
        double v = noise;
        if (t >= 8.0 && t < 53.0) {
            const double line = std::fmod(t, 0.5);
            const double px = line < 0.0094 ? (std::fmod(line * 4160.0, 4.0) < 2.0 ? 0.1 : 1.0) : 0.5 + 0.3 * std::sin(40.0 * line);
            v += 20000.0 * px * std::sin(2.0 * M_PI * 2400.0 * t);
        }
        x[i] = int16_t(std::lrint(std::max(-32768.0, std::min(32767.0, v))));
    }
    passes::Recording rec(x.data(), APT_PCM16, x.size(), Rate::hz(rate));
    const std::vector<float> want_q = rec.quality();
    const std::vector<apt_pass> want = rec.find_passes(ws.search);
    EXPECT(want.size() == 1);
    const std::vector<passes::Image> want_png = rec.decode_png(want, true, grey, png);

    std::vector<apt_pass_event> evs;
    std::vector<std::vector<uint8_t>> files;
    std::vector<int> statuses;
    passes::Watch w(Rate::hz(rate), [&](const apt_watch_event &e) {
        evs.push_back(e.ev);
        if (e.ev.kind == APT_PASS_LOS) {
            statuses.push_back(e.status);
            const uint8_t *d = static_cast<const uint8_t *>(e.data);
            files.emplace_back(d, d + e.bytes);
        }
    }, ws);
    const uint64_t bytes = w.info().device_bytes;
    std::vector<float> q;
    for (size_t at = 0; at < x.size(); at += rate) {
        const std::vector<float> part = w.push(x.data() + at, std::min<size_t>(rate, x.size() - at));
        q.insert(q.end(), part.begin(), part.end());
    }
    const std::vector<float> tail = w.finish();
    q.insert(q.end(), tail.begin(), tail.end());
    EXPECT(w.info().device_bytes == bytes);
    EXPECT(q.size() == want_q.size());
    for (size_t i = 0; i < q.size(); ++i) EXPECT(std::memcmp(&q[i], &want_q[i], sizeof(float)) == 0);
    EXPECT(evs.size() == 2 && evs[0].kind == APT_PASS_AOS && evs[1].kind == APT_PASS_LOS);
    const apt_pass &p = evs[1].pass;
    EXPECT(p.start == want[0].start && p.end == want[0].end && p.first_window == want[0].first_window &&
           p.windows == want[0].windows && p.mean_quality == want[0].mean_quality && p.peak_quality == want[0].peak_quality);
    EXPECT(statuses[0] == want_png[0].status && files[0] == want_png[0].png);
    std::printf("OK gpu %zu windows, %zu PNG bytes\n", q.size(), files[0].size());
    return 0;
}
