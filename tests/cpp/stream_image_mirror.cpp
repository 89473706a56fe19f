// Compiled and run by tests/test_cpp_stream_image.py: the image output of noaa_apt::Stream (include/noaa_apt.hpp).
// Without a GPU it checks that the calls compile and that a stream fails loudly; with one it streams a synthetic pass and
// compares finish_image() with the whole-recording image and PNG.
#include <cmath>
#include <cstdio>
#include <string>

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
    if (!gpu) {
        if (apt_device_count() == 0) {
            try {
                Stream st(Rate::hz(48000), config::Settings());
                st.set_process_mode(&grey, 100);
                EXPECT(false);
            } catch (const err::Error &e) { EXPECT(e.kind == err::Kind::Cuda); }
        }
        std::printf("OK host\n");
        return 0;
    }
    const uint32_t rate = 48000;
    Signal x(rate * 14);
    for (size_t i = 0; i < x.size(); ++i) {
        const double t = double(i) / rate;
        const double line = std::fmod(t, 0.5);
        const double px = line < 0.0094 ? (std::fmod(line * 4160.0, 4.0) < 2.0 ? 0.1 : 1.0) : 0.5 + 0.3 * std::sin(40.0 * line);
        x[i] = float(std::lrint(20000.0 * px * std::sin(2.0 * M_PI * 2400.0 * t) + 150.0 * std::sin(12345.678 * i)));
    }
    Context ctx;
    const Signal whole = decode(ctx, config::Settings(), x, Rate::hz(rate), true);
    const std::vector<uint8_t> want_png = png::decode_png(ctx, config::Settings(), x, Rate::hz(rate), true, grey, png);
    const apt_settings s = config::Settings().to_c();
    uint64_t bound = 0, n_px = 0;
    err::check(apt_decode_len_bound(x.size(), rate, &s, &bound));
    std::vector<uint8_t> want_px(bound);
    apt_image_info want_info{};
    err::check(apt_decode_image(x.data(), APT_F32, x.size(), rate, &s, 1, &grey, want_px.data(), want_px.size(), &n_px, &want_info,
                                nullptr, nullptr));
    want_px.resize(n_px);

    Stream st(Rate::hz(rate), config::Settings(), true, 20000);
    const uint64_t base = st.info().device_bytes;
    st.set_process_mode(&grey, 64);
    for (int pass = 0; pass < 2; ++pass) {   // pixels, then PNG on the next pass
        if (pass == 1) st.set_png_mode(&png);
        Signal rows;
        for (size_t at = 0; at < x.size(); at += 33333) {
            const Signal r = st.push(x.data() + at, std::min<size_t>(33333, x.size() - at));
            rows.insert(rows.end(), r.begin(), r.end());
        }
        const Stream::Image im = st.finish_image();
        rows.insert(rows.end(), im.rows.begin(), im.rows.end());
        EXPECT(rows == whole);
        EXPECT(im.bytes == (pass == 0 ? want_px : want_png));
        EXPECT(im.info.rows == want_info.rows && im.info.low == want_info.low && im.info.high == want_info.high);
        st.reset();
    }
    st.set_process_mode(nullptr);
    EXPECT(st.info().device_bytes == base);
    std::printf("OK gpu %zu rows, %zu PNG bytes\n", whole.size() / 2080, want_png.size());
    return 0;
}
