// The I/Q stage (see iq.hpp): plan, tables, launch, the chunked host upload and the stage entry points.
#include "iq.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "common.hpp"
#include "filters_host.hpp"
#include "hostpool.hpp"
#include "kernels_iq.cuh"

namespace aptb200 {

namespace {

constexpr double kTwoPi = 6.283185307179586;
constexpr size_t kSmemMax = 232448;       // dynamic shared memory of one CTA on sm_90
constexpr size_t kSmemTwoPerSm = 115712;  // two CTAs per SM (228 KB per SM, 1 KB reserved per CTA)
constexpr uint32_t kMaxTaps = 8191;

size_t tile_smem(u32 D, u32 qpad, u32 tz, u32 &lp16, u32 &ps) {
    const u32 gl = tz / kIqR, parts = kIqThreads / gl;
    lp16 = (tz + qpad - 1 + 15) / 16;
    ps = 16 * lp16 + 1;   // odd plane stride: the staging stores of consecutive planes fall in different banks
    const size_t planes = static_cast<size_t>(D) * ps + 16;
    const size_t reduce = static_cast<size_t>(parts) * (tz + tz / 16) + tz;
    return std::max(planes, reduce) * sizeof(float2);
}

}  // namespace

size_t iq_sample_bytes(int format) {
    switch (format) {
    case APT_CU8: return 2;
    case APT_CS16: return 4;
    case APT_CF32: return 8;
    default: return 0;
    }
}

void IqPlan::span(uint64_t m0, uint64_t m1, uint64_t n, uint64_t &xa, uint64_t &xb) const {
    const uint64_t first = m0 == 0 ? 0 : (m0 - 1) * D;   // z[m0 - 1] reads back to (m0 - 1) D - (N - 1)
    xa = first > h.size() - 1 ? first - (h.size() - 1) : 0;
    xb = std::min<uint64_t>(n, m1 == 0 ? 0 : (m1 - 1) * D + 1);
}

int make_iq(const apt_iq_settings &s, IqPlan &p) {
    if (s.iq_rate == 0 || s.audio_rate == 0 || s.iq_rate % s.audio_rate != 0)
        return fail(APT_ERR_BAD_ARG, "audio_rate %u does not divide iq_rate %u", s.audio_rate, s.iq_rate);
    if (!(s.cutout > 0.f) || !(s.delta_freq > 0.f) || !(s.atten > 8.f))
        return fail(APT_ERR_BAD_ARG, "channel filter needs cutout > 0, delta_freq > 0 and atten > 8 dB");
    if (!(static_cast<double>(s.cutout) < s.audio_rate / 2.0))
        return fail(APT_ERR_BAD_ARG, "cutout %g Hz is not below audio_rate / 2", static_cast<double>(s.cutout));
    if (!(std::fabs(static_cast<double>(s.offset_hz)) + s.cutout < s.iq_rate / 2.0))
        return fail(APT_ERR_BAD_ARG, "|offset_hz| + cutout is not below iq_rate / 2");
    p.s = s;
    p.D = s.iq_rate / s.audio_rate;
    const apt_filter lf{APT_FILTER_LOWPASS, Freq::hz(s.cutout, s.iq_rate).get_pi_rad(), s.atten,
                        Freq::hz(s.delta_freq, s.iq_rate).get_pi_rad()};
    // the Kaiser length first (filters.rs:164-167, as kaiser() computes it), so a tiny delta_freq is refused cheaply
    const float flen = std::ceil((s.atten - 8.f) / (2.285f * Freq::pi_rad(lf.delta_w_pi).get_rad()));
    if (!(flen >= 0.f) || flen + 2.f > static_cast<float>(kMaxTaps) + 1.f)
        return fail(APT_ERR_BAD_ARG, "channel filter has more than %u taps", kMaxTaps);
    if (design(lf, p.h) != APT_OK || p.h.size() > kMaxTaps)
        return fail(APT_ERR_BAD_ARG, "channel filter has more than %u taps", kMaxTaps);
    const u32 N = static_cast<u32>(p.h.size());
    const u32 q = (N + p.D - 1) / p.D;
    p.qpad = (q + kIqR - 1) / kIqR * kIqR;
    p.hp.assign(static_cast<size_t>(p.D) * p.qpad, 0.f);
    for (u32 r = 0; r < p.D; ++r)
        for (u32 k = 0; k < p.qpad; ++k)
            if (static_cast<uint64_t>(k) * p.D + r < N) p.hp[static_cast<size_t>(r) * p.qpad + k] = p.h[static_cast<size_t>(k) * p.D + r];

    p.f = static_cast<uint64_t>(((static_cast<int64_t>(s.offset_hz) % s.iq_rate) + s.iq_rate) % s.iq_rate);
    p.W.resize(2 * kIqBlock);
    for (u32 t = 0; t < kIqBlock; ++t) {
        const uint64_t v = (static_cast<uint64_t>(t) * p.f) % s.iq_rate;
        const double ang = -kTwoPi * static_cast<double>(v) / static_cast<double>(s.iq_rate);
        p.W[2 * t] = static_cast<float>(std::cos(ang));
        p.W[2 * t + 1] = static_cast<float>(std::sin(ang));
    }
    p.scale = static_cast<float>(s.audio_rate / kTwoPi);

    // the largest tile that lets two CTAs share an SM, else the largest that fits one.  APTB200_IQ_TILE picks a tile for
    // experiments; one that does not fit is ignored, so the switch never changes which settings are valid.
    p.tz = 0;
    u32 forced = 0;
    if (const char *e = getenv("APTB200_IQ_TILE")) forced = static_cast<u32>(strtoul(e, nullptr, 10));
    if (forced >= kIqR && forced <= 512 && (forced & (forced - 1)) == 0 &&
        tile_smem(p.D, p.qpad, forced, p.lp16, p.ps) <= kSmemMax) {
        p.tz = forced;
        p.smem = tile_smem(p.D, p.qpad, forced, p.lp16, p.ps);
    }
    for (size_t limit : {kSmemTwoPerSm, kSmemMax}) {
        for (u32 tz = 512; tz >= kIqR && !p.tz; tz /= 2) {
            const size_t b = tile_smem(p.D, p.qpad, tz, p.lp16, p.ps);
            if (b <= limit) {
                p.tz = tz;
                p.smem = b;
            }
        }
        if (p.tz) break;
    }
    if (!p.tz) return fail(APT_ERR_BAD_ARG, "iq_rate / audio_rate = %u is too large for the on-chip tile", p.D);
    tile_smem(p.D, p.qpad, p.tz, p.lp16, p.ps);
    return APT_OK;
}

int iq_default_settings(uint32_t iq_rate, int32_t offset_hz, apt_iq_settings &s) {
    s = apt_iq_settings{};
    s.iq_rate = iq_rate;
    s.offset_hz = offset_hz;
    s.cutout = 22000.f;
    s.delta_freq = 8000.f;
    s.atten = 40.f;
    if (iq_rate < 48000) return fail(APT_ERR_BAD_ARG, "iq_rate %u is below 48 kHz", iq_rate);
    // the smallest iq_rate / D >= 48 kHz: the largest divisor D with iq_rate / D >= 48000
    for (uint32_t D = iq_rate / 48000; D >= 1; --D)
        if (iq_rate % D == 0) {
            s.audio_rate = iq_rate / D;
            break;
        }
    IqPlan p;
    return make_iq(s, p);
}

int IqTables::upload(const IqPlan &p, bool taps) {
    release();
    if (taps) {
        APT_CUDA(cudaMalloc(&hp, p.hp.size() * sizeof(float)));
        APT_CUDA(cudaMemcpy(hp, p.hp.data(), p.hp.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    APT_CUDA(cudaMalloc(&W, p.W.size() * sizeof(float)));
    APT_CUDA(cudaMemcpy(W, p.W.data(), p.W.size() * sizeof(float), cudaMemcpyHostToDevice));
    return APT_OK;
}

void IqTables::release() {
    if (hp) cudaFree(hp);
    if (W) cudaFree(W);
    hp = W = nullptr;
}

namespace {
template <int FMT>
int launch_fm(const LaunchCtx &c, const IqArgs &a, size_t smem, unsigned grid) {
    // the attribute is per device: set it on the current one at every launch (a host-side call, no device work)
    APT_CUDA(cudaFuncSetAttribute(k_fm_demod<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    k_fm_demod<FMT><<<grid, kIqThreads, smem, c.stream>>>(a);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

// The launch data every channel of plan p shares, and the tiles outputs [m0, m1) take.
int iq_args(const IqPlan &p, const IqTables &t, const void *in, uint64_t w_lo, uint64_t w_hi, uint64_t m0, uint64_t m1,
            IqArgs &a, unsigned &grid) {
    a = IqArgs{};
    a.in = in;
    a.w_lo = w_lo;
    a.w_hi = w_hi;
    a.hp = t.hp;
    a.D = p.D;
    a.qpad = p.qpad;
    a.fs = p.s.iq_rate;
    a.scale = p.scale;
    a.m_begin = m0;
    a.m_end = m1;
    a.tz = p.tz;
    a.lp16 = p.lp16;
    a.ps = p.ps;
    const uint64_t g = (m1 - m0 + p.tz - 2) / (p.tz - 1);
    if (g > 0x7fffffffull) return fail(APT_ERR_BAD_ARG, "too many audio samples for one launch");
    grid = static_cast<unsigned>(g);
    return APT_OK;
}

template <int FMT>
int launch_fm_channels(const LaunchCtx &c, const IqArgs &a, const IqChannels &ch, int count, size_t smem, unsigned grid) {
    APT_CUDA(cudaFuncSetAttribute(k_fm_demod_channels<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    k_fm_demod_channels<FMT><<<dim3(grid, static_cast<unsigned>(count)), kIqThreads, smem, c.stream>>>(a, ch);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}
}  // namespace

int iq_launch(const LaunchCtx &c, const IqPlan &p, const IqTables &t, const void *in, uint64_t w_lo, uint64_t w_hi,
              int format, uint64_t m0, uint64_t m1, float *out) {
    if (m1 <= m0) return APT_OK;
    IqArgs a;
    unsigned grid = 0;
    APT_TRY(iq_args(p, t, in, w_lo, w_hi, m0, m1, a, grid));
    a.W = reinterpret_cast<const float2 *>(t.W);
    a.f = p.f;
    a.mix = p.f != 0;
    a.out = out;
    switch (format) {
    case APT_CU8: return launch_fm<APT_CU8>(c, a, p.smem, grid);
    case APT_CS16: return launch_fm<APT_CS16>(c, a, p.smem, grid);
    case APT_CF32: return launch_fm<APT_CF32>(c, a, p.smem, grid);
    default: return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    }
}

int iq_launch_channels(const LaunchCtx &c, const IqPlan *const *plans, const IqTables *const *tables, int count,
                       const void *in, uint64_t w_lo, uint64_t w_hi, int format, uint64_t m0, uint64_t m1,
                       float *const *outs) {
    if (count < 1 || count > kIqMaxChannels) return fail(APT_ERR_BAD_ARG, "channel count %d outside 1..%d", count, kIqMaxChannels);
    if (m1 <= m0) return APT_OK;
    const IqPlan &p = *plans[0];
    IqArgs a;
    unsigned grid = 0;
    APT_TRY(iq_args(p, *tables[0], in, w_lo, w_hi, m0, m1, a, grid));
    IqChannels ch{};
    for (int k = 0; k < count; ++k) {
        ch.W[k] = reinterpret_cast<const float2 *>(tables[k]->W);
        ch.out[k] = outs[k];
        ch.f[k] = plans[k]->f;
        ch.mix[k] = plans[k]->f != 0;
    }
    switch (format) {
    case APT_CU8: return launch_fm_channels<APT_CU8>(c, a, ch, count, p.smem, grid);
    case APT_CS16: return launch_fm_channels<APT_CS16>(c, a, ch, count, p.smem, grid);
    case APT_CF32: return launch_fm_channels<APT_CF32>(c, a, ch, count, p.smem, grid);
    default: return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    }
}

int iq_to_cf32(const LaunchCtx &c, const void *in, int format, uint64_t n, float *out) {
    if (n == 0) return APT_OK;
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(c.sm_count) * 8));
    float2 *o = reinterpret_cast<float2 *>(out);
    switch (format) {
    case APT_CU8: k_iq_to_cf32<APT_CU8><<<grid, 256, 0, c.stream>>>(in, n, o); break;
    case APT_CS16: k_iq_to_cf32<APT_CS16><<<grid, 256, 0, c.stream>>>(in, n, o); break;
    case APT_CF32: k_iq_to_cf32<APT_CF32><<<grid, 256, 0, c.stream>>>(in, n, o); break;
    default: return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    }
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

uint64_t iq_chunk_samples() {
    uint64_t chunk = 32ull << 20;
    if (const char *e = getenv("APTB200_IQ_CHUNK")) chunk = std::max<uint64_t>(strtoull(e, nullptr, 10), 1);
    return chunk;
}

int IqFeed::alloc(const IqPlan &q, uint64_t max_push) {
    release();
    cap = window(q, max_push);
    APT_CUDA(cudaMalloc(&d_iq, cap * 2 * sizeof(float)));
    APT_CUDA(cudaMalloc(&d_raw, max_push * 8));
    return APT_OK;
}

void IqFeed::release() {
    if (d_iq) cudaFree(d_iq);
    if (d_raw) cudaFree(d_raw);
    d_iq = nullptr;
    d_raw = nullptr;
    cap = in = base = 0;
}

int IqFeed::push(const LaunchCtx &c, const IqPlan &q, uint64_t m_next, const void *host, int format, uint64_t n) {
    // the window keeps what audio output m_next reads; its tail moves to the front when that does not overlap
    uint64_t xa, xb;
    q.span(m_next, m_next + 1, ~0ull, xa, xb);
    if (xa > base && in - xa <= xa - base) {
        if (in > xa)
            APT_CUDA(cudaMemcpyAsync(d_iq, d_iq + 2 * (xa - base), (in - xa) * 2 * sizeof(float), cudaMemcpyDeviceToDevice,
                                     c.stream));
        base = xa;
    }
    if (in - base + n > cap) return fail(APT_ERR_BAD_ARG, "internal: I/Q window overflow");
    APT_CUDA(cudaMemcpyAsync(d_raw, host, n * iq_sample_bytes(format), cudaMemcpyHostToDevice, c.stream));
    APT_TRY(iq_to_cf32(c, d_raw, format, n, d_iq + 2 * (in - base)));
    in += n;
    return APT_OK;
}

int IqWindow::reserve(uint64_t bytes) {
    if (bytes <= cap) return APT_OK;
    release();
    APT_CUDA(cudaMalloc(&p, std::max<uint64_t>(bytes, 16)));
    cap = bytes;
    return APT_OK;
}

void IqWindow::release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
}

int iq_demod_host(const LaunchCtx &c, const IqPlan &p, const IqTables &t, const void *iq, int format, uint64_t n,
                  IqWindow &win, HostStager *stager, float *d_audio, KernelHook *hook) {
    const IqPlan *pp = &p;
    const IqTables *tp = &t;
    return iq_demod_host_multi(c, &pp, &tp, &d_audio, 1, iq, format, n, win, stager, hook);
}

int iq_demod_host_multi(const LaunchCtx &c, const IqPlan *const *plans, const IqTables *const *tables,
                        float *const *d_audio, int count, const void *iq, int format, uint64_t n, IqWindow &win,
                        HostStager *stager, KernelHook *hook) {
    const size_t sb = iq_sample_bytes(format);
    if (!sb) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    const IqPlan &p = *plans[0];   // D and the tap count, hence the spans, are the same for every channel
    const uint64_t nout = p.out_len(n);
    const uint64_t chunk = std::min<uint64_t>(iq_chunk_samples(), std::max<uint64_t>(n, 1));
    // one chunk's window: its new samples and the halo in front of its first output
    APT_TRY(win.reserve((std::min<uint64_t>(n, chunk + p.h.size() + 2ull * p.D)) * sb));
    const char *src = static_cast<const char *>(iq);
    uint64_t m_done = 0;
    for (uint64_t c_hi = std::min(n, chunk); m_done < nout; c_hi = std::min(n, c_hi + chunk)) {
        const uint64_t m_b = c_hi == n ? nout : std::min(nout, (c_hi - 1) / p.D + 1);
        if (m_b == m_done) continue;
        uint64_t xa, xb;
        p.span(m_done, m_b, n, xa, xb);
        const size_t bytes = (c_hi - xa) * sb;
        if (stager) APT_CUDA(stager->upload(win.p, src + xa * sb, bytes, c.stream));
        else APT_CUDA(cudaMemcpyAsync(win.p, src + xa * sb, bytes, cudaMemcpyHostToDevice, c.stream));
        for (int k = 0; k < count; k += kIqMaxChannels) {   // one launch per chunk up to 8 channels
            KernelSlot s(hook, "fm_demod");
            APT_TRY(iq_launch_channels(c, plans + k, tables + k, std::min(count - k, kIqMaxChannels),
                                       static_cast<const char *>(win.p) - xa * sb, xa, c_hi, format, m_done, m_b, d_audio + k));
        }
        m_done = m_b;
    }
    return APT_OK;
}

}  // namespace aptb200

using namespace aptb200;

extern "C" int apt_iq_default_settings(uint32_t iq_rate, int32_t offset_hz, apt_iq_settings *s) {
    if (!s) return fail(APT_ERR_BAD_ARG, "null argument");
    return iq_default_settings(iq_rate, offset_hz, *s);
}

extern "C" int apt_fm_demod_len(uint64_t n, const apt_iq_settings *s, uint64_t *nout) {
    if (!s || !nout) return fail(APT_ERR_BAD_ARG, "null argument");
    IqPlan p;
    APT_TRY(make_iq(*s, p));
    *nout = p.out_len(n);
    return APT_OK;
}

extern "C" int apt_fm_demod(const void *iq, int format, uint64_t n, const apt_iq_settings *s, float *out, uint64_t cap,
                            uint64_t *nout) {
    if (!s || !nout || (!iq && n)) return fail(APT_ERR_BAD_ARG, "null argument");
    *nout = 0;
    if (!iq_sample_bytes(format)) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    IqPlan p;
    APT_TRY(make_iq(*s, p));
    const uint64_t ny = p.out_len(n);
    *nout = ny;
    if (ny > cap || (!out && ny)) return fail(APT_ERR_CAPACITY, "output needs %llu floats", (unsigned long long)ny);
    if (ny == 0) return APT_OK;
    int count = 0, dev = 0, sms = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device; this library has no CPU fallback");
    }
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const LaunchCtx c{nullptr, std::max(sms, 1)};
    IqTables t;
    IqWindow win;
    float *d_audio = nullptr;
    struct Free {
        float *&p;
        ~Free() { if (p) cudaFree(p); }
    } free_audio{d_audio};
    APT_TRY(t.upload(p));
    APT_CUDA(cudaMalloc(&d_audio, ny * sizeof(float)));
    APT_TRY(iq_demod_host(c, p, t, iq, format, n, win, nullptr, d_audio, nullptr));
    APT_CUDA(cudaMemcpy(out, d_audio, ny * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}

extern "C" int apt_fm_demod_channels(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const int32_t *offsets,
                                     int count, float *const *outs, uint64_t cap, uint64_t *nout) {
    if (!s || !nout || !offsets || !outs || (!iq && n)) return fail(APT_ERR_BAD_ARG, "null argument");
    *nout = 0;
    if (count < 1 || count > kIqMaxChannels) return fail(APT_ERR_BAD_ARG, "channel count %d outside 1..%d", count, kIqMaxChannels);
    if (!iq_sample_bytes(format)) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    IqPlan p[kIqMaxChannels];
    const IqPlan *pp[kIqMaxChannels];
    for (int k = 0; k < count; ++k) {
        apt_iq_settings sk = *s;
        sk.offset_hz = offsets[k];
        APT_TRY(make_iq(sk, p[k]));
        pp[k] = &p[k];
    }
    const uint64_t ny = p[0].out_len(n);
    *nout = ny;
    if (ny > cap) return fail(APT_ERR_CAPACITY, "output needs %llu floats per channel", (unsigned long long)ny);
    for (int k = 0; k < count && ny; ++k)
        if (!outs[k]) return fail(APT_ERR_BAD_ARG, "null output of channel %d", k);
    if (ny == 0) return APT_OK;
    int ndev = 0, dev = 0, sms = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device; this library has no CPU fallback");
    }
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const LaunchCtx c{nullptr, std::max(sms, 1)};
    IqTables t[kIqMaxChannels];
    const IqTables *tp[kIqMaxChannels];
    IqWindow win;
    float *d_audio = nullptr;
    struct Free {
        float *&p;
        ~Free() { if (p) cudaFree(p); }
    } free_audio{d_audio};
    float *d_out[kIqMaxChannels];
    for (int k = 0; k < count; ++k) {
        APT_TRY(t[k].upload(p[k]));
        tp[k] = &t[k];
    }
    APT_CUDA(cudaMalloc(&d_audio, static_cast<size_t>(count) * ny * sizeof(float)));
    for (int k = 0; k < count; ++k) d_out[k] = d_audio + static_cast<size_t>(k) * ny;
    APT_TRY(iq_demod_host_multi(c, pp, tp, d_out, count, iq, format, n, win, nullptr, nullptr));
    for (int k = 0; k < count; ++k) APT_CUDA(cudaMemcpy(outs[k], d_out[k], ny * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}
