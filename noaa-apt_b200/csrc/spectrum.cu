// Finding carriers (see spectrum.hpp): plan and tables, the per-device workspace, the chunked upload of the chosen
// segments, the launches, the host search and the APT test.
#include "spectrum.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>

#include "common.hpp"
#include "hostpool.hpp"
#include "iq.hpp"
#include "kernels_spectrum.cuh"

namespace aptb200 {

namespace {

constexpr double kTwoPi = 6.283185307179586;
constexpr double kBandHalfHz = 20000.0;     // +-17 kHz deviation plus the 2.4 kHz subcarrier and its sidebands
constexpr double kSuppressHz = 40000.0;
constexpr double kAptSeconds = 4.0;
constexpr uint32_t kAptNfft = 4096;
constexpr double kAptLoHz = 300.0, kAptHiHz = 4800.0;
constexpr float kAptThreshold = 0.5f;

}  // namespace

int make_spectrum(uint64_t n, uint32_t nfft, uint32_t max_segments, SpecPlan &p) {
    if (nfft < kSpecMinN || nfft > kSpecMaxN || (nfft & (nfft - 1)) != 0)
        return fail(APT_ERR_BAD_ARG, "nfft %u is not a power of two in [%u, %u]", nfft, kSpecMinN, kSpecMaxN);
    p.nfft = nfft;
    p.log2n = 0;
    while ((1u << p.log2n) < nfft) ++p.log2n;
    p.S = n / nfft;
    p.K = std::min<uint64_t>(p.S, max_segments ? max_segments : 2048);
    if (p.K == 0) return fail(APT_ERR_BAD_ARG, "%llu samples hold no segment of %u", (unsigned long long)n, nfft);
    p.win.resize(nfft);
    p.tw.resize(2 * static_cast<size_t>(nfft));
    for (uint32_t t = 0; t < nfft; ++t) {
        const double ang = kTwoPi * static_cast<double>(t) / static_cast<double>(nfft);
        p.win[t] = static_cast<float>(0.5 - 0.5 * std::cos(ang));
        p.tw[2 * t] = static_cast<float>(std::cos(ang));
        p.tw[2 * t + 1] = static_cast<float>(-std::sin(ang));
    }
    return APT_OK;
}

int make_search(const apt_carrier_search *cs, uint32_t iq_rate, SearchParams &sp) {
    sp = SearchParams{};
    if (cs) {
        if ((cs->lo_hz != 0 || cs->hi_hz != 0) && !(cs->lo_hz < cs->hi_hz))
            return fail(APT_ERR_BAD_ARG, "search window [%d, %d] Hz is inverted", cs->lo_hz, cs->hi_hz);
        sp.lo = cs->lo_hz;
        sp.hi = cs->hi_hz;
        sp.nfft = cs->nfft;
        sp.max_segments = cs->max_segments;
        if (cs->min_snr_db != 0.f) sp.min_snr_db = cs->min_snr_db;
    }
    if (sp.nfft == 0) {
        sp.nfft = kSpecMinN;
        while (sp.nfft < kSpecMaxN && static_cast<double>(iq_rate) / sp.nfft > 200.0) sp.nfft *= 2;
    }
    if (sp.max_segments == 0) sp.max_segments = 2048;
    return APT_OK;
}

int search_carriers(const float *psd, uint32_t nfft, uint32_t iq_rate, float cutout, const SearchParams &sp,
                    std::vector<apt_carrier> &out) {
    out.clear();
    const long N = nfft;
    const double bw = static_cast<double>(iq_rate) / nfft;
    auto freq = [&](long b) { return static_cast<double>(b - N / 2) * bw; };
    const bool whole = sp.lo == 0 && sp.hi == 0;
    long wa = -1, wb = -1;   // the window's bins: an interval
    for (long b = 0; b < N; ++b) {
        const double f = freq(b);
        if ((whole || (f >= sp.lo && f <= sp.hi)) && std::fabs(f) + cutout < iq_rate / 2.0) {
            if (wa < 0) wa = b;
            wb = b;
        }
    }
    if (wa < 0) return APT_OK;
    std::vector<double> v(psd + wa, psd + wb + 1);
    std::sort(v.begin(), v.end());
    const size_t m = v.size();
    const double floor = m % 2 ? v[m / 2] : (v[m / 2 - 1] + v[m / 2]) / 2.0;
    if (!(floor > 0.0)) return APT_OK;
    const long hb = static_cast<long>(static_cast<uint64_t>(kBandHalfHz) * nfft / iq_rate);
    std::vector<double> P(N + 1, 0.0);
    for (long i = 0; i < N; ++i) P[i + 1] = P[i] + static_cast<double>(psd[i]);
    std::vector<double> E(N);
    std::vector<long> nb(N);
    for (long b = 0; b < N; ++b) {
        const long a = std::max(0L, b - hb), c = std::min(N - 1, b + hb);
        E[b] = P[c + 1] - P[a];
        nb[b] = c - a + 1;
    }
    // a peak: the first bin of a run of equal E whose neighbours in the window are lower (the window's ends count as lower)
    struct Cand { long b; double snr; };
    std::vector<Cand> cands;
    for (long i = wa; i <= wb;) {
        long j = i;
        while (j < wb && E[j + 1] == E[i]) ++j;
        const bool left = i == wa || E[i - 1] < E[i];
        const bool right = j == wb || E[j + 1] < E[j];
        if (left && right) {
            const double snr = 10.0 * std::log10(E[i] / (floor * static_cast<double>(nb[i])));
            if (snr >= sp.min_snr_db) cands.push_back({i, snr});
        }
        i = j + 1;
    }
    std::stable_sort(cands.begin(), cands.end(), [&](const Cand &x, const Cand &y) { return E[x.b] > E[y.b]; });
    std::vector<Cand> kept;
    for (const Cand &c : cands) {
        bool near = false;
        for (const Cand &k : kept) near = near || std::fabs(static_cast<double>(c.b - k.b)) * bw <= kSuppressHz;
        if (!near) kept.push_back(c);
    }
    std::stable_sort(kept.begin(), kept.end(), [](const Cand &x, const Cand &y) { return x.snr > y.snr; });
    for (const Cand &c : kept) {
        double sw = 0.0, swf = 0.0;
        for (long b = std::max(0L, c.b - hb); b <= std::min(N - 1, c.b + hb); ++b) {
            const double w = static_cast<double>(psd[b]) - floor;
            if (w > 0.0) {
                sw += w;
                swf += w * freq(b);
            }
        }
        const double centre = sw > 0.0 ? swf / sw : freq(c.b);
        apt_carrier r{};
        r.offset_hz = static_cast<int32_t>(std::llround(centre));
        r.centre_hz = static_cast<float>(centre);
        r.snr_db = static_cast<float>(c.snr);
        out.push_back(r);
    }
    return APT_OK;
}

namespace {

// apt_iq_spectrum / apt_iq_find_carriers keep one workspace per device (a stream, the staging ring and copy threads,
// the segment window, the tables and sums, and the APT test's buffers) for the next call, one call per device at a
// time, as apt_png_encode keeps its encoder; apt_cache_clear frees them.
constexpr int kSpecDevices = 64;

struct SpecWork {
    std::mutex mu;
    cudaStream_t stream = nullptr;
    int sms = 1;
    std::unique_ptr<HostStager> stager;
    IqWindow seg;                                  // one chunk's packed segments (also the APT test's I/Q window)
    float2 *tw = nullptr;
    float *win = nullptr;
    u32 tab_n = 0;                                 // nfft of tw / win
    float *partial = nullptr, *psd = nullptr;
    u64 partial_cap = 0, psd_cap = 0;
    IqTables iqt;
    float *audio = nullptr;
    float2 *acf = nullptr;
    u64 audio_cap = 0, acf_cap = 0;
    void release() {
        if (stream) cudaStreamSynchronize(stream);
        stager.reset();
        seg.release();
        iqt.release();
        for (void *p : {static_cast<void *>(tw), static_cast<void *>(win), static_cast<void *>(partial),
                        static_cast<void *>(psd), static_cast<void *>(audio), static_cast<void *>(acf)})
            if (p) cudaFree(p);
        tw = nullptr;
        win = partial = psd = audio = nullptr;
        acf = nullptr;
        tab_n = 0;
        partial_cap = psd_cap = audio_cap = acf_cap = 0;
        if (stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
};
std::mutex g_spec_mu;
SpecWork *g_spec[kSpecDevices] = {};

template <typename T>
int grow(T *&p, u64 &cap, u64 n) {
    if (n <= cap) return APT_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    APT_CUDA(cudaMalloc(&p, std::max<u64>(n, 1) * sizeof(T)));
    cap = n;
    return APT_OK;
}

int require_gpu() {
    int count = 0;
    const cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    return APT_OK;
}

// The workspace of the current device, locked by the caller; created on first use.
int spec_work(SpecWork *&w) {
    APT_TRY(require_gpu());
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kSpecDevices) return fail(APT_ERR_CUDA, "device %d out of range", dev);
    std::lock_guard<std::mutex> lk(g_spec_mu);
    if (!g_spec[dev]) g_spec[dev] = new SpecWork();
    w = g_spec[dev];
    return APT_OK;
}

int spec_setup(SpecWork &w, const SpecPlan &p) {
    if (!w.stream) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&w.sms, cudaDevAttrMultiProcessorCount, dev);
        APT_CUDA(cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking));
    }
    if (w.tab_n != p.nfft) {
        APT_CUDA(cudaStreamSynchronize(w.stream));   // the previous launches have read the old tables
        if (w.tw) cudaFree(w.tw);
        if (w.win) cudaFree(w.win);
        w.tw = nullptr;
        w.win = nullptr;
        w.tab_n = 0;
        APT_CUDA(cudaMalloc(&w.tw, p.nfft * sizeof(float2)));
        APT_CUDA(cudaMalloc(&w.win, p.nfft * sizeof(float)));
        APT_CUDA(cudaMemcpyAsync(w.tw, p.tw.data(), p.nfft * sizeof(float2), cudaMemcpyHostToDevice, w.stream));
        APT_CUDA(cudaMemcpyAsync(w.win, p.win.data(), p.nfft * sizeof(float), cudaMemcpyHostToDevice, w.stream));
        APT_CUDA(cudaStreamSynchronize(w.stream));   // the host tables may go away with the plan
        w.tab_n = p.nfft;
    }
    const u64 slots = std::min<u64>(p.K, kSpecSlots);
    APT_TRY(grow(w.partial, w.partial_cap, slots * p.nfft));
    APT_CUDA(cudaMemsetAsync(w.partial, 0, slots * p.nfft * sizeof(float), w.stream));
    return APT_OK;
}

template <int FMT, int B4>
int launch_spec_b(SpecWork &w, const SpecPlan &p, const void *in, u64 k0, u64 k1) {
    SpecArgs a{};
    a.in = in;
    a.nfft = p.nfft;
    a.log2n = p.log2n;
    a.tw = w.tw;
    a.win = w.win;
    a.k0 = k0;
    a.k1 = k1;
    a.partial = w.partial;
    const size_t smem = static_cast<size_t>(p.nfft) * (sizeof(float2) + sizeof(float));
    APT_CUDA(cudaFuncSetAttribute(k_spectrum<FMT, B4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    const unsigned grid = static_cast<unsigned>(std::min<u64>(k1 - k0, kSpecSlots));
    k_spectrum<FMT, B4><<<grid, spec_threads(p.nfft), smem, w.stream>>>(a);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

template <int FMT>
int launch_spec(SpecWork &w, const SpecPlan &p, const void *in, u64 k0, u64 k1) {
    switch (p.nfft / 4 / spec_threads(p.nfft)) {
    case 1: return launch_spec_b<FMT, 1>(w, p, in, k0, k1);
    case 2: return launch_spec_b<FMT, 2>(w, p, in, k0, k1);
    case 4: return launch_spec_b<FMT, 4>(w, p, in, k0, k1);
    default: return launch_spec_b<FMT, 8>(w, p, in, k0, k1);
    }
}

int spec_launch(SpecWork &w, const SpecPlan &p, int format, const void *in, u64 k0, u64 k1) {
    if (k1 <= k0) return APT_OK;
    switch (format) {
    case APT_CU8: return launch_spec<APT_CU8>(w, p, in, k0, k1);
    case APT_CS16: return launch_spec<APT_CS16>(w, p, in, k0, k1);
    case APT_CF32: return launch_spec<APT_CF32>(w, p, in, k0, k1);
    default: return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    }
}

int spec_finish(SpecWork &w, const SpecPlan &p, float *d_psd) {
    const u32 slots = static_cast<u32>(std::min<u64>(p.K, kSpecSlots));
    k_spectrum_finish<<<(p.nfft + 255) / 256, 256, 0, w.stream>>>(w.partial, slots, p.nfft, static_cast<float>(p.K), d_psd);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

// The staging ring for an upload from `host`, made on first use: nullptr for pinned input, or when there is no ring
// (the upload is then a cudaMemcpyAsync).
HostStager *stager_for(SpecWork &w, const void *host) {
    if (!is_pageable(host)) return nullptr;
    if (!w.stager) {
        int dev = 0;
        cudaGetDevice(&dev);
        w.stager = make_stager(dev);
    }
    return w.stager.get();
}

// The spectrum of host I/Q into w.psd: the K segments uploaded in chunks of whole segments (APTB200_IQ_CHUNK samples at
// most, one segment at least), each chunk packed in w.seg and transformed by one launch.
int spec_host(SpecWork &w, const SpecPlan &p, const void *iq, int format) {
    const size_t sb = iq_sample_bytes(format);
    const size_t piece = static_cast<size_t>(p.nfft) * sb;
    const u64 per = std::min<u64>(p.K, std::max<u64>(iq_chunk_samples() / p.nfft, 1));
    APT_TRY(spec_setup(w, p));
    APT_TRY(grow(w.psd, w.psd_cap, p.nfft));
    APT_TRY(w.seg.reserve(per * piece));
    HostStager *const stager = stager_for(w, iq);
    const char *src = static_cast<const char *>(iq);
    std::vector<uint64_t> offs;
    for (u64 k0 = 0; k0 < p.K; k0 += per) {
        const u64 k1 = std::min<u64>(p.K, k0 + per);
        offs.resize(k1 - k0);
        for (u64 k = k0; k < k1; ++k) offs[k - k0] = p.start(k) * sb;
        if (stager) {
            APT_CUDA(stager->upload_pieces(w.seg.p, src, offs.data(), offs.size(), piece, w.stream));
        } else {
            // pinned input: one copy per run of adjacent segments
            for (u64 i = 0; i < offs.size();) {
                u64 j = i + 1;
                while (j < offs.size() && offs[j] == offs[j - 1] + piece) ++j;
                APT_CUDA(cudaMemcpyAsync(static_cast<char *>(w.seg.p) + i * piece, src + offs[i], (j - i) * piece,
                                         cudaMemcpyHostToDevice, w.stream));
                i = j;
            }
        }
        APT_TRY(spec_launch(w, p, format, w.seg.p, k0, k1));
    }
    return spec_finish(w, p, w.psd);
}

// apt_score of the carrier at `offset`: kAptSeconds of audio from the middle of the recording, demodulated by k_fm_demod
// with s's channel filter, its spectrum (kAptNfft bins of a complex copy with imaginary part 0), and the fraction of its
// power between kAptLoHz and kAptHiHz.
int apt_test(SpecWork &w, const void *iq, int format, uint64_t n, apt_iq_settings s, int32_t offset, float &score) {
    score = 0.f;
    s.offset_hz = offset;
    IqPlan ip;
    if (make_iq(s, ip) != APT_OK) return APT_OK;   // a centre too close to the band edge to demodulate: not APT
    const uint64_t na = ip.out_len(n);
    const uint64_t L = std::min<uint64_t>(na, static_cast<uint64_t>(kAptSeconds * s.audio_rate));
    if (L < kAptNfft) return APT_OK;
    const uint64_t m0 = (na - L) / 2, m1 = m0 + L;
    uint64_t xa, xb;
    ip.span(m0, m1, n, xa, xb);
    const size_t sb = iq_sample_bytes(format);
    APT_CUDA(cudaStreamSynchronize(w.stream));     // IqTables::upload replaces the tables the last launch read
    APT_TRY(w.iqt.upload(ip));
    APT_TRY(w.seg.reserve((xb - xa) * sb));
    APT_TRY(grow(w.audio, w.audio_cap, L));
    APT_TRY(grow(w.acf, w.acf_cap, L));
    const char *src = static_cast<const char *>(iq) + xa * sb;
    if (HostStager *stager = stager_for(w, iq)) APT_CUDA(stager->upload(w.seg.p, src, (xb - xa) * sb, w.stream));
    else APT_CUDA(cudaMemcpyAsync(w.seg.p, src, (xb - xa) * sb, cudaMemcpyHostToDevice, w.stream));
    const LaunchCtx c{w.stream, w.sms};
    APT_TRY(iq_launch(c, ip, w.iqt, static_cast<const char *>(w.seg.p) - xa * sb, xa, xb, format, m0, m1, w.audio - m0));
    APT_CUDA(cudaMemsetAsync(w.acf, 0, L * sizeof(float2), w.stream));
    APT_CUDA(cudaMemcpy2DAsync(w.acf, sizeof(float2), w.audio, sizeof(float), sizeof(float), L, cudaMemcpyDeviceToDevice,
                               w.stream));
    SpecPlan ap;
    APT_TRY(make_spectrum(L, kAptNfft, static_cast<uint32_t>(L / kAptNfft), ap));   // K = S: the segments are adjacent
    APT_TRY(spec_setup(w, ap));
    APT_TRY(grow(w.psd, w.psd_cap, ap.nfft));
    APT_TRY(spec_launch(w, ap, APT_CF32, w.acf, 0, ap.K));
    APT_TRY(spec_finish(w, ap, w.psd));
    std::vector<float> h(ap.nfft);
    APT_CUDA(cudaMemcpyAsync(h.data(), w.psd, ap.nfft * sizeof(float), cudaMemcpyDeviceToHost, w.stream));
    APT_CUDA(cudaStreamSynchronize(w.stream));
    double in = 0.0, all = 0.0;
    for (uint32_t b = 0; b < ap.nfft; ++b) {
        const double f = std::fabs((static_cast<double>(b) - ap.nfft / 2) * s.audio_rate / ap.nfft);
        all += h[b];
        if (f >= kAptLoHz && f <= kAptHiHz) in += h[b];
    }
    score = all > 0.0 ? static_cast<float>(in / all) : 0.f;
    return APT_OK;
}

}  // namespace

void spectrum_cache_clear() {
    int cur = 0;
    const bool have = cudaGetDevice(&cur) == cudaSuccess;
    std::lock_guard<std::mutex> lk(g_spec_mu);
    for (int d = 0; d < kSpecDevices; ++d) {
        if (!g_spec[d]) continue;
        std::lock_guard<std::mutex> lk2(g_spec[d]->mu);
        cudaSetDevice(d);
        g_spec[d]->release();
    }
    if (have) cudaSetDevice(cur);
}

}  // namespace aptb200

using namespace aptb200;

extern "C" int apt_iq_spectrum(const void *iq, int format, uint64_t n, uint32_t iq_rate, const apt_spectrum_settings *ss,
                               float *psd, uint64_t cap, uint32_t *nseg) {
    if (!iq || !ss || !psd || !nseg) return fail(APT_ERR_BAD_ARG, "null argument");
    *nseg = 0;
    if (!iq_sample_bytes(format)) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    if (iq_rate == 0) return fail(APT_ERR_BAD_ARG, "iq_rate is 0");
    SpecPlan p;
    APT_TRY(make_spectrum(n, ss->nfft, ss->max_segments, p));
    if (cap < p.nfft) return fail(APT_ERR_CAPACITY, "psd needs %u floats", p.nfft);
    SpecWork *w = nullptr;
    APT_TRY(spec_work(w));
    std::lock_guard<std::mutex> lk(w->mu);
    int st = spec_host(*w, p, iq, format);
    if (st == APT_OK) {
        const cudaError_t e = cudaMemcpyAsync(psd, w->psd, p.nfft * sizeof(float), cudaMemcpyDeviceToHost, w->stream);
        const cudaError_t e2 = cudaStreamSynchronize(w->stream);
        if (e != cudaSuccess || e2 != cudaSuccess)
            st = fail(APT_ERR_CUDA, "spectrum: %s", cudaGetErrorString(e != cudaSuccess ? e : e2));
    } else if (w->stream) {
        cudaStreamSynchronize(w->stream);
    }
    if (st == APT_OK) *nseg = static_cast<uint32_t>(p.K);
    return st;
}

extern "C" int apt_find_carriers_psd(const float *psd, uint32_t nfft, uint32_t iq_rate, float cutout,
                                     const apt_carrier_search *cs, apt_carrier *out, uint32_t cap, uint32_t *count) {
    if (!psd || !count || (!out && cap)) return fail(APT_ERR_BAD_ARG, "null argument");
    *count = 0;
    if (nfft < 2 || (nfft & (nfft - 1)) != 0 || iq_rate == 0 || !(cutout >= 0.f))
        return fail(APT_ERR_BAD_ARG, "nfft must be a power of two, iq_rate > 0 and cutout >= 0");
    SearchParams sp;
    APT_TRY(make_search(cs, iq_rate, sp));
    std::vector<apt_carrier> found;
    APT_TRY(search_carriers(psd, nfft, iq_rate, cutout, sp, found));
    *count = static_cast<uint32_t>(found.size());
    std::copy(found.begin(), found.begin() + std::min<size_t>(found.size(), cap), out);
    return found.size() > cap ? fail(APT_ERR_CAPACITY, "%zu carriers found", found.size()) : APT_OK;
}

extern "C" int apt_iq_find_carriers(const void *iq, int format, uint64_t n, const apt_iq_settings *s,
                                    const apt_carrier_search *cs, apt_carrier *out, uint32_t cap, uint32_t *count) {
    if (!iq || !s || !count || (!out && cap)) return fail(APT_ERR_BAD_ARG, "null argument");
    *count = 0;
    if (!iq_sample_bytes(format)) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    apt_iq_settings s0 = *s;
    s0.offset_hz = 0;
    {
        IqPlan ip;
        APT_TRY(make_iq(s0, ip));
    }
    SearchParams sp;
    APT_TRY(make_search(cs, s->iq_rate, sp));
    SpecPlan p;
    APT_TRY(make_spectrum(n, sp.nfft, sp.max_segments, p));
    SpecWork *w = nullptr;
    APT_TRY(spec_work(w));
    std::lock_guard<std::mutex> lk(w->mu);
    std::vector<apt_carrier> found;
    auto run = [&]() -> int {
        APT_TRY(spec_host(*w, p, iq, format));
        std::vector<float> psd(p.nfft);
        APT_CUDA(cudaMemcpyAsync(psd.data(), w->psd, p.nfft * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
        APT_CUDA(cudaStreamSynchronize(w->stream));
        APT_TRY(search_carriers(psd.data(), p.nfft, s->iq_rate, s->cutout, sp, found));
        for (size_t i = 0; i < found.size() && i < cap; ++i) {
            APT_TRY(apt_test(*w, iq, format, n, s0, found[i].offset_hz, found[i].apt_score));
            found[i].is_apt = found[i].apt_score >= kAptThreshold;
        }
        return APT_OK;
    };
    const int st = run();
    if (st != APT_OK) {
        if (w->stream) cudaStreamSynchronize(w->stream);
        return st;
    }
    *count = static_cast<uint32_t>(found.size());
    std::copy(found.begin(), found.begin() + std::min<size_t>(found.size(), cap), out);
    return found.size() > cap ? fail(APT_ERR_CAPACITY, "%zu carriers found", found.size()) : APT_OK;
}
