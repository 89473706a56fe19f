// Decoder object and kernel sequence of decode::decode (decode.rs:43-162).
#include "decoder.hpp"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "common.hpp"
#include "launch.hpp"

namespace aptb200 {

std::string &last_error_slot() {
    static thread_local std::string slot;
    return slot;
}

int fail(int status, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    last_error_slot() = buf;
    return status;
}

// ------------------------------------------------------------------------------------- plan

int make_plan(uint32_t input_rate, const apt_settings &s, Plan &p) {
    p = Plan{};
    p.input_rate = input_rate;
    p.st = s;
    if (s.work_rate > UINT32_MAX / kPxPerRow)   // PX_PER_ROW * work_rate overflows u32 (decode.rs:55)
        return fail(APT_ERR_BAD_ARG, "work_rate %u is too large", s.work_rate);

    // decode.rs:65-77 -> dsp::resample_with_filter (dsp.rs:62-98)
    Ratio first{};
    int st = resample_ratio(input_rate, s.work_rate, first);
    if (st == APT_ERR_RESAMPLE_TO_ZERO) return fail(st, "Can't resample to 0Hz");
    if (st == APT_ERR_RATE_OVERFLOW)
        return fail(st, "Can't resample, looks like the sample rates do not have a big divisor in common. "
                        "input_rate: %u, output_rate: %u, l: %u, m: %u",
                    input_rate, s.work_rate, first.l, first.m);
    if (st != APT_OK) return fail(st, "invalid input rate %u", input_rate);

    apt_filter rf{APT_FILTER_LOWPASS_DC, Freq::hz(s.resample_cutout, input_rate).get_pi_rad(), s.resample_atten,
                  Freq::hz(s.resample_delta_freq, input_rate).get_pi_rad()};
    if (first.l > 1) resample_filter(rf, input_rate, input_rate * first.l);   // dsp.rs:93
    std::vector<float> h;
    st = design(rf, h);
    if (st != APT_OK) return fail(st, "resampling filter cannot be designed (atten %g, delta_w %g)",
                                  (double)rf.atten, (double)rf.delta_w_pi);
    p.front = make_front(first, std::move(h));

    // decode.rs:95-100
    const float cut = static_cast<float>(kFinalRate) / static_cast<float>(s.work_rate);
    apt_filter lf{APT_FILTER_LOWPASS, cut, s.demodulation_atten, cut / 5.f};
    st = design(lf, p.lp);
    if (st != APT_OK) return fail(st, "demodulation filter cannot be designed (atten %g)", (double)lf.atten);

    // decode.rs:89 + dsp.rs:360-363
    const float phi = 2.f * Freq::hz(static_cast<float>(kCarrierHz), s.work_rate).get_rad();
    p.cosphi2 = std::cos(phi) * 2.f;
    p.sinphi = std::sin(phi);

    p.row = kPxPerRow * s.work_rate / kFinalRate;                       // decode.rs:55
    if (p.row == 0)   // work_rate < 2: the reference divides by zero (decode.rs:141); a status is the safe equivalent
        return fail(APT_ERR_BAD_ARG, "work_rate %u is too low: zero samples per image row", s.work_rate);
    p.dist = static_cast<uint32_t>(static_cast<uint64_t>(p.row) * 8 / 10);   // decode.rs:216
    p.work_multiple = s.work_rate % kFinalRate == 0;
    p.dec = s.work_rate / kFinalRate;
    if (p.work_multiple) sync_frame(s.work_rate, p.guard);
    // final stage ratio, decode.rs:158-159 (errors surface when the stage runs)
    p.last = Ratio{0, 0};
    resample_ratio(s.work_rate, kFinalRate, p.last);
    return APT_OK;
}

uint64_t plan_out_bound(const Plan &p, uint64_t n) {
    const uint64_t nw = p.front.work_len(n);
    if (p.row == 0) return 0;
    const uint64_t rows = nw / p.row;
    if (p.work_multiple) return rows * kPxPerRow;
    return polyphase_len(rows * p.row, p.last.l, p.last.m, 1);
}

// ---------------------------------------------------------------------------------- helpers

int prof_begin(apt_decoder *d, const char *name) {
    d->launches++;
    if (!d->profiling) return -1;
    const int slot = d->ev_used++;
    if (slot >= static_cast<int>(d->ev_begin.size())) {
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        d->ev_begin.push_back(a);
        d->ev_end.push_back(b);
        d->kernel_names.emplace_back();
    }
    d->kernel_names[slot] = name;
    cudaEventRecord(d->ev_begin[slot], d->stream);
    return slot;
}

void prof_end(apt_decoder *d, int slot) {
    if (slot >= 0) cudaEventRecord(d->ev_end[slot], d->stream);
}

void DecoderHook::extra(int kernels) { d->launches += static_cast<uint64_t>(kernels); }

namespace {

struct Prof : DecoderHook {   // a slot around a scope
    Prof(apt_decoder *dec, const char *name) : DecoderHook(dec) { begin(name); }
    ~Prof() { end(); }
};

}  // namespace

int ensure_conv(apt_decoder *d, uint64_t need, uint64_t alloc) {
    if (d->conv_cap >= need) return APT_OK;
    if (d->d_conv) APT_CUDA(cudaFree(d->d_conv));
    d->d_conv = nullptr;
    d->conv_cap = 0;
    APT_CUDA(cudaMalloc(&d->d_conv, alloc * sizeof(float)));
    d->conv_cap = alloc;
    return APT_OK;
}

// Long host recording: upload in chunks (with the filter-length overlap each chunk needs) on the copy stream while
// the previous chunk is resampled on the compute stream.  Only a polyphase first stage is chunked.
static int enqueue_front_chunked(apt_decoder *d, const void *host, int format, uint64_t n, uint64_t nwork) {
    const Plan &p = d->plan;
    const FrontPlan &f = p.front;
    const LaunchCtx c{d->stream, d->sm_count};
    const size_t sb = format == APT_PCM16 ? 2 : 4;
    const uint64_t cap = d->chunk_samples;
    const uint64_t units = f.units(nwork);
    uint64_t per_chunk;
    APT_TRY(f.chunk_units(cap, per_chunk));
    char *stage[2] = {static_cast<char *>(d->d_in), static_cast<char *>(d->d_in) + cap * 4};
    uint64_t chunk = 0;
    Prof pr(d, kFrontSlot);
    for (uint64_t u0 = 0; u0 < units; u0 += per_chunk, ++chunk) {
        const uint64_t u1 = std::min(units, u0 + per_chunk);
        const int b = static_cast<int>(chunk & 1);
        uint64_t xa, xb;
        f.span(u0, u1, n, xa, xb);
        if (xb <= xa || xb - xa > cap) return fail(APT_ERR_BAD_ARG, "internal: chunk geometry (%llu..%llu, cap %llu)",
                                                   (unsigned long long)xa, (unsigned long long)xb, (unsigned long long)cap);
        // copy stream: wait until the compute stream has finished with this buffer, then upload
        if (chunk >= 2) APT_CUDA(cudaStreamWaitEvent(d->copy_stream, d->ev_free[b], 0));
        if (d->job_in_pageable && d->stager)
            APT_CUDA(d->stager->upload(stage[b], static_cast<const char *>(host) + xa * sb, (xb - xa) * sb, d->copy_stream));
        else
            APT_CUDA(cudaMemcpyAsync(stage[b], static_cast<const char *>(host) + xa * sb, (xb - xa) * sb, cudaMemcpyHostToDevice,
                                     d->copy_stream));
        APT_CUDA(cudaEventRecord(d->ev_copied[b], d->copy_stream));
        APT_CUDA(cudaStreamWaitEvent(d->stream, d->ev_copied[b], 0));
        // compute stream: (cast,) resample + envelope of this chunk's units
        float *conv_biased = nullptr;
        if (format == APT_PCM16 && f.wants_f32()) {
            APT_TRY(launch_pcm16_to_f32(c, reinterpret_cast<const int16_t *>(stage[b]), xb - xa, d->d_conv));
            d->launches++;
            conv_biased = d->d_conv - xa;
        }
        d->launches++;
        APT_TRY(front_launch(c, f, d->front, stage[b] - xa * sb, format, conv_biased, n, nwork, u0, u1, true, p.cosphi2, p.sinphi,
                             nullptr, d->d_e, nullptr));
        APT_CUDA(cudaEventRecord(d->ev_free[b], d->stream));
    }
    d->job_chunks = chunk;
    return APT_OK;
}

static int enqueue_front(apt_decoder *d, const void *in, int format, uint64_t n, uint64_t nwork, const void *host_chunked) {
    const Plan &p = d->plan;
    const LaunchCtx c{d->stream, d->sm_count};
    if (d->cb) {
        char msg[64];
        snprintf(msg, sizeof(msg), "Resampling to %u", p.st.work_rate);
        d->cb(0.1f, msg, d->cb_user);                                       // decode.rs:63
    }
    d->job_chunks = 0;
    if (host_chunked) {
        APT_TRY(enqueue_front_chunked(d, host_chunked, format, n, nwork));
    } else {
        const float *conv = nullptr;
        if (format == APT_PCM16 && p.front.wants_f32() && (reinterpret_cast<uintptr_t>(in) & 15) == 0) {
            // the WAV's int16 samples: `as f32` (wav.rs:37) on the device, then the f32 kernel
            APT_TRY(ensure_conv(d, n, std::max<uint64_t>(d->max_samples, n)));
            APT_TRY(launch_pcm16_to_f32(c, static_cast<const int16_t *>(in), n, d->d_conv));
            d->launches++;
            conv = d->d_conv;
        }
        // resample (decode.rs:77) + demodulate (decode.rs:89)
        DecoderHook hook(d);
        APT_TRY(front_launch(c, p.front, d->front, in, format, conv, n, nwork, 0, p.front.units(nwork), true, p.cosphi2, p.sinphi,
                             d->d_r, d->d_e, &hook));
    }
    if (d->cb) d->cb(0.4f, "Demodulating", d->cb_user);                     // decode.rs:87
    if (d->cb) d->cb(0.42f, "Filtering", d->cb_user);                       // decode.rs:93
    return APT_OK;
}

// Enqueues the whole of decode() on the decoder's stream.  `in` and `rows_out` are device pointers.
std::atomic<int> g_jobs_in_flight[64];      // per CUDA device: decodes submitted and not yet waited for

// The envelope e (4 N_w bytes, 45 MB for 15 min) is written by the resampler and read by the record and the gather
// kernels; between those, the resampler's 173 MB input stream pushes it out of the 50 MB L2, so e goes to DRAM and comes
// back.  When this is the only decode on the device, e can get a PERSISTING access-policy window on the decoder's stream
// (everything else the stream touches is treated as streaming) for as much of it as the set-aside holds.
// With several decodes in flight the set-aside would only shrink the cache, so the window is dropped then.
// OPT-IN (APTB200_L2_WINDOW=1): not validated next to NCCL or in a multi-device process, and a device-wide L2 carve-out
// is not something to switch on unverified.
static void set_envelope_l2_window(apt_decoder *d, uint64_t nwork, bool alone) {
    static const bool disabled = getenv("APTB200_L2_WINDOW") == nullptr;
    static std::atomic<int> setaside[64];              // per device: bytes set aside (0 not tried yet, -1 unsupported)
    static std::atomic<int> window_max[64];            // per device: largest access-policy window
    if (disabled || d->device < 0 || d->device >= 64 || !d->d_e) return;
    int have = setaside[d->device].load(std::memory_order_acquire);
    if (have == 0) {
        int max_persist = 0, max_window = 0;
        cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, d->device);
        cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, d->device);
        have = -1;
        if (max_persist > 0 && max_window > 0) {
            const size_t want = std::min<size_t>(static_cast<size_t>(max_persist), 64u << 20);
            if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) have = static_cast<int>(want);
        }
        cudaGetLastError();
        window_max[d->device].store(max_window, std::memory_order_release);
        setaside[d->device].store(have, std::memory_order_release);
    }
    if (have <= 0) return;
    const uint64_t wmax = static_cast<uint64_t>(window_max[d->device].load(std::memory_order_acquire));
    const uint64_t bytes = alone ? std::min<uint64_t>(nwork * sizeof(float), wmax) : 0;   // larger than the set-aside: hitRatio < 1
    if (bytes == d->l2_window_bytes) return;
    cudaStreamAttrValue v{};
    v.accessPolicyWindow.base_ptr = d->d_e;
    v.accessPolicyWindow.num_bytes = static_cast<size_t>(bytes);
    v.accessPolicyWindow.hitRatio = bytes ? std::min(1.0f, static_cast<float>(have) / static_cast<float>(bytes)) : 0.f;
    v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    if (cudaStreamSetAttribute(d->stream, cudaStreamAttributeAccessPolicyWindow, &v) == cudaSuccess) d->l2_window_bytes = bytes;
    if (bytes == 0) cudaCtxResetPersistingL2Cache();   // lines that still persist would keep the set-aside from everybody else
    cudaGetLastError();
}

int decoder_enqueue(apt_decoder *d, const void *in, int format, uint64_t n, int sync, float *rows_out,
                    const void *host_chunked) {
    const Plan &p = d->plan;
    LaunchCtx c{d->stream, d->sm_count};
    c.busy = d->device >= 0 && d->device < 64 && g_jobs_in_flight[d->device].load(std::memory_order_relaxed) > 0 ? 1 : 0;
    const uint64_t nwork = p.front.work_len(n);
    d->job_work = nwork;
    d->ev_used = 0;
    set_envelope_l2_window(d, nwork, c.busy == 0);

    APT_TRY(enqueue_front(d, in, format, n, nwork, host_chunked));
    if (sync) {
        if (d->cb) d->cb(0.5f, "Syncing", d->cb_user);                      // decode.rs:107
        if (!p.work_multiple) return fail(APT_ERR_WORK_RATE, "work_rate is not multiple of FINAL_RATE");   // decode.rs:172-176
    } else {
        if (d->cb) d->cb(0.5f, "Skipping Syncing", d->cb_user);             // decode.rs:136
        if (d->cb) d->cb(0.9f, "Resampling to 4160", d->cb_user);           // decode.rs:154
    }
    DecoderHook hook(d);
    d->stages_materialised = false;
    APT_TRY(back_launch(c, p, d->back_plan, d->back, d->d_lp, d->d_one, d->d_e, nwork, sync != 0, rows_out, &hook, d->last_back));
    if (sync && d->cb) d->cb(0.9f, "Resampling to 4160", d->cb_user);
    d->job_fixed_out = sync ? 0 : plan_out_bound(p, n);
    return APT_OK;
}

}  // namespace aptb200
