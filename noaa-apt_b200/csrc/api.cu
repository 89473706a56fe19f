// C ABI (include/aptb200.h) over the decoder object and the stage kernels.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "aptb200.h"
#include "common.hpp"
#include "decoder.hpp"
#include "filters_host.hpp"
#include "launch.hpp"
#include "spectrum.hpp"

using namespace aptb200;

namespace aptb200 {
int decoder_enqueue(apt_decoder *d, const void *in, int format, uint64_t n, int sync, float *rows_out,
                    const void *host_chunked);
extern std::atomic<int> g_jobs_in_flight[64];
}  // namespace aptb200

namespace {

inline size_t sample_bytes(int format) { return format == APT_PCM16 ? 2 : 4; }

// RAII device buffer for the one-shot stage entry points.
struct DevBuf {
    void *p = nullptr;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    int alloc(size_t bytes) {
        APT_CUDA(cudaMalloc(&p, bytes ? bytes : 4));
        return APT_OK;
    }
    template <typename T>
    T *as() const { return static_cast<T *>(p); }
};

int require_device() {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    return APT_OK;
}

// Launch context of the one-shot stage entry points: default stream, SM count of the current device.
LaunchCtx stage_ctx() {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return LaunchCtx{nullptr, std::max(sms, 1)};
}

// The decoder's staging ring for pageable buffers, made on first use (make_stager: it may have none).
void ensure_stager(apt_decoder *d) {
    if (d->stager) return;
    d->own_stager = make_stager(d->device);
    d->stager = d->own_stager.get();
}

// The decode's errors that need no device, in the reference's order: the plan, fewer than 10 rows, sync without a
// work_rate multiple of 4160.  need (optional): the floats of the rows of n samples.
int check_decode(uint32_t rate, const apt_settings &s, uint64_t n, int sync, uint64_t *need = nullptr) {
    Plan p;
    APT_TRY(make_plan(rate, s, p));
    const uint64_t nwork = p.front.work_len(n);
    if (nwork < 10ull * p.row) return fail(APT_ERR_TOO_SHORT, "Got less than 10 rows of samples, audio file is too short");
    if (sync && !p.work_multiple) return fail(APT_ERR_WORK_RATE, "work_rate is not multiple of FINAL_RATE");
    if (need) *need = sync ? (nwork / p.row) * kPxPerRow : plan_out_bound(p, n);
    return APT_OK;
}

}  // namespace

int aptb200::free_decoder_buffers(apt_decoder *d) {
    cudaSetDevice(d->device);
    if (d->stream) cudaStreamSynchronize(d->stream);
    d->front.release();
    d->back.release();
    for (void *p : {(void *)d->d_lp, (void *)d->d_one, d->d_in, (void *)d->d_r, (void *)d->d_e, (void *)d->d_out, (void *)d->d_conv})
        if (p) cudaFree(p);
    if (d->h_res) cudaFreeHost(d->h_res);
    if (d->h_out) cudaFreeHost(d->h_out);
    d->img.release();
    d->iq_tables.release();
    d->iq_win.release();
    if (d->d_audio) cudaFree(d->d_audio);
    d->own_stager.reset();
    for (auto e : d->ev_begin) cudaEventDestroy(e);
    for (auto e : d->ev_end) cudaEventDestroy(e);
    for (int i = 0; i < 2; ++i) {
        if (d->ev_copied[i]) cudaEventDestroy(d->ev_copied[i]);
        if (d->ev_free[i]) cudaEventDestroy(d->ev_free[i]);
    }
    if (d->copy_stream) cudaStreamDestroy(d->copy_stream);
    if (d->stream) cudaStreamDestroy(d->stream);
    return APT_OK;
}

// ============================================================================ misc / status

extern "C" const char *apt_strerror(int status) {
    switch (status) {
    case APT_OK: return "ok";
    case APT_ERR_RESAMPLE_TO_ZERO: return "Can't resample to 0Hz";
    case APT_ERR_TOO_SHORT: return "Got less than 10 rows of samples, audio file is too short";
    case APT_ERR_FEW_SYNC_FRAMES: return "Found less than 5 sync frames, audio file is too short or too noisy";
    case APT_ERR_WORK_RATE: return "work_rate is not multiple of FINAL_RATE";
    case APT_ERR_RATE_OVERFLOW: return "Can't resample, looks like the sample rates do not have a big divisor in common";
    case APT_ERR_CUDA: return "CUDA error or no CUDA device (no CPU fallback)";
    case APT_ERR_BAD_ARG: return "invalid argument";
    case APT_ERR_NOMEM: return "out of memory";
    case APT_ERR_CAPACITY: return "output buffer too small";
    case APT_ERR_EMPTY_RESULT: return "Got zero samples after resampling, audio file too short or output sampling frequency too low";
    case APT_ERR_IO: return "WAV file cannot be opened, parsed or written";
    default: return "unknown status";
    }
}

extern "C" const char *apt_last_error(void) { return last_error_slot().c_str(); }
extern "C" int apt_abi_version(void) { return APTB200_ABI_VERSION; }

extern "C" int apt_device_count(void) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return count;
}

extern "C" void apt_default_settings(apt_settings *s) {
    if (!s) return;
    // default_settings.toml:108-116
    s->work_rate = 12480;
    s->resample_atten = 30.f;
    s->resample_delta_freq = 1000.f;
    s->resample_cutout = 4800.f;
    s->demodulation_atten = 25.f;
}

extern "C" int apt_profile_settings(const char *profile, apt_settings *s) {
    if (!profile || !s) return fail(APT_ERR_BAD_ARG, "null argument");
    if (!strcmp(profile, "standard")) {
        apt_default_settings(s);
    } else if (!strcmp(profile, "fast")) {      // default_settings.toml:120-128
        *s = apt_settings{16640, 30.f, 3000.f, 4800.f, 23.f};
    } else if (!strcmp(profile, "slow")) {      // default_settings.toml:132-140
        *s = apt_settings{20800, 40.f, 500.f, 4800.f, 25.f};
    } else {
        return fail(APT_ERR_BAD_ARG, "unknown profile '%s'", profile);
    }
    return APT_OK;
}

// ================================================================================ filters

extern "C" float apt_freq_hz(float f_hz, uint32_t rate_hz) { return Freq::hz(f_hz, rate_hz).get_pi_rad(); }
extern "C" float apt_bessel_i0(float x) { return bessel_i0(x); }

extern "C" void apt_filter_resample(apt_filter *f, uint32_t input_rate, uint32_t output_rate) {
    if (f) resample_filter(*f, input_rate, output_rate);
}

extern "C" int apt_filter_design(const apt_filter *f, float *out, size_t cap, size_t *n) {
    if (!f || !n) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<float> taps;
    int st = design(*f, taps);
    if (st != APT_OK) return fail(st, "filter cannot be designed (kind %d, atten %g, delta_w %g)", f->kind,
                                  (double)f->atten, (double)f->delta_w_pi);
    *n = taps.size();
    if (out && cap) memcpy(out, taps.data(), std::min(cap, taps.size()) * sizeof(float));
    return APT_OK;
}

extern "C" int apt_generate_sync_frame(uint32_t work_rate, int8_t *out, size_t cap, size_t *n) {
    if (!n) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<int8_t> g;
    int st = sync_frame(work_rate, g);
    if (st != APT_OK) return fail(st, "work_rate is not multiple of FINAL_RATE");
    *n = g.size();
    if (out && cap) memcpy(out, g.data(), std::min(cap, g.size()));
    return APT_OK;
}

// ============================================================================ stage: resample

namespace {

// The first stage of dsp::resample_with_filter (dsp.rs:62-98) for the caller's filter, and its output length.
int plan_resample(uint64_t n, uint32_t in_rate, uint32_t out_rate, const apt_filter *f, FrontPlan &fp, uint64_t &nout) {
    if (!f) return fail(APT_ERR_BAD_ARG, "null filter");
    Ratio r{};
    int st = resample_ratio(in_rate, out_rate, r);
    if (st == APT_ERR_RESAMPLE_TO_ZERO) return fail(st, "Can't resample to 0Hz");
    if (st == APT_ERR_RATE_OVERFLOW)
        return fail(st, "Can't resample, looks like the sample rates do not have a big divisor in common. "
                        "input_rate: %u, output_rate: %u, l: %u, m: %u", in_rate, out_rate, r.l, r.m);
    if (st != APT_OK) return fail(st, "invalid input rate");
    apt_filter ff = *f;
    if (r.l > 1) resample_filter(ff, in_rate, in_rate * r.l);   // dsp.rs:93
    std::vector<float> taps;
    st = design(ff, taps);
    if (st != APT_OK) return fail(st, "filter cannot be designed");
    fp = make_front(r, std::move(taps));
    nout = fp.work_len(n);
    return APT_OK;
}

}  // namespace

extern "C" int apt_resample_len(uint64_t n, uint32_t input_rate, uint32_t output_rate, const apt_filter *f,
                                uint64_t *nout) {
    if (!nout) return fail(APT_ERR_BAD_ARG, "null argument");
    FrontPlan fp;
    return plan_resample(n, input_rate, output_rate, f, fp, *nout);
}

extern "C" int apt_resample_with_filter(const float *signal, uint64_t n, uint32_t input_rate, uint32_t output_rate,
                                        const apt_filter *f, float *out, uint64_t cap, uint64_t *nout) {
    if (!nout || (!signal && n)) return fail(APT_ERR_BAD_ARG, "null argument");
    FrontPlan fp;
    APT_TRY(plan_resample(n, input_rate, output_rate, f, fp, *nout));
    const uint64_t ny = *nout;
    if (ny > cap || (!out && ny)) return fail(APT_ERR_CAPACITY, "output needs %llu floats", (unsigned long long)ny);
    if (ny == 0) return APT_OK;
    APT_TRY(require_device());
    FrontTables tables;
    DevBuf dx, dy;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(dy.alloc(ny * sizeof(float)));
    APT_CUDA(cudaMemcpy(dx.p, signal, n * sizeof(float), cudaMemcpyHostToDevice));
    APT_TRY(tables.upload(fp));
    APT_TRY(front_launch(stage_ctx(), fp, tables, dx.p, APT_F32, nullptr, n, ny, 0, fp.units(ny), false, 0.f, 1.f, nullptr,
                         dy.as<float>(), nullptr));
    APT_CUDA(cudaMemcpy(out, dy.p, ny * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}

extern "C" int apt_resample(const float *signal, uint64_t n, uint32_t input_rate, uint32_t output_rate, float atten,
                            float delta_w_pi, float *out, uint64_t cap, uint64_t *nout) {
    if (input_rate == 0) return fail(APT_ERR_BAD_ARG, "invalid input rate");
    // dsp.rs:140-149: keep what fits below the lower of the two Nyquist frequencies
    const float cut_hz = output_rate > input_rate ? static_cast<float>(input_rate) / 2.f
                                                  : static_cast<float>(output_rate) / 2.f;
    apt_filter f{APT_FILTER_LOWPASS, Freq::hz(cut_hz, input_rate).get_pi_rad(), atten, delta_w_pi};
    return apt_resample_with_filter(signal, n, input_rate, output_rate, &f, out, cap, nout);
}

// ===================================================================== stage: demod / filter

extern "C" int apt_demodulate(const float *signal, uint64_t n, float carrier_pi, float *out) {
    if (n == 0) return fail(APT_ERR_BAD_ARG, "empty signal");   // signal[0] panics, dsp.rs:367
    if (!signal || !out) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(require_device());
    const float phi = 2.f * Freq::pi_rad(carrier_pi).get_rad();
    const float cosphi2 = std::cos(phi) * 2.f;
    const float sinphi = std::sin(phi);
    DevBuf dx, dy;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(dy.alloc(n * sizeof(float)));
    APT_CUDA(cudaMemcpy(dx.p, signal, n * sizeof(float), cudaMemcpyHostToDevice));
    APT_TRY(launch_envelope(stage_ctx(), dx.as<float>(), n, cosphi2, sinphi, dy.as<float>()));
    APT_CUDA(cudaMemcpy(out, dy.p, n * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}

extern "C" int apt_filter_taps(const float *signal, uint64_t n, const float *coeff, size_t ncoeff, float *out) {
    if ((!signal || !out) && n) return fail(APT_ERR_BAD_ARG, "null argument");
    if (!coeff && ncoeff) return fail(APT_ERR_BAD_ARG, "null coefficients");
    if (n == 0) return APT_OK;
    APT_TRY(require_device());
    DevBuf dx, dc, dy;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(dc.alloc(ncoeff * sizeof(float)));
    APT_TRY(dy.alloc(n * sizeof(float)));
    APT_CUDA(cudaMemcpy(dx.p, signal, n * sizeof(float), cudaMemcpyHostToDevice));
    if (ncoeff) APT_CUDA(cudaMemcpy(dc.p, coeff, ncoeff * sizeof(float), cudaMemcpyHostToDevice));
    APT_TRY(launch_fir_decimate(stage_ctx(), dx.p, APT_F32, dc.as<float>(), static_cast<u32>(ncoeff), 1, n,
                                dy.as<float>()));
    APT_CUDA(cudaMemcpy(out, dy.p, n * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}

extern "C" int apt_filter_signal(const float *signal, uint64_t n, const apt_filter *f, float *out) {
    if (!f) return fail(APT_ERR_BAD_ARG, "null filter");
    std::vector<float> taps;
    int st = design(*f, taps);
    if (st != APT_OK) return fail(st, "filter cannot be designed");
    return apt_filter_taps(signal, n, taps.data(), taps.size(), out);
}

// ============================================================================ stage: find_sync

extern "C" int apt_find_sync(const float *signal, uint64_t n, uint32_t work_rate, uint64_t *positions, size_t cap,
                             size_t *npositions, float *corr) {
    if (!signal || !npositions) return fail(APT_ERR_BAD_ARG, "null argument");
    Plan p;
    p.st.work_rate = work_rate;
    int st = sync_frame(work_rate, p.guard);
    if (st != APT_OK) return fail(st, "work_rate is not multiple of FINAL_RATE");
    if (work_rate > UINT32_MAX / kPxPerRow) return fail(APT_ERR_BAD_ARG, "work_rate too large");
    p.work_multiple = true;
    p.row = kPxPerRow * work_rate / kFinalRate;
    p.dist = static_cast<uint32_t>(static_cast<uint64_t>(p.row) * 8 / 10);
    if (n < p.guard.size()) return fail(APT_ERR_BAD_ARG, "signal shorter than the sync frame");   // decode.rs:225 underflow
    if (n >= (1ull << 32)) return fail(APT_ERR_BAD_ARG, "signal too long");
    APT_TRY(require_device());
    if (n == p.guard.size()) {
        // empty correlation: the peak list is just the seed (0, 0.0) (decode.rs:208-209)
        if (positions && cap > 0) positions[0] = 0;
        *npositions = 1;
        return APT_OK;
    }
    // the stage takes an already filtered signal: the plan has no low-pass, so the kind is Generic (exact-order kernels)
    const BackPlan bp = make_back(p, n);
    if (!bp.can_sync) return fail(APT_ERR_BAD_ARG, "work_rate %u is too high for the sync picker (min_distance %u > 16384)",
                                  work_rate, p.dist);
    BackBuffers b;
    struct Stream {                          // drains before b is freed
        cudaStream_t s = nullptr;
        ~Stream() {
            if (s) cudaStreamSynchronize(s), cudaStreamDestroy(s);
        }
    } stream;
    APT_TRY(b.alloc(p, bp));
    APT_CUDA(cudaStreamCreateWithFlags(&stream.s, cudaStreamNonBlocking));
    LaunchCtx c = stage_ctx();
    c.stream = stream.s;
    APT_CUDA(cudaMemcpyAsync(b.f, signal, n * sizeof(float), cudaMemcpyHostToDevice, c.stream));
    APT_TRY(back_find_sync(c, p, bp, b, n));
    SyncResult res;
    APT_CUDA(cudaMemcpyAsync(&res, b.res, sizeof(res), cudaMemcpyDeviceToHost, c.stream));
    APT_CUDA(cudaStreamSynchronize(c.stream));
    const size_t got = res.n_peaks;
    *npositions = got;
    if (positions) {
        std::vector<u32> tmp(got);
        APT_CUDA(cudaMemcpy(tmp.data(), b.pos, got * sizeof(u32), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < std::min(got, cap); ++i) positions[i] = tmp[i];
    }
    if (corr) APT_CUDA(cudaMemcpy(corr, b.corr, (n - p.guard.size()) * sizeof(float), cudaMemcpyDeviceToHost));
    if (positions && got > cap) return fail(APT_ERR_CAPACITY, "positions needs %zu entries", got);
    return APT_OK;
}

// ================================================================================= decoder

extern "C" int apt_decode_len_bound(uint64_t n, uint32_t input_rate, const apt_settings *s, uint64_t *bound) {
    if (!s || !bound) return fail(APT_ERR_BAD_ARG, "null argument");
    Plan p;
    APT_TRY(make_plan(input_rate, *s, p));
    *bound = plan_out_bound(p, n);
    return APT_OK;
}

namespace aptb200 {

int upload_plan(apt_decoder *d) {
    const Plan &p = d->plan;
    const float one = 1.f;
    APT_TRY(d->front.upload(p.front));
    APT_CUDA(cudaMalloc(&d->d_lp, p.lp.size() * sizeof(float)));
    APT_CUDA(cudaMemcpy(d->d_lp, p.lp.data(), p.lp.size() * sizeof(float), cudaMemcpyHostToDevice));
    APT_CUDA(cudaMalloc(&d->d_one, sizeof(float)));
    APT_CUDA(cudaMemcpy(d->d_one, &one, sizeof(float), cudaMemcpyHostToDevice));
    return APT_OK;
}

uint64_t plan_table_bytes(const Plan &p) { return FrontTables::bytes(p.front) + (p.lp.size() + 1) * sizeof(float); }

}  // namespace aptb200

extern "C" int apt_decoder_create(int device, uint32_t input_rate, const apt_settings *s, uint64_t max_samples,
                                  apt_decoder **dec) {
    if (!s || !dec) return fail(APT_ERR_BAD_ARG, "null argument");
    *dec = nullptr;
    std::unique_ptr<apt_decoder> d(new (std::nothrow) apt_decoder);
    if (!d) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(make_plan(input_rate, *s, d->plan));
    APT_TRY(require_device());
    const Plan &p = d->plan;
    d->device = device;
    APT_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    APT_CUDA(cudaGetDeviceProperties(&prop, device));
    d->sm_count = prop.multiProcessorCount;

    struct Rollback {
        apt_decoder *d;
        bool armed = true;
        ~Rollback() {
            if (armed) free_decoder_buffers(d);
        }
    } rollback{d.get()};

    APT_CUDA(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
    d->max_samples = max_samples;
    {
        // staging for host submits: whole recording up to 64 Mi samples, else two chunks of 32 Mi (APTB200_CHUNK_SAMPLES overrides)
        uint64_t chunk = 32ull << 20;
        if (const char *e = getenv("APTB200_CHUNK_SAMPLES")) chunk = std::max<uint64_t>(strtoull(e, nullptr, 10), 1u << 16);
        chunk &= ~7ull;   // both staging halves stay 16-byte aligned for f32 and PCM16 samples
        d->chunk_samples = (max_samples > 2 * chunk && p.front.chunkable()) ? chunk : 0;
        if (getenv("APTB200_CHUNK_SAMPLES") && max_samples > chunk && p.front.chunkable()) d->chunk_samples = chunk;
    }
    d->max_work = p.front.work_len(max_samples);
    d->max_out = plan_out_bound(p, max_samples);
    if (d->max_work >= (1ull << 32))
        return fail(APT_ERR_BAD_ARG, "recording too long: %llu work-rate samples (limit 2^32-1)",
                    (unsigned long long)d->max_work);

    APT_TRY(upload_plan(d.get()));
    const size_t work_bytes = std::max<uint64_t>(d->max_work, 1) * sizeof(float);
    if (p.front.needs_scratch()) APT_CUDA(cudaMalloc(&d->d_r, work_bytes));
    APT_CUDA(cudaMalloc(&d->d_e, work_bytes));
    d->back_plan = make_back(p, d->max_work);
    APT_TRY(d->back.alloc(p, d->back_plan));
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&d->h_res), sizeof(SyncResult), cudaHostAllocDefault));
    memset(d->h_res, 0, sizeof(SyncResult));
    rollback.armed = false;
    *dec = d.release();
    return APT_OK;
}

extern "C" void apt_decoder_destroy(apt_decoder *dec) {
    if (!dec) return;
    free_decoder_buffers(dec);
    delete dec;
}

namespace {

// The job after the rows, at submit and again after a sync redo: the image stage on the rows in d_out (its head follows
// to the pinned copy), the SyncResult and, for host jobs, the rows or the image to the caller.
int enqueue_job_tail(apt_decoder *d) {
    ImageOut &o = d->img;
    if (o.plan.image) {
        const u32 max_rows = static_cast<u32>(std::max<uint64_t>(d->max_out / kPxPerRow, 1));
        const u32 fixed = d->job_sync ? 0u : static_cast<u32>(d->job_fixed_out / kPxPerRow);
        DecoderHook hook(d);
        APT_TRY(o.launch(LaunchCtx{d->stream, d->sm_count}, d->d_out, d->job_sync ? d->back.res : nullptr, fixed, max_rows,
                         d->job_host || o.plan.png ? nullptr : d->job_out, &hook));
    }
    if (d->job_sync) APT_CUDA(cudaMemcpyAsync(d->h_res, d->back.res, sizeof(SyncResult), cudaMemcpyDeviceToHost, d->stream));
    if (d->job_host && d->job_d2h_floats)
        APT_CUDA(cudaMemcpyAsync(d->job_out_pageable ? static_cast<void *>(d->h_out) : static_cast<void *>(d->job_out),
                                 o.plan.image ? static_cast<const void *>(o.px) : static_cast<const void *>(d->d_out),
                                 o.plan.px_bytes(d->job_d2h_floats), cudaMemcpyDeviceToHost, d->stream));
    return APT_OK;
}

int submit_common(apt_decoder *d, const void *signal, int format, uint64_t n, int sync, float *out, uint64_t cap,
                  bool host) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder already has a job in flight; call apt_decoder_wait first");
    if (format != APT_F32 && format != APT_PCM16) return fail(APT_ERR_BAD_ARG, "unknown sample format %d", format);
    if (n == 0 || !signal) return fail(APT_ERR_BAD_ARG, "empty signal");   // signal[0] panics in demodulate, dsp.rs:367
    if (n > d->max_samples)
        return fail(APT_ERR_BAD_ARG, "recording of %llu samples exceeds the decoder's max_samples %llu",
                    (unsigned long long)n, (unsigned long long)d->max_samples);
    const Plan &p = d->plan;
    APT_CUDA(cudaSetDevice(d->device));

    d->job_status = APT_OK;
    d->job_host = host;
    d->job_sync = sync != 0;
    d->job_n = n;
    d->job_out = out;
    d->job_cap = cap;
    d->job_fixed_out = 0;

    const uint64_t nwork = p.front.work_len(n);
    d->job_work = nwork;
    if (nwork < 10ull * p.row) {   // decode.rs:79-83
        d->job_status = fail(APT_ERR_TOO_SHORT, "Got less than 10 rows of samples, audio file is too short");
        return d->job_status;
    }
    if (d->job_sync && p.work_multiple && !d->back_plan.can_sync)
        return fail(APT_ERR_BAD_ARG, "work_rate %u is too high for the sync picker (min_distance %u > 16384); decode without "
                                     "sync or use a work_rate <= 37440", p.st.work_rate, p.dist);
    const uint64_t need = d->job_sync ? (nwork / p.row) * kPxPerRow : plan_out_bound(p, n);
    ImageOut &o = d->img;
    const bool post = o.plan.image;
    // cap counts bytes of an image job, floats of an f32 one; in PNG mode PNG bytes, checked at wait() once the file's
    // length is known
    const uint64_t per_px = post ? o.plan.post.bpp : 1;
    const bool png = post && o.plan.png;
    const bool keep = post && o.keep && host;
    if (png && o.plan.png_s.rgb_from_rgba && per_px != 4) return fail(APT_ERR_BAD_ARG, "rgb_from_rgba needs RGBA process output");
    if (png && !out) return fail(APT_ERR_BAD_ARG, "null output");
    if (!png && !keep && (!out || cap < need * per_px))
        return fail(APT_ERR_CAPACITY, "output needs room for %llu %s", (unsigned long long)(need * per_px), post ? "bytes" : "floats");
    if (post) {
        if (!p.work_multiple) return fail(APT_ERR_BAD_ARG, "the image stage needs rows of 2080 pixels (work_rate multiple of 4160)");
        APT_TRY(o.post.alloc(o.plan.post, static_cast<u32>(std::max<uint64_t>(d->max_out / kPxPerRow, 1))));
        if (!d->d_out) APT_CUDA(cudaMalloc(&d->d_out, std::max<uint64_t>(d->max_out, 1) * sizeof(float)));
        if (host || png) APT_TRY(o.reserve_px(std::max<uint64_t>(d->max_out, 1) * per_px));
    }

    const void *dev_in = signal;
    float *rows_dst = out;
    const void *host_chunked = nullptr;
    d->job_in_pageable = d->job_out_pageable = false;
    if (host) {
        d->job_in_pageable = is_pageable(signal);
        d->job_out_pageable = !png && !keep && is_pageable(out);   // PNG mode copies the file straight into `out` at wait()
        if (d->job_in_pageable || d->job_out_pageable) ensure_stager(d);
        if (d->job_out_pageable && !d->h_out)
            APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&d->h_out), std::max<uint64_t>(d->max_out, 1) * sizeof(float),
                                   cudaHostAllocDefault));   // sized for f32 rows: also holds the u8 image
        // Recordings longer than the chunk size are uploaded in chunks that overlap the resampling; shorter ones
        // (and the L == 1 first stage) are staged whole.
        const bool chunked = d->chunk_samples != 0 && n > d->chunk_samples && p.front.chunkable();
        if (d->chunk_samples != 0 && n > d->chunk_samples && !chunked)
            return fail(APT_ERR_BAD_ARG, "recording longer than the staging buffer and the first stage is not polyphase");
        const uint64_t stage_samples = d->chunk_samples ? 2 * d->chunk_samples : d->max_samples;
        if (!d->d_in) APT_CUDA(cudaMalloc(&d->d_in, std::max<uint64_t>(stage_samples, 1) * sizeof(float)));
        if (!d->d_out) APT_CUDA(cudaMalloc(&d->d_out, std::max<uint64_t>(d->max_out, 1) * sizeof(float)));
        if (chunked) {
            if (!d->copy_stream) {
                APT_CUDA(cudaStreamCreateWithFlags(&d->copy_stream, cudaStreamNonBlocking));
                for (int i = 0; i < 2; ++i) {
                    APT_CUDA(cudaEventCreateWithFlags(&d->ev_copied[i], cudaEventDisableTiming));
                    APT_CUDA(cudaEventCreateWithFlags(&d->ev_free[i], cudaEventDisableTiming));
                }
            }
            if (format == APT_PCM16) APT_TRY(ensure_conv(d, d->chunk_samples, d->chunk_samples));
            host_chunked = signal;
            dev_in = nullptr;
        } else if (d->job_in_pageable && d->stager) {
            APT_CUDA(d->stager->upload(d->d_in, signal, n * sample_bytes(format), d->stream));
            dev_in = d->d_in;
        } else {
            APT_CUDA(cudaMemcpyAsync(d->d_in, signal, n * sample_bytes(format), cudaMemcpyHostToDevice, d->stream));
            dev_in = d->d_in;
        }
        rows_dst = d->d_out;
    }
    if (post) rows_dst = d->d_out;      // the f32 rows are an intermediate of the image job
    d->job_rows_src = rows_dst;
    int st = decoder_enqueue(d, dev_in, format, n, sync, rows_dst, host_chunked);
    // the rows come back with the job: when syncing n_rows is only known on the device, so the copy covers the bound
    // (at most one row more than is produced)
    d->job_d2h_floats = !host || png || keep ? 0 : d->job_sync ? need : d->job_fixed_out;
    if (st == APT_OK) st = enqueue_job_tail(d);
    if (st != APT_OK) {
        cudaStreamSynchronize(d->stream);
        d->job_status = st;
        return st;
    }
    d->in_flight = true;
    if (d->device >= 0 && d->device < 64) g_jobs_in_flight[d->device].fetch_add(1, std::memory_order_relaxed);
    return APT_OK;
}

}  // namespace

extern "C" int apt_decoder_submit_device(apt_decoder *dec, const void *signal, int format, uint64_t n, int sync,
                                         float *out, uint64_t cap) {
    return submit_common(dec, signal, format, n, sync, out, cap, false);
}

extern "C" int apt_decoder_submit_host(apt_decoder *dec, const void *signal, int format, uint64_t n, int sync,
                                       float *out, uint64_t cap) {
    return submit_common(dec, signal, format, n, sync, out, cap, true);
}

namespace {

// PNG mode, at wait(): encode the job's image on the decoder's stream, read the file's length, then copy exactly that many
// bytes to the caller's buffer.  Two stream synchronisations.
int png_job(apt_decoder *d, uint64_t rows, uint64_t *bytes) {
    DecoderHook hook(d);
    APT_TRY(d->img.encode_px(LaunchCtx{d->stream, d->sm_count}, rows, &hook));
    APT_CUDA(cudaStreamSynchronize(d->stream));
    *bytes = d->img.length(0);
    APT_TRY(d->img.copy_out(0, d->job_out, d->job_cap, d->job_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, d->stream));
    APT_CUDA(cudaStreamSynchronize(d->stream));
    return APT_OK;
}

}  // namespace

extern "C" int apt_decoder_wait(apt_decoder *d, uint64_t *nout) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (nout) *nout = 0;
    if (!d->in_flight) return d->job_status;
    APT_CUDA(cudaSetDevice(d->device));
    d->in_flight = false;
    if (d->device >= 0 && d->device < 64) g_jobs_in_flight[d->device].fetch_sub(1, std::memory_order_relaxed);
    static const bool trace = getenv("APTB200_TRACE_HOST") != nullptr;
    const auto t_begin = std::chrono::steady_clock::now();
    APT_CUDA(cudaStreamSynchronize(d->stream));
    const auto t_synced = std::chrono::steady_clock::now();
    uint64_t produced = d->job_fixed_out;
    d->last_work = d->job_work;
    d->last_peaks = 0;
    if (d->job_sync) {
        if (d->h_res->status == kSyncRedo) {
            // the record pool overflowed (silence, ramps: every index a record): the sync decode runs again with the Hbm
            // kernels on the envelope that is still in d_e
            DecoderHook hook(d);
            APT_TRY(back_redo(LaunchCtx{d->stream, d->sm_count}, d->plan, d->back_plan, d->back, d->d_e, d->job_work,
                              const_cast<float *>(d->job_rows_src), &hook, d->last_back));
            APT_TRY(enqueue_job_tail(d));
            APT_CUDA(cudaStreamSynchronize(d->stream));
        }
        const SyncResult res = *d->h_res;
        d->last_peaks = res.n_peaks;
        if (res.status != APT_OK) {
            d->job_status = fail(static_cast<int>(res.status),
                                 "Found less than 5 sync frames, audio file is too short or too noisy");
            return d->job_status;
        }
        produced = static_cast<uint64_t>(res.n_rows) * kPxPerRow;
    }
    const bool png = d->img.plan.png;
    if (d->job_host && d->job_out_pageable && produced && !png) {
        if (d->stager) d->stager->scatter(d->job_out, d->h_out, d->img.plan.px_bytes(produced));
        else memcpy(d->job_out, d->h_out, d->img.plan.px_bytes(produced));
    }
    if (trace)
        fprintf(stderr, "[aptb200 host] wait: stream sync %.2f ms, copy-out %.2f ms (%s)\n",
                std::chrono::duration<double>(t_synced - t_begin).count() * 1e3,
                std::chrono::duration<double>(std::chrono::steady_clock::now() - t_synced).count() * 1e3,
                d->job_out_pageable ? "pageable" : "direct");
    if (d->img.plan.image) {
        d->job_status = post_result(*d->img.post.head, &d->img.info);
        if (d->job_status != APT_OK) return d->job_status;
    }
    d->last_rows = d->plan.work_multiple ? produced / kPxPerRow : 0;
    d->last_out = produced;
    uint64_t png_bytes = 0;
    if (png) {
        const int st = png_job(d, produced / kPxPerRow, &png_bytes);
        if (st != APT_OK) {
            if (st == APT_ERR_CAPACITY && nout) *nout = png_bytes;
            d->job_status = st;
            return st;
        }
    }
    if (d->profiling) {
        d->kernel_ms.assign(d->ev_used, 0.f);
        for (int i = 0; i < d->ev_used; ++i) cudaEventElapsedTime(&d->kernel_ms[i], d->ev_begin[i], d->ev_end[i]);
    }
    if (nout) *nout = png ? png_bytes : produced * (d->img.plan.image ? d->img.plan.post.bpp : 1);
    return APT_OK;
}

extern "C" int apt_decoder_set_image_mode(apt_decoder *d, int contrast, float percent) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder has a job in flight");
    if (contrast < 0) {
        d->img.plan = OutPlan{};
        return APT_OK;
    }
    if (contrast == APT_CONTRAST_HISTOGRAM) return fail(APT_ERR_BAD_ARG, "unknown contrast mode %d", contrast);
    PostPlan plan;
    APT_TRY(make_post(image_settings(contrast, percent), plan));
    d->img.plan.post = plan;
    d->img.plan.image = true;
    return APT_OK;
}

namespace {

// The output plan of the entry points that make an image from process settings taken by pointer: null process settings
// are an error, and so are null PNG settings when `file`.
int image_plan(const apt_process_settings *ps, const apt_png_settings *png, bool file, OutPlan &plan) {
    if (!ps) return fail(APT_ERR_BAD_ARG, "null process settings");
    APT_TRY(make_out_plan(ps, png, plan));
    if (file && !png) return fail(APT_ERR_BAD_ARG, "null PNG settings");
    return APT_OK;
}

}  // namespace

extern "C" int apt_decoder_set_process_mode(apt_decoder *d, const apt_process_settings *ps) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder has a job in flight");
    if (!ps) {
        d->img.plan = OutPlan{};
        return APT_OK;
    }
    PostPlan plan;
    APT_TRY(make_post(*ps, plan));
    if (plan.palette) {
        APT_CUDA(cudaSetDevice(d->device));
        APT_TRY(d->img.post.upload_palette(ps->palette, d->stream));
    }
    d->img.plan.post = plan;
    d->img.plan.image = true;
    return APT_OK;
}

extern "C" int apt_decoder_set_png_mode(apt_decoder *d, const apt_png_settings *ps) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder has a job in flight");
    if (ps && !d->img.plan.image) return fail(APT_ERR_BAD_ARG, "PNG mode needs image or process mode");
    return d->img.plan.set_png(ps);
}

extern "C" void apt_default_track_settings(apt_track_settings *ts) {
    if (ts) *ts = apt_track_settings{2, 0.25f};
}

extern "C" int apt_decoder_set_sync_mode(apt_decoder *d, int mode, const apt_track_settings *ts) {
    if (mode != APT_SYNC_PEAKS && mode != APT_SYNC_TRACK) return fail(APT_ERR_BAD_ARG, "unknown sync mode %d", mode);
    apt_track_settings t;
    apt_default_track_settings(&t);
    if (ts) t = *ts;
    if (mode == APT_SYNC_TRACK) APT_TRY(track_settings_check(t));
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder has a job in flight");
    if (mode == APT_SYNC_PEAKS) return back_set_track(d->plan, d->back_plan, d->back, nullptr);
    if (!d->back_plan.can_sync)
        return fail(APT_ERR_BAD_ARG, "tracked sync needs a decoder that can sync (work rate a multiple of 4160, at most 37440)");
    APT_CUDA(cudaSetDevice(d->device));
    return back_set_track(d->plan, d->back_plan, d->back, &t);
}

extern "C" int apt_decoder_image_info(apt_decoder *d, apt_image_info *info) {
    if (!d || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    *info = d->img.info;
    return APT_OK;
}

extern "C" int apt_decoder_last_sync(apt_decoder *d, uint64_t *positions, size_t cap, size_t *npositions) {
    if (!d || !npositions) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_CUDA(cudaSetDevice(d->device));
    const size_t got = d->last_peaks;
    *npositions = got;
    if (positions && got) {
        std::vector<u32> tmp(got);
        APT_CUDA(cudaMemcpy(tmp.data(), d->back.pos, got * sizeof(u32), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < std::min(got, cap); ++i) positions[i] = tmp[i];
    }
    return APT_OK;
}

extern "C" int apt_decoder_last_counts(apt_decoder *d, uint64_t *n_work, uint64_t *n_rows, uint64_t *n_peaks) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    if (n_work) *n_work = d->last_work;
    if (n_rows) *n_rows = d->last_rows;
    if (n_peaks) *n_peaks = d->last_peaks;
    return APT_OK;
}

extern "C" int apt_decoder_last_root_count(apt_decoder *d, uint64_t *n_roots) {
    if (!d || !n_roots) return fail(APT_ERR_BAD_ARG, "null argument");
    *n_roots = d->h_res ? d->h_res->n_roots : 0;
    return APT_OK;
}

extern "C" int apt_decoder_last_roots(apt_decoder *d, uint64_t *roots, size_t cap, size_t *nroots) {
    if (!d || !nroots) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_CUDA(cudaSetDevice(d->device));
    return back_roots(d->plan, d->back_plan, d->back, d->last_back, d->last_work, roots, cap, nroots);
}

extern "C" int apt_decoder_last_records(apt_decoder *d, apt_tile_records *tiles, size_t tiles_cap, size_t *ntiles,
                                        apt_record *records, size_t records_cap, size_t *nrecords) {
    if (!d || !ntiles || !nrecords) return fail(APT_ERR_BAD_ARG, "null argument");
    *ntiles = *nrecords = 0;
    if (d->in_flight) return fail(APT_ERR_BAD_ARG, "decoder has a job in flight");
    if (d->last_back != BackKind::Records || !d->job_sync)
        return fail(APT_ERR_BAD_ARG, "the last job did not run the record kernel (a Records sync job whose pool did not overflow)");
    APT_CUDA(cudaSetDevice(d->device));
    return back_records(d->plan, d->back_plan, d->back, d->last_work, tiles, tiles_cap, ntiles, records, records_cap, nrecords);
}

extern "C" int apt_decoder_read_stage(apt_decoder *d, int which, float *out, uint64_t cap, uint64_t *n) {
    if (!d || !n) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_CUDA(cudaSetDevice(d->device));
    const float *src = nullptr;
    uint64_t len = d->last_work;
    if (which != 0 && d->last_back == BackKind::Records && !d->stages_materialised && len) {
        // f / corr were never written: compute them now (the roots and records of the job stay where they are)
        APT_TRY(back_materialise(LaunchCtx{d->stream, d->sm_count}, d->plan, d->back_plan, d->back, d->d_e, len));
        d->stages_materialised = true;
    }
    switch (which) {
    case 0: src = d->d_e; break;
    case 1: src = d->back.f; break;
    case 2:
        src = d->back.corr;
        len = d->last_work > d->plan.guard.size() ? d->last_work - d->plan.guard.size() : 0;
        break;
    default: return fail(APT_ERR_BAD_ARG, "unknown stage %d", which);
    }
    if (!src) len = 0;
    *n = len;
    if (out && len) {
        if (cap < len) return fail(APT_ERR_CAPACITY, "stage needs %llu floats", (unsigned long long)len);
        APT_CUDA(cudaMemcpy(out, src, len * sizeof(float), cudaMemcpyDeviceToHost));
    }
    return APT_OK;
}

extern "C" int apt_decoder_set_profiling(apt_decoder *d, int enabled) {
    if (!d) return fail(APT_ERR_BAD_ARG, "null decoder");
    d->profiling = enabled != 0;
    return APT_OK;
}

extern "C" int apt_decoder_kernel_count(apt_decoder *d) { return d ? static_cast<int>(d->kernel_ms.size()) : 0; }

extern "C" const char *apt_decoder_kernel_name(apt_decoder *d, int i) {
    if (!d || i < 0 || i >= static_cast<int>(d->kernel_names.size())) return "";
    return d->kernel_names[i].c_str();
}

extern "C" int apt_decoder_kernel_ms(apt_decoder *d, float *ms, int cap, int *count) {
    if (!d || !count) return fail(APT_ERR_BAD_ARG, "null argument");
    *count = static_cast<int>(d->kernel_ms.size());
    for (int i = 0; i < std::min(cap, *count); ++i) ms[i] = d->kernel_ms[i];
    return APT_OK;
}

extern "C" void *apt_decoder_stream(apt_decoder *d) { return d ? static_cast<void *>(d->stream) : nullptr; }
extern "C" uint64_t apt_decoder_launch_count(apt_decoder *d) { return d ? d->launches : 0; }

// ============================================================================ memory helpers

extern "C" int apt_host_alloc(void **ptr, size_t bytes) {
    if (!ptr) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(require_device());
    APT_CUDA(cudaHostAlloc(ptr, bytes ? bytes : 4, cudaHostAllocPortable));
    return APT_OK;
}

extern "C" void apt_host_free(void *ptr) {
    if (ptr) cudaFreeHost(ptr);
}

extern "C" int apt_device_alloc(int device, void **ptr, size_t bytes) {
    if (!ptr) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(require_device());
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaMalloc(ptr, bytes ? bytes : 4));
    return APT_OK;
}

extern "C" void apt_device_free(int device, void *ptr) {
    if (!ptr) return;
    cudaSetDevice(device);
    cudaFree(ptr);
}

extern "C" int apt_memcpy_h2d(int device, void *dst, const void *src, size_t bytes) {
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    return APT_OK;
}

extern "C" int apt_memcpy_d2h(int device, void *dst, const void *src, size_t bytes) {
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return APT_OK;
}

// ============================================================================ one-shot decode

namespace {

// apt_decode() is what the Rust shim binds (rust/decode.rs): one call per recording, ordinary pageable buffers.  Creating a
// decoder costs ~14 cudaMalloc + a stream + pinned staging, so finished decoders are parked here, keyed by what their plan
// depends on, and the next call with the same (device, rate, settings) takes one over.  apt_cache_clear() frees them.
struct CacheEntry {
    apt_decoder *dec;
    uint64_t stamp;
};
std::mutex g_cache_mutex;
std::vector<CacheEntry> g_cache;
uint64_t g_cache_stamp = 0;
constexpr size_t kCacheMaxIdle = 8;

bool cache_on() {
    static const bool on = getenv("APTB200_NO_CACHE") == nullptr;
    return on;
}

bool same_key(const apt_decoder *d, int device, uint32_t rate, const apt_settings &st) {
    return d->device == device && d->plan.input_rate == rate && memcmp(&d->plan.st, &st, sizeof(st)) == 0;
}

}  // namespace

int aptb200::take_decoder(int device, uint32_t rate, const apt_settings &st, uint64_t n, bool headroom, apt_decoder **d) {
    *d = nullptr;
    if (!cache_on()) return apt_decoder_create(device, rate, &st, n, d);
    {
        std::lock_guard<std::mutex> lk(g_cache_mutex);
        for (size_t i = 0; i < g_cache.size(); ++i) {
            if (same_key(g_cache[i].dec, device, rate, st) && g_cache[i].dec->max_samples >= n) {
                *d = g_cache[i].dec;
                g_cache.erase(g_cache.begin() + static_cast<long>(i));
                return APT_OK;
            }
        }
    }
    // head-room so that the next, slightly longer recording of a series reuses the decoder
    const uint64_t room = headroom ? ((n + n / 8 + (1u << 20)) & ~((1ull << 20) - 1)) : n;
    return apt_decoder_create(device, rate, &st, room, d);
}

void aptb200::park_decoder(apt_decoder *d, bool several) {
    cudaStreamSynchronize(d->stream);
    d->img.plan = OutPlan{};
    d->img.keep = false;
    d->cb = nullptr;
    d->cb_user = nullptr;
    d->stager = d->own_stager.get();   // never keep a pointer into another decoder
    if (!cache_on()) {
        apt_decoder_destroy(d);
        return;
    }
    apt_decoder *victim = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_cache_mutex);
        size_t drop = g_cache.size();
        // one idle decoder per key is enough for a sequential caller: a smaller one of the same key is replaced
        for (size_t i = 0; i < g_cache.size() && !several && drop == g_cache.size(); ++i)
            if (same_key(g_cache[i].dec, d->device, d->plan.input_rate, d->plan.st) && g_cache[i].dec->max_samples <= d->max_samples)
                drop = i;
        if (drop == g_cache.size() && g_cache.size() >= kCacheMaxIdle) {
            drop = 0;
            for (size_t i = 1; i < g_cache.size(); ++i)
                if (g_cache[i].stamp < g_cache[drop].stamp) drop = i;
        }
        if (drop < g_cache.size()) {
            victim = g_cache[drop].dec;
            g_cache.erase(g_cache.begin() + static_cast<long>(drop));
        }
        g_cache.push_back(CacheEntry{d, ++g_cache_stamp});
    }
    if (victim) apt_decoder_destroy(victim);
}

namespace {

// ps: the image of process(), else (nullptr) f32 rows; png: that image as a PNG file.
int decode_oneshot(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                   float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user,
                   const apt_process_settings *ps = nullptr, apt_image_info *info = nullptr,
                   const apt_png_settings *png = nullptr) {
    if (!s || !nout) return fail(APT_ERR_BAD_ARG, "null argument");
    *nout = 0;
    if (n == 0 || !signal) return fail(APT_ERR_BAD_ARG, "empty signal");
    APT_TRY(check_decode(input_rate, *s, n, sync));
    APT_TRY(require_device());
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;
    apt_decoder *d = nullptr;
    APT_TRY(take_decoder(device, input_rate, *s, n, true, &d));
    d->cb = cb;
    d->cb_user = user;
    int st = ps ? apt_decoder_set_process_mode(d, ps) : APT_OK;
    if (st == APT_OK && png) st = apt_decoder_set_png_mode(d, png);
    if (st == APT_OK) st = apt_decoder_submit_host(d, signal, format, n, sync, out, cap);
    if (st == APT_OK) st = apt_decoder_wait(d, nout);
    if (st == APT_OK && info) *info = d->img.info;
    park_decoder(d, false);
    return st;
}

}  // namespace

extern "C" int apt_bind_thread_to_device(int device) {
    if (require_device() != APT_OK) return 0;
    return bind_thread_to_device(device) ? 1 : 0;
}

extern "C" void apt_cache_clear(void) {
    std::vector<CacheEntry> drop;
    {
        std::lock_guard<std::mutex> lk(g_cache_mutex);
        drop.swap(g_cache);
    }
    for (auto &e : drop) apt_decoder_destroy(e.dec);
    png_stage_cache_clear();
    spectrum_cache_clear();
}

extern "C" int apt_decode(const float *signal, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                          float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user) {
    return decode_oneshot(signal, APT_F32, n, input_rate, s, sync, out, cap, nout, cb, user);
}

extern "C" int apt_decode_pcm16(const int16_t *pcm, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                                float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user) {
    return decode_oneshot(pcm, APT_PCM16, n, input_rate, s, sync, out, cap, nout, cb, user);
}

namespace {

// apt_decode_iq_channels, with a status callback for every channel's decode.
int decode_iq_channels(const void *iq, int format, uint64_t n, const apt_iq_settings *is, const int32_t *offsets, int count,
                       const apt_settings *s, int sync, float *const *outs, const uint64_t *caps, uint64_t *nouts,
                       int *statuses, apt_status_cb cb, void *user) {
    if (!is || !s || !offsets || !outs || !caps || !nouts || !statuses || count < 1)
        return fail(APT_ERR_BAD_ARG, "null argument or count < 1");
    auto fail_all = [&](int st) {
        for (int c = 0; c < count; ++c) statuses[c] = st;
        return st;
    };
    for (int c = 0; c < count; ++c) {
        nouts[c] = 0;
        statuses[c] = APT_ERR_CUDA;   // overwritten by the channel's own status; never left "ok" by default
    }
    if (n == 0 || !iq) return fail_all(fail(APT_ERR_BAD_ARG, "empty signal"));
    if (!iq_sample_bytes(format)) return fail_all(fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format));
    // every channel's argument errors before any device work, in decode_oneshot's order
    std::vector<IqPlan> ips(count);
    std::vector<apt_iq_settings> iss(count, *is);
    for (int c = 0; c < count; ++c) {
        iss[c].offset_hz = offsets[c];
        const int st = make_iq(iss[c], ips[c]);
        if (st != APT_OK) return fail_all(st);
    }
    const uint64_t na = ips[0].out_len(n);
    const uint32_t rate = is->audio_rate;
    uint64_t need = 0;
    if (const int st = check_decode(rate, *s, na, sync, &need); st != APT_OK) return fail_all(st);
    std::vector<int> live;
    for (int c = 0; c < count; ++c) {
        if (!outs[c] || caps[c] < need)
            statuses[c] = fail(APT_ERR_CAPACITY, "output needs room for %llu floats", (unsigned long long)need);
        else
            live.push_back(c);
    }
    auto first_status = [&]() {
        for (int c = 0; c < count; ++c)
            if (statuses[c] != APT_OK) return statuses[c];
        return static_cast<int>(APT_OK);
    };
    if (live.empty()) return first_status();
    if (const int st = require_device(); st != APT_OK) return fail_all(st);
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;
    // one parked decoder per live channel; the first one's stream, stager and I/Q window carry the upload
    std::vector<apt_decoder *> decs;
    const bool pageable = is_pageable(iq);
    cudaEvent_t demod_done = nullptr;
    auto setup = [&]() -> int {
        for (int c : live) {
            apt_decoder *d = nullptr;
            APT_TRY(take_decoder(device, rate, *s, na, true, &d));
            decs.push_back(d);
            d->cb = cb;
            d->cb_user = user;
            APT_CUDA(cudaSetDevice(d->device));
            if (!d->iq_tables_valid || memcmp(&d->iq_settings, &iss[c], sizeof(iss[c])) != 0) {
                d->iq_tables_valid = false;
                APT_TRY(d->iq_tables.upload(ips[c]));
                d->iq_settings = iss[c];
                d->iq_tables_valid = true;
            }
            if (d->audio_cap < d->max_samples) {
                if (d->d_audio) APT_CUDA(cudaFree(d->d_audio));
                d->d_audio = nullptr;
                d->audio_cap = 0;
                APT_CUDA(cudaMalloc(&d->d_audio, std::max<uint64_t>(d->max_samples, 1) * sizeof(float)));
                d->audio_cap = d->max_samples;
            }
            if (!d->d_out) APT_CUDA(cudaMalloc(&d->d_out, std::max<uint64_t>(d->max_out, 1) * sizeof(float)));
        }
        apt_decoder *d0 = decs[0];
        if (pageable) ensure_stager(d0);
        std::vector<const IqPlan *> pl;
        std::vector<const IqTables *> tb;
        std::vector<float *> au;
        for (size_t k = 0; k < live.size(); ++k) {
            pl.push_back(&ips[live[k]]);
            tb.push_back(&decs[k]->iq_tables);
            au.push_back(decs[k]->d_audio);
        }
        APT_TRY(iq_demod_host_multi(LaunchCtx{d0->stream, d0->sm_count}, pl.data(), tb.data(), au.data(),
                                    static_cast<int>(live.size()), iq, format, n, d0->iq_win, pageable ? d0->stager : nullptr,
                                    nullptr));
        APT_CUDA(cudaEventCreateWithFlags(&demod_done, cudaEventDisableTiming));
        APT_CUDA(cudaEventRecord(demod_done, d0->stream));
        return APT_OK;
    };
    const int st = setup();
    if (st == APT_OK) {
        // every channel's decode on its own decoder's stream, after the demodulation; they run side by side
        std::vector<int> submitted(live.size(), APT_OK);
        for (size_t k = 0; k < live.size(); ++k) {
            apt_decoder *d = decs[k];
            submitted[k] = cudaStreamWaitEvent(d->stream, demod_done, 0) == cudaSuccess
                               ? apt_decoder_submit_device(d, d->d_audio, APT_F32, na, sync, d->d_out, d->max_out)
                               : fail(APT_ERR_CUDA, "cudaStreamWaitEvent failed");
        }
        for (size_t k = 0; k < live.size(); ++k) {
            apt_decoder *d = decs[k];
            const int c = live[k];
            uint64_t produced = 0;
            int cst = submitted[k];
            if (cst == APT_OK) cst = apt_decoder_wait(d, &produced);
            if (cst == APT_OK && cudaMemcpy(outs[c], d->d_out, produced * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess)
                cst = fail(APT_ERR_CUDA, "copying the rows of channel %d failed", c);
            if (cst == APT_OK) nouts[c] = produced;
            statuses[c] = cst;
        }
    } else {
        for (int c : live) statuses[c] = st;
    }
    if (demod_done) cudaEventDestroy(demod_done);
    for (apt_decoder *d : decs) park_decoder(d, decs.size() > 1);
    return st != APT_OK ? st : first_status();
}

}  // namespace

// apt_decode at audio_rate of the audio the FM kernel writes into the parked decoder's device input: the one channel at
// is->offset_hz.
extern "C" int apt_decode_iq(const void *iq, int format, uint64_t n, const apt_iq_settings *is, const apt_settings *s, int sync,
                             float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user) {
    if (!is || !s || !nout) return fail(APT_ERR_BAD_ARG, "null argument");
    int status = APT_OK;
    return decode_iq_channels(iq, format, n, is, &is->offset_hz, 1, s, sync, &out, &cap, nout, &status, cb, user);
}

extern "C" int apt_decode_iq_channels(const void *iq, int format, uint64_t n, const apt_iq_settings *is, const int32_t *offsets,
                                      int count, const apt_settings *s, int sync, float *const *outs, const uint64_t *caps,
                                      uint64_t *nouts, int *statuses) {
    return decode_iq_channels(iq, format, n, is, offsets, count, s, sync, outs, caps, nouts, statuses, nullptr, nullptr);
}

extern "C" int apt_decode_iq_auto(const void *iq, int format, uint64_t n, const apt_iq_settings *is, const apt_carrier_search *cs,
                                  const apt_settings *s, int sync, apt_carrier *found, uint32_t cap_found, uint32_t *nfound,
                                  float *const *outs, const uint64_t *caps, uint64_t *nouts, int *statuses) {
    if (!is || !s || !nfound || (cap_found && (!found || !outs || !caps || !nouts || !statuses)))
        return fail(APT_ERR_BAD_ARG, "null argument");
    *nfound = 0;
    if (n == 0 || !iq) return fail(APT_ERR_BAD_ARG, "empty signal");
    if (!iq_sample_bytes(format)) return fail(APT_ERR_BAD_ARG, "unknown I/Q sample format %d", format);
    {
        // the decode's argument errors (on offset 0) and the search's, before any device work
        apt_iq_settings s0 = *is;
        s0.offset_hz = 0;
        IqPlan ip;
        APT_TRY(make_iq(s0, ip));
        SearchParams sp;
        APT_TRY(make_search(cs, is->iq_rate, sp));
        SpecPlan spec;
        APT_TRY(make_spectrum(n, sp.nfft, sp.max_segments, spec));
        APT_TRY(check_decode(is->audio_rate, *s, ip.out_len(n), sync));
    }
    // kept carriers are more than 40 kHz apart inside a band narrower than iq_rate: this many always suffice
    std::vector<apt_carrier> all(is->iq_rate / 40000 + 2);
    uint32_t total = 0;
    APT_TRY(apt_iq_find_carriers(iq, format, n, is, cs, all.data(), static_cast<uint32_t>(all.size()), &total));
    std::vector<int32_t> offsets;
    for (uint32_t i = 0; i < total && offsets.size() < cap_found; ++i)
        if (all[i].is_apt) {
            found[offsets.size()] = all[i];
            offsets.push_back(all[i].offset_hz);
        }
    *nfound = static_cast<uint32_t>(offsets.size());
    if (offsets.empty()) return APT_OK;
    return apt_decode_iq_channels(iq, format, n, is, offsets.data(), static_cast<int>(offsets.size()), s, sync, outs, caps,
                                  nouts, statuses);
}

// ============================================================================== image stage

extern "C" int apt_decode_image_u8(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s,
                                   int sync, int contrast, float percent, uint8_t *out, uint64_t cap, uint64_t *nout,
                                   apt_image_info *info, apt_status_cb cb, void *user) {
    if (contrast == APT_CONTRAST_HISTOGRAM) return fail(APT_ERR_BAD_ARG, "unknown contrast mode %d", contrast);
    const apt_process_settings ps = image_settings(contrast, percent);
    PostPlan plan;
    APT_TRY(make_post(ps, plan));
    return decode_oneshot(signal, format, n, input_rate, s, sync, reinterpret_cast<float *>(out), cap, nout, cb, user, &ps, info);
}

extern "C" int apt_decode_image(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                                const apt_process_settings *ps, uint8_t *out, uint64_t cap, uint64_t *nout, apt_image_info *info,
                                apt_status_cb cb, void *user) {
    OutPlan plan;
    APT_TRY(image_plan(ps, nullptr, false, plan));
    return decode_oneshot(signal, format, n, input_rate, s, sync, reinterpret_cast<float *>(out), cap, nout, cb, user, ps, info);
}

extern "C" int apt_decode_png(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                              const apt_process_settings *ps, const apt_png_settings *png, uint8_t *out, uint64_t cap,
                              uint64_t *nout, apt_image_info *info, apt_status_cb cb, void *user) {
    OutPlan plan;
    APT_TRY(image_plan(ps, png, true, plan));
    if (!out) return fail(APT_ERR_BAD_ARG, "null output");
    return decode_oneshot(signal, format, n, input_rate, s, sync, reinterpret_cast<float *>(out), cap, nout, cb, user, ps, info, png);
}

extern "C" int apt_decode_wav_png(const char *input_path, const char *output_path, const apt_settings *s, int sync,
                                  const apt_process_settings *ps, const apt_png_settings *png, apt_image_info *info) {
    if (!input_path || !output_path || !s) return fail(APT_ERR_BAD_ARG, "null argument");
    OutPlan plan;
    APT_TRY(image_plan(ps, png, true, plan));
    apt_wav_info wi;
    APT_TRY(apt_wav_info_read(input_path, &wi));
    uint32_t rate = 0;
    uint64_t n = 0;
    std::vector<int16_t> pcm;
    std::vector<float> x;
    const bool pcm16 = !wi.is_float && wi.bits_per_sample == 16;
    if (pcm16) {
        pcm.resize(std::max<uint64_t>(wi.frames, 1));
        APT_TRY(apt_wav_load_pcm16(input_path, pcm.data(), pcm.size(), &n, &rate));
    } else {
        x.resize(std::max<uint64_t>(wi.frames, 1));
        APT_TRY(apt_wav_load(input_path, x.data(), x.size(), &n, &rate));
    }
    uint64_t px_bound = 0, cap = 0;
    APT_TRY(apt_decode_len_bound(n, rate, s, &px_bound));
    APT_TRY(plan.bytes(px_bound, cap));
    std::vector<uint8_t> bytes(cap);
    uint64_t nout = 0;
    APT_TRY(apt_decode_png(pcm16 ? static_cast<const void *>(pcm.data()) : static_cast<const void *>(x.data()),
                           pcm16 ? APT_PCM16 : APT_F32, n, rate, s, sync, ps, png, bytes.data(), cap, &nout, info, nullptr,
                           nullptr));
    FILE *fp = fopen(output_path, "wb");
    if (!fp) return fail(APT_ERR_IO, "cannot open %s for writing", output_path);
    const bool ok = fwrite(bytes.data(), 1, nout, fp) == nout;
    if (fclose(fp) != 0 || !ok) return fail(APT_ERR_IO, "cannot write %s", output_path);
    return APT_OK;
}

namespace {

// rows on the host -> device, image-mode stage, results back (stage entry points; one call, no retained state).  bounds:
// map with these; out == nullptr: statistics and bounds only.  A signal that is not whole rows is one row of n pixels.
int image_stage_host(const float *signal, uint64_t n, int contrast, float percent, const float *bounds, apt_image_info *info,
                     uint8_t *out, float *mean_a, float *mean_b, float *variance) {
    if (!signal || n == 0) return fail(APT_ERR_BAD_ARG, "empty signal");   // get_min of an empty vector is an error, dsp.rs:21-25
    APT_TRY(require_device());
    const uint64_t rows = n / kPxPerRow;
    const bool whole = rows * kPxPerRow == n && rows > 0;
    if (!whole && (contrast == APT_CONTRAST_TELEMETRY || mean_a)) return fail(APT_ERR_BAD_ARG, "not a whole number of 2080-px rows");
    if (!whole && n >= (1ull << 32)) return fail(APT_ERR_BAD_ARG, "signal too long");
    PostPlan plan;
    APT_TRY(make_post(image_settings(contrast, percent), plan));
    // a partial last row cannot occur in an image; min/max, percent and the map treat the signal as one row of n pixels then
    const u32 nrows = whole ? static_cast<u32>(rows) : 1u;
    const u32 px = whole ? kPxPerRow : static_cast<u32>(n);
    DevBuf dx, dout, dbounds;
    PostBuffers b;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(b.alloc(plan, nrows));
    if (out) APT_TRY(dout.alloc(n));
    APT_CUDA(cudaMemcpy(dx.p, signal, n * sizeof(float), cudaMemcpyHostToDevice));
    if (bounds) {
        APT_TRY(dbounds.alloc(2 * sizeof(float)));
        APT_CUDA(cudaMemcpy(dbounds.p, bounds, 2 * sizeof(float), cudaMemcpyHostToDevice));
    }
    APT_TRY(post_launch(stage_ctx(), plan, b, dx.as<float>(), nullptr, nrows, nrows, px, dbounds.as<float>(), dout.p, nullptr));
    APT_CUDA(cudaDeviceSynchronize());
    if (!bounds) {
        apt_image_info ii{};
        APT_TRY(post_result(*b.head, &ii));
        if (info) *info = ii;
        if (info && !whole) info->rows = 0;
    }
    if (out) APT_CUDA(cudaMemcpy(out, dout.p, n, cudaMemcpyDeviceToHost));
    if (mean_a) APT_CUDA(cudaMemcpy(mean_a, b.tel, rows * sizeof(float), cudaMemcpyDeviceToHost));
    if (mean_b) APT_CUDA(cudaMemcpy(mean_b, b.tel + rows, rows * sizeof(float), cudaMemcpyDeviceToHost));
    if (variance) APT_CUDA(cudaMemcpy(variance, b.tel + 2 * rows, rows * sizeof(float), cudaMemcpyDeviceToHost));
    return APT_OK;
}

}  // namespace

extern "C" int apt_map_signal_u8(const float *signal, uint64_t n, float low, float high, uint8_t *out) {
    if (n == 0) return APT_OK;
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    const float b[2] = {low, high};
    return image_stage_host(signal, n, APT_CONTRAST_MINMAX, 0.f, b, nullptr, out, nullptr, nullptr, nullptr);
}

extern "C" int apt_contrast_bounds(const float *signal, uint64_t n, int contrast, float percent, apt_image_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    if (contrast == APT_CONTRAST_HISTOGRAM) return fail(APT_ERR_BAD_ARG, "unknown contrast mode %d", contrast);
    PostPlan plan;
    APT_TRY(make_post(image_settings(contrast, percent), plan));
    memset(info, 0, sizeof(*info));
    return image_stage_host(signal, n, contrast, percent, nullptr, info, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int apt_telemetry_rows(const float *signal, uint64_t n, float *mean_a, float *mean_b, float *variance) {
    if (!mean_a || !mean_b || !variance) return fail(APT_ERR_BAD_ARG, "null argument");
    return image_stage_host(signal, n, APT_CONTRAST_MINMAX, 0.f, nullptr, nullptr, nullptr, mean_a, mean_b, variance);
}

extern "C" int apt_process(const float *rows, uint64_t n, const apt_process_settings *ps, uint8_t *out, uint64_t cap,
                           uint64_t *nout, apt_image_info *info) {
    OutPlan op;
    APT_TRY(image_plan(ps, nullptr, false, op));
    const PostPlan &plan = op.post;
    if (!nout) return fail(APT_ERR_BAD_ARG, "null argument");
    *nout = 0;
    if (!rows || n == 0) return fail(APT_ERR_BAD_ARG, "empty signal");   // get_min of an empty vector is an error, dsp.rs:21-25
    const uint64_t nrows = n / kPxPerRow;
    if (nrows * kPxPerRow != n) return fail(APT_ERR_BAD_ARG, "not a whole number of 2080-px rows");
    if (nrows >= (1ull << 32) / kPxPerRow) return fail(APT_ERR_BAD_ARG, "image too large");
    const uint64_t bytes = n * plan.bpp;
    if (!out || cap < bytes) return fail(APT_ERR_CAPACITY, "output needs room for %llu bytes", (unsigned long long)bytes);
    APT_TRY(require_device());
    DevBuf dx, dout;
    PostBuffers b;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(b.alloc(plan, static_cast<u32>(nrows)));
    APT_TRY(dout.alloc(bytes));
    APT_CUDA(cudaMemcpy(dx.p, rows, n * sizeof(float), cudaMemcpyHostToDevice));
    if (plan.palette) APT_TRY(b.upload_palette(ps->palette, nullptr));
    APT_TRY(post_launch(stage_ctx(), plan, b, dx.as<float>(), nullptr, static_cast<u32>(nrows), static_cast<u32>(nrows), kPxPerRow,
                        nullptr, dout.p, nullptr));
    APT_CUDA(cudaDeviceSynchronize());
    apt_image_info ii{};
    APT_TRY(post_result(*b.head, &ii));
    APT_CUDA(cudaMemcpy(out, dout.p, bytes, cudaMemcpyDeviceToHost));
    if (info) *info = ii;
    *nout = bytes;
    return APT_OK;
}

// ======================================================================= resample tool (WAV -> WAV)

extern "C" int apt_quantize_i16(const float *signal, uint64_t n, int16_t *out) {
    if (n == 0 || !signal) return fail(APT_ERR_BAD_ARG, "Can't get maximum of a zero length vector");   // dsp.rs:21-25
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(require_device());
    DevBuf dx, dctl, dout;
    APT_TRY(dx.alloc(n * sizeof(float)));
    APT_TRY(dctl.alloc(sizeof(PostCtl)));
    APT_TRY(dout.alloc(n * sizeof(int16_t)));
    APT_CUDA(cudaMemcpy(dx.p, signal, n * sizeof(float), cudaMemcpyHostToDevice));
    APT_TRY(launch_quantize_i16(stage_ctx(), dx.as<float>(), n, dctl.as<PostCtl>(), dout.as<short>()));
    APT_CUDA(cudaMemcpy(out, dout.p, n * sizeof(int16_t), cudaMemcpyDeviceToHost));
    return APT_OK;
}

extern "C" int apt_resample_wav(const char *input_path, const char *output_path, uint32_t output_rate, float atten,
                                float delta_w_pi, uint64_t *nout) {
    if (nout) *nout = 0;
    apt_wav_info wi{};
    APT_TRY(apt_wav_info_read(input_path, &wi));
    std::vector<float> x(wi.frames);
    uint64_t n = 0;
    uint32_t rate = 0;
    APT_TRY(apt_wav_load(input_path, x.data(), x.size(), &n, &rate));
    if (rate == 0) return fail(APT_ERR_BAD_ARG, "invalid input rate");
    const float cut_hz = output_rate > rate ? static_cast<float>(rate) / 2.f : static_cast<float>(output_rate) / 2.f;   // dsp.rs:140-149
    apt_filter f{APT_FILTER_LOWPASS, Freq::hz(cut_hz, rate).get_pi_rad(), atten, delta_w_pi};
    uint64_t ny = 0;
    APT_TRY(apt_resample_len(n, rate, output_rate, &f, &ny));
    if (ny == 0)   // resample.rs:46-52
        return fail(APT_ERR_EMPTY_RESULT, "Got zero samples after resampling, audio file too short or output sampling frequency too low");
    std::vector<float> y(ny);
    APT_TRY(apt_resample_with_filter(x.data(), n, rate, output_rate, &f, y.data(), y.size(), &ny));
    std::vector<int16_t> q(ny);
    APT_TRY(apt_quantize_i16(y.data(), ny, q.data()));
    APT_TRY(apt_wav_write_i16(output_path, q.data(), ny, output_rate));
    if (nout) *nout = ny;
    return APT_OK;
}

// ============================================================================= introspection

extern "C" int apt_tile_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_tile_info *info,
                             float *tile_taps, size_t cap_taps, uint32_t *group_xs, size_t cap_groups) {
    if (!taps || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<float> h(taps, taps + ntaps), tt;
    std::vector<u32> xs;
    TilePlan tp{};
    memset(info, 0, sizeof(*info));
    if (!make_tile_plan(l, m, h, tp, tt, xs)) return APT_OK;
    *info = apt_tile_info{1, tp.groups, tp.p_out, tp.p_in, tp.usteps, tp.row_len, tp.qt, tp.smem_bytes, 4,
                          tp.slice_stride, tp.half_taps, tp.shift, tp.iters, tp.group_stride, tp.ctas_per_sm,
                          tp.pair_pitch, tp.halves, tp.rows_per_copy};
    if (tile_taps) memcpy(tile_taps, tt.data(), std::min(cap_taps, tt.size()) * sizeof(float));
    if (group_xs) memcpy(group_xs, xs.data(), std::min(cap_groups, xs.size()) * sizeof(u32));
    return APT_OK;
}

extern "C" int apt_ut_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_ut_info *info, float *stream,
                           size_t cap_stream) {
    if (!taps || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<float> h(taps, taps + ntaps), st;
    UtPlan up{};
    memset(info, 0, sizeof(*info));
    if (!make_ut_plan(l, m, h, up, st)) return APT_OK;
    info->usable = 1;
    info->l = up.l; info->m = up.m; info->np = up.np; info->q = up.q; info->rows_per_block = up.rb; info->vec = up.vec;
    info->back = up.back; info->chunks = up.chunks; info->slot_floats = up.slot_floats; info->slot_stride = up.slot_stride;
    info->nslot = up.nslot; info->warps = up.warps; info->smem_bytes = up.smem_bytes; info->nvec = up.nvec;
    info->stream_b = up.stream_b; info->halo_u0 = up.halo_u0; info->halo_n = up.halo_n; info->chunk_len = kUtChunk;
    for (int p = 0; p < 8; ++p) {
        info->cs[p] = up.cs[p];
        info->ce[p] = up.ce[p];
    }
    if (stream) memcpy(stream, st.data(), std::min(cap_stream, st.size()) * sizeof(float));
    return APT_OK;
}

extern "C" int apt_ph_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_ph_info *info, float *table,
                           size_t cap_table, uint16_t *xs, size_t cap_xs) {
    if (!taps || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<float> h(taps, taps + ntaps), tb;
    std::vector<unsigned short> x;
    PhPlan pp{};
    memset(info, 0, sizeof(*info));
    if (!make_ph_plan(l, m, h, pp, tb, x)) return APT_OK;
    *info = apt_ph_info{1, pp.l, pp.m, pp.j, pp.jpad, pp.pitch, pp.row_len, pp.smem_bytes};
    if (table) memcpy(table, tb.data(), std::min(cap_table, tb.size()) * sizeof(float));
    if (xs) memcpy(xs, x.data(), std::min(cap_xs, x.size()) * sizeof(uint16_t));
    return APT_OK;
}

// ===================================================================================== batch

extern "C" int apt_decoder_poll(apt_decoder *d) {
    if (!d || !d->in_flight) return 1;
    cudaSetDevice(d->device);
    const cudaError_t e = cudaStreamQuery(d->stream);
    if (e == cudaErrorNotReady) return 0;
    return 1;   // finished (or failed: wait() reports it)
}

namespace {

// The image side of apt_decode_batch_image: every decoder runs in process mode; with PNG output each feeder also has a
// PngFeed.
struct BatchImage {
    const apt_process_settings *ps;
    OutPlan plan;                  // plan.png false: the images go to the caller
    std::vector<apt_image_info> *infos;
};

// One feeder's PNG side.  The decoders keep their images on the device (img.keep); at reap the image is copied into a
// free slot of a fixed pool, so the decoder takes its next recording at once.  When the encoder is idle, every ready
// slot forms one group, encoded on the feeder's own stream after the events of the copies; the feeder reads the
// lengths back once the encode's event has fired and copies each file to its caller.
struct PngFeed {
    ImageOut out;                    // plan: the batch's; work and h_ctl: the encode in flight
    u64 slot_bytes = 0;
    unsigned char *pool = nullptr;
    std::vector<int> job;            // per slot: the recording, -1 free
    std::vector<u32> rows;
    std::vector<char> encoding;      // per slot: part of the encode in flight
    std::vector<cudaEvent_t> ready;  // per slot: the copy into it has finished
    std::vector<int> group;          // slots of the encode in flight, in the order of its images
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    int sms = 1;
    size_t max_group = SIZE_MAX;     // the largest group whose workspace could be allocated

    // `slots` slots of `bytes` each; fewer when the device is short of memory, at least one
    int init(int device, int slots, u64 bytes) {
        APT_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        APT_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        APT_CUDA(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
        slot_bytes = (bytes + 255) & ~255ull;
        for (;; slots /= 2) {
            if (cudaMalloc(&pool, slots * slot_bytes) == cudaSuccess) break;
            cudaGetLastError();
            pool = nullptr;
            if (slots == 1) return fail(APT_ERR_CUDA, "out of device memory for the PNG image pool");
        }
        job.assign(slots, -1);
        rows.assign(slots, 0);
        encoding.assign(slots, 0);
        ready.assign(slots, nullptr);
        for (auto &e : ready) APT_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        return APT_OK;
    }
    ~PngFeed() {
        if (stream) cudaStreamSynchronize(stream);
        out.release();
        if (pool) cudaFree(pool);
        for (auto e : ready)
            if (e) cudaEventDestroy(e);
        if (done) cudaEventDestroy(done);
        if (stream) cudaStreamDestroy(stream);
    }
    int free_slot() const {
        for (size_t k = 0; k < job.size(); ++k)
            if (job[k] < 0) return static_cast<int>(k);
        return -1;
    }
    bool busy() const { return !group.empty(); }
    bool pending() const { return std::any_of(job.begin(), job.end(), [](int j) { return j >= 0; }); }
    bool any_ready() const {
        for (size_t k = 0; k < job.size(); ++k)
            if (job[k] >= 0 && !encoding[k]) return true;
        return false;
    }
    // the image of decoder d's finished job (in its img.px) into a free slot, on the decoder's stream
    int put(apt_decoder *d, int jb, u64 bytes) {
        const int k = free_slot();
        if (k < 0) return fail(APT_ERR_CUDA, "no free slot in the PNG image pool");
        if (bytes > slot_bytes) return fail(APT_ERR_CUDA, "image of %llu bytes exceeds the pool's slots", (unsigned long long)bytes);
        APT_CUDA(cudaMemcpyAsync(pool + k * slot_bytes, d->img.px, bytes, cudaMemcpyDeviceToDevice, d->stream));
        APT_CUDA(cudaEventRecord(ready[k], d->stream));
        job[k] = jb;
        rows[k] = static_cast<u32>(bytes / (static_cast<u64>(kPxPerRow) * out.plan.post.bpp));
        return APT_OK;
    }
    // one encode over every ready slot, at most max_group of them
    void launch(std::vector<int> &status) {
        std::vector<int> slots;
        std::vector<PngPlan> plans;
        for (size_t k = 0; k < job.size(); ++k) {
            if (job[k] < 0 || encoding[k]) continue;
            PngPlan p;
            const int st = out.plan.png_plan(rows[k], p);
            if (st != APT_OK) {
                status[job[k]] = st;
                job[k] = -1;
                continue;
            }
            slots.push_back(static_cast<int>(k));
            plans.push_back(p);
        }
        std::vector<const unsigned char *> px;
        for (int k : slots) {
            px.push_back(pool + k * slot_bytes);
            if (cudaStreamWaitEvent(stream, ready[k], 0) != cudaSuccess) {
                for (int j : slots) {
                    status[job[j]] = fail(APT_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(cudaGetLastError()));
                    job[j] = -1;
                }
                return;
            }
        }
        // the workspace first: while it cannot be allocated the group is halved, and the largest group that fitted is
        // remembered so that later launches do not try a larger one again
        size_t g = std::min(slots.size(), max_group);
        for (;;) {
            PngLayout lay;
            int st = png_layout(plans.data(), px.data(), static_cast<u32>(g), lay);
            if (st == APT_OK) st = out.work.reserve(lay);
            if (st == APT_OK) break;
            cudaGetLastError();
            out.work.release();
            if (g == 1) {   // not even one image fits: that recording fails, the rest wait for the next launch
                status[job[slots[0]]] = st;
                job[slots[0]] = -1;
                return;
            }
            g /= 2;         // a smaller group: the rest stay ready for the next launch
            max_group = g;
        }
        int st = out.encode(LaunchCtx{stream, sms}, plans.data(), px.data(), static_cast<u32>(g), nullptr);
        if (st == APT_OK && cudaEventRecord(done, stream) != cudaSuccess)
            st = fail(APT_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(cudaGetLastError()));
        if (st != APT_OK) {   // the encode itself failed: its recordings have that status
            cudaStreamSynchronize(stream);
            for (size_t i = 0; i < g; ++i) {
                status[job[slots[i]]] = st;
                job[slots[i]] = -1;
            }
            return;
        }
        group.assign(slots.begin(), slots.begin() + g);
        for (int k : group) encoding[k] = 1;
    }
    // waits for the encode in flight and copies each file to its caller (or reports the capacity it needs)
    void finish(uint8_t *const *outs, const uint64_t *caps, uint64_t *nouts, std::vector<int> &status) {
        cudaError_t e = cudaEventSynchronize(done);
        for (size_t i = 0; i < group.size(); ++i) {
            const int k = group[i], jb = job[k];
            if (e != cudaSuccess) {
                status[jb] = fail(APT_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
                continue;
            }
            nouts[jb] = out.length(static_cast<u32>(i));
            status[jb] = out.copy_out(static_cast<u32>(i), outs[jb], caps[jb], cudaMemcpyDeviceToHost, stream);
        }
        const cudaError_t es = cudaStreamSynchronize(stream);
        for (size_t i = 0; i < group.size(); ++i) {
            const int k = group[i];
            if (es != cudaSuccess && status[job[k]] == APT_OK)
                status[job[k]] = fail(APT_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(es));
            job[k] = -1;
            encoding[k] = 0;
        }
        group.clear();
    }
};

// Pool slots per feeder with PNG output: enough to group the images of several rounds of decoders, bounded so that the
// pool's memory does not grow with the batch.
constexpr int kPngPoolSlots = 16;

// One feeder thread per device: binds itself to the device's NUMA node, owns `streams_per_device` decoders and one copy
// stager, keeps every decoder busy and reaps the jobs in the order they complete.  Nothing is shared between devices.
// img == nullptr: f32 rows (apt_decode_batch); else process mode, and with img->plan.png the feeder's PngFeed.
int run_batch(const void *const *signals, int format, const uint64_t *lens, int count, uint32_t input_rate, const apt_settings *s,
              int sync, const BatchImage *img, void *const *outs, const uint64_t *caps, uint64_t *nouts, int *statuses,
              const int *devices, int ndevices, int streams_per_device) {
    APT_TRY(require_device());
    int default_device = 0;
    if (!devices || ndevices <= 0) {
        devices = &default_device;
        ndevices = 1;
    }
    if (streams_per_device <= 0) streams_per_device = 4;
    uint64_t max_len = 0;
    for (int i = 0; i < count; ++i) {
        max_len = std::max(max_len, lens[i]);
        nouts[i] = 0;
        if (statuses) statuses[i] = APT_ERR_CUDA;      // overwritten by the job's own status; never left "ok" by default
    }
    std::vector<int> local_status(count, APT_ERR_CUDA);
    std::vector<std::string> messages(ndevices);
    std::vector<int> fatal(ndevices, APT_OK);

    const int streams_wanted = streams_per_device;
    auto feeder = [&](int g) {
        const int device = devices[g];
        int streams_per_device = streams_wanted;       // per feeder: one device running out of memory does not limit the others
        bind_thread_to_device(device);
        std::vector<apt_decoder *> decs;
        std::vector<int> job_of;
        int next = g;                                  // recording i -> device i % G   (SURVEY.md §8e)
        int in_flight = 0;
        std::unique_ptr<PngFeed> feed;
        auto reap = [&](size_t k) {
            uint64_t got = 0;
            int st = apt_decoder_wait(decs[k], &got);
            const int job = job_of[k];
            if (img && st == APT_OK) (*img->infos)[job] = decs[k]->img.info;
            if (feed && st == APT_OK) {
                st = feed->put(decs[k], job, got);
                got = 0;                               // the file's length comes with its encode
                if (st == APT_OK) st = APT_ERR_CUDA;   // until the encode reports
            }
            nouts[job] = got;
            local_status[job] = st;
            job_of[k] = -1;
            --in_flight;
        };
        auto fail_rest = [&](int st) {
            fatal[g] = st;
            messages[g] = apt_last_error();
            for (; next < count; next += ndevices) local_status[next] = st;
        };
        if (img && img->plan.png && next < count) {
            Plan p;
            uint64_t bound = 0;
            int st = make_plan(input_rate, *s, p);
            if (st == APT_OK) st = cudaSetDevice(device) == cudaSuccess ? APT_OK : fail(APT_ERR_CUDA, "cannot select device %d", device);
            if (st == APT_OK) {
                bound = img->plan.px_bytes(std::max<uint64_t>(plan_out_bound(p, max_len), kPxPerRow));
                feed.reset(new PngFeed());
                feed->out.plan = img->plan;
                st = feed->init(device, std::min(kPngPoolSlots, (count - g + ndevices - 1) / ndevices), bound);
            }
            if (st != APT_OK) {
                feed.reset();
                fail_rest(st);
            }
        }
        while (next < count || in_flight > 0 || (feed && feed->pending())) {
            if (feed && feed->busy() && cudaEventQuery(feed->done) != cudaErrorNotReady) {
                feed->finish(reinterpret_cast<uint8_t *const *>(outs), caps, nouts, local_status);
                continue;
            }
            if (feed && !feed->busy() && feed->any_ready()) {
                feed->launch(local_status);
                continue;
            }
            // a free decoder takes the next recording of this device
            size_t free_k = decs.size();
            for (size_t k = 0; k < decs.size(); ++k)
                if (job_of[k] < 0) { free_k = k; break; }
            if (next < count && (free_k < decs.size() || static_cast<int>(decs.size()) < streams_per_device)) {
                if (free_k == decs.size()) {
                    apt_decoder *d = nullptr;
                    int st = take_decoder(device, input_rate, *s, max_len, false, &d);
                    if (st == APT_OK && img) {
                        st = apt_decoder_set_process_mode(d, img->ps);
                        if (st != APT_OK) park_decoder(d, true);
                    }
                    if (st != APT_OK) {
                        if (decs.empty()) { fail_rest(st); continue; }
                        streams_per_device = static_cast<int>(decs.size());   // out of memory: make do with what exists
                        continue;
                    }
                    // one stager (ring + copy threads) serves all decoders of this feeder: the first decoder's own
                    if (decs.empty()) ensure_stager(d);
                    else d->stager = decs[0]->stager;
                    d->img.keep = feed != nullptr;
                    decs.push_back(d);
                    job_of.push_back(-1);
                }
                const int job = next;
                next += ndevices;
                const int st = apt_decoder_submit_host(decs[free_k], signals[job], format, lens[job], sync,
                                                       static_cast<float *>(outs[job]), caps[job]);
                if (st == APT_OK) {
                    job_of[free_k] = job;
                    ++in_flight;
                } else {
                    local_status[job] = st;
                }
                continue;
            }
            if (in_flight > 0 && (!feed || feed->free_slot() >= 0)) {
                // every decoder is busy (or nothing is left to submit): take whichever job has finished, else the oldest
                bool reaped = false;
                for (size_t k = 0; k < decs.size() && !reaped; ++k)
                    if (job_of[k] >= 0 && apt_decoder_poll(decs[k])) { reap(k); reaped = true; }
                if (!reaped) {
                    size_t oldest = decs.size();
                    for (size_t k = 0; k < decs.size(); ++k)
                        if (job_of[k] >= 0 && (oldest == decs.size() || job_of[k] < job_of[oldest])) oldest = k;
                    if (oldest < decs.size()) reap(oldest);
                }
                continue;
            }
            if (feed && feed->busy()) feed->finish(reinterpret_cast<uint8_t *const *>(outs), caps, nouts, local_status);   // the pool is full
        }
        for (auto *d : decs) park_decoder(d, true);   // drains the last copy into the PNG pool
        feed.reset();
    };

    if (ndevices == 1) {
        feeder(0);
    } else {
        std::vector<std::thread> threads;
        for (int g = 0; g < ndevices; ++g) threads.emplace_back(feeder, g);
        for (auto &t : threads) t.join();
    }
    int first_error = APT_OK;
    for (int i = 0; i < count; ++i) {
        if (statuses) statuses[i] = local_status[i];
        if (local_status[i] != APT_OK && first_error == APT_OK) first_error = local_status[i];
    }
    for (int g = 0; g < ndevices; ++g)
        if (fatal[g] != APT_OK) return fail(fatal[g], "device %d: %s", devices[g], messages[g].c_str());
    return first_error;
}

}  // namespace

extern "C" int apt_decode_batch(const void *const *signals, int format, const uint64_t *lens, int count,
                                uint32_t input_rate, const apt_settings *s, int sync, float *const *outs,
                                const uint64_t *caps, uint64_t *nouts, int *statuses, const int *devices, int ndevices,
                                int streams_per_device) {
    if (!signals || !lens || !s || !outs || !caps || !nouts || count < 0)
        return fail(APT_ERR_BAD_ARG, "null argument");
    if (count == 0) return APT_OK;
    return run_batch(signals, format, lens, count, input_rate, s, sync, nullptr, reinterpret_cast<void *const *>(outs), caps, nouts,
                     statuses, devices, ndevices, streams_per_device);
}

extern "C" int apt_decode_batch_image(const void *const *signals, int format, const uint64_t *lens, int count,
                                      uint32_t input_rate, const apt_settings *s, int sync, const apt_process_settings *ps,
                                      const apt_png_settings *png, uint8_t *const *outs, const uint64_t *caps, uint64_t *nouts,
                                      apt_image_info *infos, int *statuses, const int *devices, int ndevices,
                                      int streams_per_device) {
    if (!signals || !lens || !s || !outs || !caps || !nouts || count < 0) return fail(APT_ERR_BAD_ARG, "null argument");
    OutPlan plan;
    APT_TRY(image_plan(ps, png, false, plan));
    {
        Plan p;
        APT_TRY(make_plan(input_rate, *s, p));
        if (!p.work_multiple) {
            if (sync) return fail(APT_ERR_WORK_RATE, "work_rate is not multiple of FINAL_RATE");
            return fail(APT_ERR_BAD_ARG, "the image stage needs rows of 2080 pixels (work_rate multiple of 4160)");
        }
    }
    if (format != APT_F32 && format != APT_PCM16) return fail(APT_ERR_BAD_ARG, "unknown sample format %d", format);
    for (int i = 0; i < count; ++i)
        if (!outs[i]) return fail(APT_ERR_BAD_ARG, "null output of recording %d", i);
    if (count == 0) return APT_OK;
    std::vector<apt_image_info> got(count);
    std::vector<int> st(count, APT_ERR_CUDA);
    const BatchImage bi{ps, plan, &got};
    const int rc = run_batch(signals, format, lens, count, input_rate, s, sync, &bi, reinterpret_cast<void *const *>(outs), caps,
                             nouts, st.data(), devices, ndevices, streams_per_device);
    for (int i = 0; i < count; ++i) {
        if (statuses) statuses[i] = st[i];
        if (infos) infos[i] = st[i] == APT_OK ? got[i] : apt_image_info{};   // as the one-shot calls: info of a success only
    }
    return rc;
}
