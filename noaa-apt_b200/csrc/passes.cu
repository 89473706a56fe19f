// Finding the satellite passes in a long recording (passes.hpp, DESIGN.md §12).
#include "passes.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>

#include "common.hpp"
#include "hostpool.hpp"
#include "kernels_passes.cuh"

using namespace aptb200;

namespace {

inline size_t sample_bytes(int format) { return format == APT_PCM16 ? 2 : 4; }

int require_device() {
    int count = 0;
    const cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    return APT_OK;
}

void free_recording(apt_recording *r) {
    cudaSetDevice(r->device);
    if (r->stream) cudaStreamSynchronize(r->stream);
    r->front.release();
    for (void *p : {r->d_sig, static_cast<void *>(r->d_e), static_cast<void *>(r->d_conv), static_cast<void *>(r->d_scratch),
                    static_cast<void *>(r->d_q)})
        if (p) cudaFree(p);
    if (r->stream) cudaStreamDestroy(r->stream);
    cudaGetLastError();   // an allocation failure leaves nothing behind for the next call to trip over
}

template <typename T>
int device_alloc(apt_recording *r, T *&p, uint64_t count) {
    const uint64_t bytes = std::max<uint64_t>(count, 1) * sizeof(T);
    APT_CUDA(cudaMalloc(reinterpret_cast<void **>(&p), bytes));
    r->device_bytes += bytes;
    return APT_OK;
}

// The chunk geometry of apt_recording_quality.  A chunk is at most the units the decoder's chunked upload puts in one
// staging buffer (APTB200_CHUNK_SAMPLES, default 32 Mi samples), and at least enough for two rows past its first window;
// consecutive chunks share the one row that joins their windows.  The decimating first stage (L = 1) runs in one chunk.
int plan_chunks(apt_recording *r, uint64_t &e_cap, uint64_t &conv_cap) {
    const FrontPlan &f = r->plan.front;
    const uint64_t R = r->row, uo = f.unit_out, units = f.units(r->nwork);
    uint64_t per_chunk = units;
    if (f.chunkable()) {
        uint64_t cap = 32ull << 20;
        if (const char *e = getenv("APTB200_CHUNK_SAMPLES")) cap = std::max<uint64_t>(strtoull(e, nullptr, 10), 1u << 16);
        cap &= ~7ull;
        APT_TRY(f.chunk_units(cap, per_chunk));
        per_chunk = std::max<uint64_t>(per_chunk, (2 * R + uo - 1) / uo + 2);
    }
    const bool conv = r->format == APT_PCM16 && f.wants_f32();
    e_cap = conv_cap = 0;
    r->chunks.clear();
    for (uint64_t w0 = 0; w0 < r->windows;) {
        const uint64_t u0 = w0 * R / uo, u1 = std::min(units, u0 + per_chunk);
        const uint64_t wend = std::min(r->nwork, u1 * uo);
        if (wend / R < w0 + 2) return fail(APT_ERR_BAD_ARG, "internal: pass-search chunk holds no window");
        const uint64_t w1 = std::min(wend / R - 1, r->windows);
        const uint64_t e0 = (u0 * uo) & ~3ull;
        e_cap = std::max(e_cap, wend - e0);
        if (conv) {
            uint64_t xa, xb;
            f.span(u0, u1, r->n, xa, xb);
            conv_cap = std::max<uint64_t>(conv_cap, xb - (xa & ~7ull));
        }
        r->chunks.push_back(PassChunk{u0, u1, e0, w0, w1});
        w0 = w1;
    }
    return APT_OK;
}

}  // namespace

int aptb200::launch_pass_quality(cudaStream_t s, const float *e, uint64_t w0, uint64_t count, uint32_t R, float *q) {
    k_pass_quality<<<static_cast<unsigned>(count), kPassQualityThreads, 0, s>>>(e, w0, R, q);
    APT_CUDA(cudaGetLastError());
    return APT_OK;
}

int aptb200::make_pass_rule(const apt_pass_search *ps, PassRule &r) {
    r = PassRule{};
    if (!ps) return APT_OK;
    for (float v : {ps->enter, ps->exit, ps->max_gap_s, ps->min_length_s})
        if (!std::isfinite(v)) return fail(APT_ERR_BAD_ARG, "pass search: non-finite setting");
    if (ps->max_gap_s < 0.f || ps->min_length_s < 0.f) return fail(APT_ERR_BAD_ARG, "pass search: negative time");
    if (ps->enter != 0.f) r.enter = ps->enter;
    if (ps->exit != 0.f) r.exit = ps->exit;
    if (!(r.exit > 0.f && r.exit <= r.enter && r.enter <= 1.f))
        return fail(APT_ERR_BAD_ARG, "pass search: need 0 < exit <= enter <= 1 (enter %g, exit %g)", (double)r.enter,
                    (double)r.exit);
    if (ps->max_gap_s != 0.f) r.max_gap = static_cast<uint64_t>(std::floor(2.0 * static_cast<double>(ps->max_gap_s)));
    if (ps->min_length_s != 0.f) r.min_length = static_cast<uint64_t>(std::floor(2.0 * static_cast<double>(ps->min_length_s)));
    return APT_OK;
}

extern "C" int apt_recording_create(int device, const void *signal, int format, uint64_t n, uint32_t input_rate,
                                    const apt_settings *s, apt_recording **rec) {
    if (!rec || !s) return fail(APT_ERR_BAD_ARG, "null argument");
    *rec = nullptr;
    if (format != APT_F32 && format != APT_PCM16) return fail(APT_ERR_BAD_ARG, "unknown sample format %d", format);
    if (n == 0 || !signal) return fail(APT_ERR_BAD_ARG, "empty signal");
    std::unique_ptr<apt_recording> r(new (std::nothrow) apt_recording);
    if (!r) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(make_plan(input_rate, *s, r->plan));
    const Plan &p = r->plan;
    if (!p.work_multiple) return fail(APT_ERR_WORK_RATE, "work_rate is not multiple of FINAL_RATE");
    r->format = format;
    r->n = n;
    r->nwork = p.front.work_len(n);
    r->row = p.row;
    r->windows = r->nwork / p.row >= 1 ? r->nwork / p.row - 1 : 0;
    uint64_t e_cap = 0, conv_cap = 0;
    APT_TRY(plan_chunks(r.get(), e_cap, conv_cap));
    APT_TRY(require_device());
    r->device = device;
    APT_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    APT_CUDA(cudaGetDeviceProperties(&prop, device));
    r->sm_count = prop.multiProcessorCount;

    struct Rollback {
        apt_recording *r;
        bool armed = true;
        ~Rollback() {
            if (armed) free_recording(r);
        }
    } rollback{r.get()};

    APT_CUDA(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
    const uint64_t bytes = n * sample_bytes(format);
    char *sig = nullptr;
    APT_TRY(device_alloc(r.get(), sig, bytes));
    r->d_sig = sig;
    APT_TRY(r->front.upload(p.front));
    r->device_bytes += FrontTables::bytes(p.front);
    APT_TRY(device_alloc(r.get(), r->d_e, e_cap));
    if (conv_cap) APT_TRY(device_alloc(r.get(), r->d_conv, conv_cap));
    if (p.front.needs_scratch()) APT_TRY(device_alloc(r.get(), r->d_scratch, r->nwork));
    APT_TRY(device_alloc(r.get(), r->d_q, r->windows));

    // the one upload: pageable buffers through the pinned ring and its copy threads, pinned ones straight
    const std::unique_ptr<HostStager> stager = is_pageable(signal) ? make_stager(device) : nullptr;
    if (stager)
        APT_CUDA(stager->upload(r->d_sig, signal, bytes, r->stream));
    else
        APT_CUDA(cudaMemcpyAsync(r->d_sig, signal, bytes, cudaMemcpyHostToDevice, r->stream));
    APT_CUDA(cudaStreamSynchronize(r->stream));
    rollback.armed = false;
    *rec = r.release();
    return APT_OK;
}

extern "C" void apt_recording_destroy(apt_recording *rec) {
    if (!rec) return;
    free_recording(rec);
    delete rec;
}

extern "C" int apt_recording_get_info(apt_recording *rec, apt_recording_info *info) {
    if (!rec || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    *info = apt_recording_info{rec->n, rec->nwork, rec->windows, rec->device_bytes, rec->plan.input_rate, rec->row};
    return APT_OK;
}

extern "C" int apt_recording_quality(apt_recording *rec, float *q, uint64_t cap, uint64_t *nq) {
    if (!rec || !nq) return fail(APT_ERR_BAD_ARG, "null argument");
    *nq = rec->windows;
    if (!q && cap == 0) return APT_OK;
    if (!q) return fail(APT_ERR_BAD_ARG, "null output");
    if (cap < rec->windows) return fail(APT_ERR_CAPACITY, "q needs room for %llu floats", (unsigned long long)rec->windows);
    if (rec->windows == 0) return APT_OK;
    APT_CUDA(cudaSetDevice(rec->device));
    const Plan &p = rec->plan;
    const FrontPlan &f = p.front;
    const LaunchCtx c{rec->stream, rec->sm_count};
    const bool conv = rec->format == APT_PCM16 && f.wants_f32();
    auto run = [&]() -> int {
        for (const PassChunk &k : rec->chunks) {
            float *e = rec->d_e - k.e0;
            const float *conv_biased = nullptr;
            if (conv) {   // the kernel reads f32: convert this chunk's span, from a 16-byte aligned start
                uint64_t xa, xb;
                f.span(k.u0, k.u1, rec->n, xa, xb);
                xa &= ~7ull;
                APT_TRY(launch_pcm16_to_f32(c, static_cast<const int16_t *>(rec->d_sig) + xa, xb - xa, rec->d_conv));
                conv_biased = rec->d_conv - xa;
            }
            APT_TRY(front_launch(c, f, rec->front, rec->d_sig, rec->format, conv_biased, rec->n, rec->nwork, k.u0, k.u1, true,
                                 p.cosphi2, p.sinphi, rec->d_scratch ? rec->d_scratch - k.e0 : nullptr, e, nullptr));
            APT_TRY(launch_pass_quality(rec->stream, e, k.w0, k.w1 - k.w0, rec->row, rec->d_q));
        }
        APT_CUDA(cudaMemcpyAsync(q, rec->d_q, rec->windows * sizeof(float), cudaMemcpyDeviceToHost, rec->stream));
        APT_CUDA(cudaStreamSynchronize(rec->stream));
        return APT_OK;
    };
    const int st = run();
    if (st != APT_OK) cudaStreamSynchronize(rec->stream);
    return st;
}

extern "C" int apt_find_passes_quality(const float *q, uint64_t nq, uint64_t n, uint32_t input_rate, const apt_pass_search *ps,
                                       apt_pass *out, uint32_t cap, uint32_t *count) {
    if (!count || (nq && !q) || (cap && !out)) return fail(APT_ERR_BAD_ARG, "null argument");
    *count = 0;
    if (input_rate == 0) return fail(APT_ERR_BAD_ARG, "input_rate is 0");
    PassRule rule;
    APT_TRY(make_pass_rule(ps, rule));
    uint32_t total = 0;
    auto keep = [&](const apt_pass_event &e) {
        if (e.kind != APT_PASS_LOS) return;
        if (total < cap) {
            out[total] = e.pass;
            out[total].end = std::min(out[total].end, n);
        }
        ++total;
    };
    PassTracker t(rule, input_rate);
    try {
        for (uint64_t w = 0; w < nq; ++w) t.feed(q[w], keep);
        t.finish(n, keep);
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    *count = total;
    if (total > cap) return fail(APT_ERR_CAPACITY, "%u passes, room for %u", total, cap);
    return APT_OK;
}

extern "C" int apt_pass_tracker_create(uint32_t input_rate, const apt_pass_search *search, apt_pass_tracker **t) {
    if (!t) return fail(APT_ERR_BAD_ARG, "null argument");
    *t = nullptr;
    if (input_rate == 0) return fail(APT_ERR_BAD_ARG, "input_rate is 0");
    PassRule rule;
    APT_TRY(make_pass_rule(search, rule));
    *t = new (std::nothrow) apt_pass_tracker{PassTracker(rule, input_rate)};
    return *t ? APT_OK : fail(APT_ERR_NOMEM, "out of host memory");
}

extern "C" int apt_pass_tracker_feed(apt_pass_tracker *t, const float *q, uint64_t nq, apt_pass_event *events, uint64_t cap,
                                     uint64_t *nev) {
    if (!t || !nev || (nq && (!q || !events))) return fail(APT_ERR_BAD_ARG, "null argument");
    *nev = 0;
    if (cap < 2 * nq) return fail(APT_ERR_CAPACITY, "events needs room for %llu entries", 2ull * (unsigned long long)nq);
    uint64_t k = 0;
    try {
        for (uint64_t w = 0; w < nq; ++w) t->t.feed(q[w], [&](const apt_pass_event &e) { events[k++] = e; });
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    *nev = k;
    return APT_OK;
}

extern "C" int apt_pass_tracker_finish(apt_pass_tracker *t, uint64_t n, apt_pass_event *events, uint64_t cap, uint64_t *nev) {
    if (!t || !nev) return fail(APT_ERR_BAD_ARG, "null argument");
    *nev = 0;
    if (!events || cap < 1) return fail(APT_ERR_CAPACITY, "events needs room for 1 entry");
    uint64_t k = 0;
    t->t.finish(n, [&](const apt_pass_event &e) { events[k++] = e; });
    *nev = k;
    return APT_OK;
}

extern "C" void apt_pass_tracker_destroy(apt_pass_tracker *t) { delete t; }

extern "C" int apt_recording_decode(apt_recording *rec, const apt_pass *ranges, uint32_t count, int sync,
                                    const apt_process_settings *ps, const apt_png_settings *png, void *const *outs,
                                    const uint64_t *caps, uint64_t *nouts, apt_image_info *infos, int *statuses) {
    if (!rec || (count && (!ranges || !outs || !caps || !nouts || !statuses))) return fail(APT_ERR_BAD_ARG, "null argument");
    auto fail_all = [&](int st) {
        for (uint32_t i = 0; i < count; ++i) statuses[i] = st;
        return st;
    };
    for (uint32_t i = 0; i < count; ++i) {
        nouts[i] = 0;
        statuses[i] = APT_ERR_CUDA;   // overwritten by the range's own status; never left "ok" by default
        if (infos) memset(&infos[i], 0, sizeof(infos[i]));
    }
    // every argument error before any device work: the settings rules of apt_process / apt_png_encode, then the ranges
    OutPlan op;
    if (const int st = make_out_plan(ps, png, op); st != APT_OK) return fail_all(st);
    const Plan &p = rec->plan;
    const size_t sb = sample_bytes(rec->format);
    uint64_t max_len = 0, max_out = 0;
    for (uint32_t i = 0; i < count; ++i) {
        const uint64_t a = ranges[i].start, b = ranges[i].end;
        if (a >= b || b > rec->n)
            return fail_all(fail(APT_ERR_BAD_ARG, "range %u [%llu, %llu) is empty or outside the recording's %llu samples", i,
                                 (unsigned long long)a, (unsigned long long)b, (unsigned long long)rec->n));
        if (!outs[i]) return fail_all(fail(APT_ERR_BAD_ARG, "null output %u", i));
        const uint64_t len = b - a;
        const uint64_t need = sync ? (p.front.work_len(len) / p.row) * kPxPerRow : plan_out_bound(p, len);
        uint64_t bytes = 0;
        if (const int st = op.bytes(need, bytes); st != APT_OK) return fail_all(st);
        max_len = std::max(max_len, len);
        max_out = std::max(max_out, bytes);
    }
    if (count == 0) return APT_OK;

    if (cudaSetDevice(rec->device) != cudaSuccess) return fail_all(fail(APT_ERR_CUDA, "cudaSetDevice failed"));
    apt_decoder *d = nullptr;
    void *slice = nullptr, *dout = nullptr;
    auto release = [&]() {
        if (d) park_decoder(d, false);
        if (slice) cudaFree(slice);
        if (dout) cudaFree(dout);
        cudaGetLastError();
    };
    auto setup = [&]() -> int {
        APT_TRY(take_decoder(rec->device, p.input_rate, p.st, max_len, true, &d));
        // each range starts at an arbitrary sample: the decoder gets it at the start of a fresh (256-byte aligned) buffer,
        // as apt_decode's own staging buffer, so that every first-stage kernel sees the alignment it would see there
        APT_CUDA(cudaMalloc(&slice, max_len * sb));
        APT_CUDA(cudaMalloc(&dout, std::max<uint64_t>(max_out, 1)));
        if (ps) APT_TRY(apt_decoder_set_process_mode(d, ps));
        if (png) APT_TRY(apt_decoder_set_png_mode(d, png));
        return APT_OK;
    };
    if (const int st = setup(); st != APT_OK) {
        release();
        return fail_all(st);
    }
    const size_t elem = ps ? 1 : sizeof(float);
    for (uint32_t i = 0; i < count; ++i) {
        const uint64_t len = ranges[i].end - ranges[i].start;
        int st = APT_OK;
        if (cudaMemcpyAsync(slice, static_cast<const char *>(rec->d_sig) + ranges[i].start * sb, len * sb,
                            cudaMemcpyDeviceToDevice, d->stream) != cudaSuccess)
            st = fail(APT_ERR_CUDA, "copying range %u failed", i);
        if (st == APT_OK) st = apt_decoder_submit_device(d, slice, rec->format, len, sync, static_cast<float *>(dout), caps[i]);
        uint64_t got = 0;
        if (st == APT_OK) st = apt_decoder_wait(d, &got);
        if (st == APT_OK || (st == APT_ERR_CAPACITY && png)) nouts[i] = got;
        if (st == APT_OK && cudaMemcpy(outs[i], dout, got * elem, cudaMemcpyDeviceToHost) != cudaSuccess)
            st = fail(APT_ERR_CUDA, "copying the output of range %u failed", i);
        if (st == APT_OK && infos && ps) infos[i] = d->img.info;
        statuses[i] = st;
    }
    release();
    for (uint32_t i = 0; i < count; ++i)
        if (statuses[i] != APT_OK) return statuses[i];
    return APT_OK;
}
