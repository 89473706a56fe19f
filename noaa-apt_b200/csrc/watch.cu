// Watching a continuous audio feed for satellite passes (include/aptb200.h apt_watch_*, DESIGN.md §13).
//
// Every step (one slice of at most max_push samples) runs on one CUDA stream, the pass stream's:
//   upload into the f32 input window -> first stage over the units whose input is complete (FrontWindow, front.hpp, as
//   in the streaming decoder) -> k_pass_quality over the windows whose two rows are final -> the new q back to the host ->
//   the pass rule (PassTracker) -> the open group fed device to device from the input window to the pass stream, an
//   apt_stream with the caller's image / PNG output, which is finished at the group's LOS and reset.
// The input window keeps what the pass stream or a later window can still read; the envelope window keeps the rows of the
// next window.  Both are sized at create from the arguments alone.
//
// The I/Q watcher (apt_watch_iq_*, DESIGN.md §14) is one apt_watch per channel on that channel's FM audio.  Its step uploads
// the I/Q slice once into a cf32 window the channels share (IqFeed, the I/Q stream's), demodulates every channel in one
// launch straight into the channels' input windows, and then runs the rest of each channel's step (advance()).  CUDA events
// order the shared stream after each channel's compaction and each channel's stream after the demodulation.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "aptb200.h"
#include "common.hpp"
#include "decoder.hpp"
#include "iq.hpp"
#include "passes.hpp"
#include "png.hpp"
#include "post.hpp"
#include "stream.hpp"

using namespace aptb200;

namespace {


// Work samples after which a segment ends at the next step with no group open (a group still open at 2T is closed).
uint64_t segment_length() {
    if (const char *e = getenv("APTB200_WATCH_SEGMENT")) {
        const uint64_t v = strtoull(e, nullptr, 10);
        if (v > 0) return std::min<uint64_t>(v, 1ull << 31);   // 2T stays within the 2^32 work-index limit
    }
    return 1ull << 31;
}

// Everything apt_watch_create derives from its arguments, on the host.
struct WatchPlan {
    Plan p;
    PassRule rule;
    int sync = 0;
    OutPlan out;                       // out.image: the pass stream's process settings are ps
    apt_process_settings ps{};
    uint64_t max_rows = 0, max_push = 0;
    uint64_t cap_in = 0, cap_e = 0, q_cap = 0, out_bytes = 0, rows_cap = 0;
    uint64_t own_bytes = 0, stream_bytes = 0, latency = 0, step_work = 0, extra_rows = 0;
};

int make_watch_plan(uint32_t input_rate, const apt_settings *s, const apt_watch_settings *ws, WatchPlan &w) {
    if (!s || !ws) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(make_pass_rule(&ws->search, w.rule));
    w.sync = ws->sync ? 1 : 0;
    w.max_rows = ws->max_rows ? ws->max_rows : 2400;
    if (w.max_rows >= (1ull << 32) / kPxPerRow)
        return fail(APT_ERR_BAD_ARG, "max_rows %llu: image too large", (unsigned long long)w.max_rows);
    w.max_push = ws->max_push ? ws->max_push : input_rate;
    APT_TRY(make_out_plan(ws->ps, ws->png, w.out));
    if (ws->ps) w.ps = *ws->ps;
    if (w.out.image) APT_TRY(w.out.bytes(w.max_rows * kPxPerRow, w.out_bytes));
    apt_stream_info si{};
    APT_TRY(apt_stream_geometry(input_rate, s, w.sync, w.max_push, &si));   // the settings the pass stream refuses
    APT_TRY(make_plan(input_rate, *s, w.p));
    const FrontPlan &f = w.p.front;
    const uint64_t R = w.p.row, rate = input_rate;
    if (w.rule.max_gap > (1ull << 32) / (rate / 2 + 1))   // the input window holds max_gap windows of samples
        return fail(APT_ERR_BAD_ARG, "pass search: max_gap_s %g is too long for a watcher's input window", (double)ws->search.max_gap_s);
    // input: with no group open, from the next window's first sample; with one open, from the pass stream's position, at
    // most max_gap + 2 windows behind the next window; either way less than the first stage's unit span behind the last
    // sample.  Compaction moves the tail only when that does not overlap, so the window holds twice that, plus one step.
    const uint64_t t_in = (w.rule.max_gap + 4) * (rate / 2 + 1) + 2 * (f.tail() + f.unit_in) + 64;
    const uint64_t w_new = FrontWindow::step_outputs(f, w.max_push);
    // envelope: the two rows of the next window (k_pass_quality reads nothing else) and the units of one step
    const uint64_t t_e = 2 * R + f.unit_out + 64;
    w.cap_in = 2 * t_in + w.max_push + 64;
    w.cap_e = 2 * t_e + w_new + 64;
    w.q_cap = w_new / R + 4;
    // the pass stream's rows for one push: rows_bound is the rows of everything pushed less the rows released, and a
    // released row lags the newest work sample by the first stage's tail, the sync template, the picker's min_distance
    // and its latency (apt_stream_info.latency_work), and the row the next peak closes
    w.step_work = w_new;
    w.extra_rows = (w_new + f.tail() * f.r.l / f.r.m + f.unit_out + w.p.guard.size() + 2 * w.p.dist + si.latency_work) / R + 8;
    w.rows_cap = (w.max_rows + w.extra_rows) * kPxPerRow;
    w.latency = (f.tail() * f.r.l / f.r.m + f.unit_out + R - 1) / R + 2;
    w.own_bytes = FrontTables::bytes(f) + FrontWindow::bytes(f, w.cap_in, w.cap_e, w.max_push) + w.q_cap * 4;
    w.stream_bytes = si.device_bytes + (w.out.image ? stream_image_bytes(w.out, w.max_rows) : 0);
    return APT_OK;
}

}  // namespace

struct apt_watch {
    WatchPlan wp;
    int device = 0, sm_count = 0;
    apt_watch_cb cb = nullptr;
    void *user = nullptr;
    apt_stream *pass = nullptr;        // the pass stream; its CUDA stream carries every step
    cudaStream_t cs = nullptr;
    FrontTables front;
    FrontWindow win;                   // the segment's input and envelope windows and first-stage progress
    float *d_q = nullptr;
    float *h_q = nullptr, *h_rows = nullptr;   // pinned
    std::vector<uint8_t> h_out;                // the image or PNG file of the last pass
    uint64_t T = 1ull << 31;
    // the feed
    uint64_t seg_start = 0;            // the segment's first sample; the feed holds seg_start + win.samples_in
    PassTracker tracker{PassRule{}, 1};
    bool active = false;               // the pass stream holds the open group's samples [start_of(first), fed)
    bool lost = false;                 // the pass stream's rows outgrew the row buffer: this pass fails, the feed goes on
    uint64_t fed = 0;
    uint32_t passes = 0;
    bool finished = false, in_cb = false;
};

namespace {

void free_watch(apt_watch *w) {
    cudaSetDevice(w->device);
    if (w->cs) cudaStreamSynchronize(w->cs);
    w->win.release();
    if (w->d_q) cudaFree(w->d_q);
    for (void *p : {(void *)w->h_q, (void *)w->h_rows})
        if (p) cudaFreeHost(p);
    w->front.release();
    if (w->pass) apt_stream_destroy(w->pass);
    cudaGetLastError();
}

void clear_segment(apt_watch *w) {
    w->win.clear();
    w->tracker = PassTracker(w->wp.rule, w->wp.p.input_rate);
    w->active = false;
    w->fed = 0;
}

void call(apt_watch *w, const apt_watch_event &e) {
    if (!w->cb) return;
    w->in_cb = true;
    w->cb(&e, w->user);
    w->in_cb = false;
}

// The pass stream's row buffer for its next push: rows land at their place in the pass up to max_rows; beyond, the
// rows past max_rows overwrite each other (the pass is refused its image then).
float *rows_at(apt_watch *w, uint64_t &cap) {
    const uint64_t off = std::min(stream_rows_out(w->pass), w->wp.max_rows) * kPxPerRow;
    cap = w->wp.rows_cap - off;
    return w->h_rows + off;
}

// Feeds the pass stream the input samples [fed, to) of the segment, one max_push slice at a time.
int feed_to(apt_watch *w, uint64_t to) {
    if (to > w->win.samples_in) return fail(APT_ERR_BAD_ARG, "internal: the pass reaches past the samples pushed");
    while (w->fed < to) {
        if (w->fed < w->win.in_base) return fail(APT_ERR_BAD_ARG, "internal: the pass's samples left the input window");
        const uint64_t k = std::min(w->wp.max_push, to - w->fed);
        uint64_t cap = 0, nout = 0, need = 0;
        float *rows = rows_at(w, cap);
        APT_TRY(apt_stream_push_bound(w->pass, k, &need));
        w->lost = w->lost || need > cap;
        if (!w->lost) APT_TRY(stream_push_device(w->pass, w->win.in_origin() + w->fed, k, rows, cap, &nout));
        w->fed += k;
    }
    return APT_OK;
}

void start_pass(apt_watch *w, uint64_t first) {
    if (w->active) return;
    w->active = true;
    w->lost = false;
    w->fed = w->tracker.start_of(first);
}

// The LOS of a kept group: the pass stream is fed to the pass's end and finished, and the callback gets the result.
int los(apt_watch *w, apt_pass_event ev) {
    start_pass(w, ev.pass.first_window);
    APT_TRY(feed_to(w, ev.pass.end));
    apt_watch_event e{};
    uint64_t cap = 0, nout = 0, need = 0;
    float *rows = rows_at(w, cap);
    APT_TRY(apt_stream_push_bound(w->pass, 0, &need));
    if (w->lost || need > cap) {
        e.status = fail(APT_ERR_CAPACITY, "the pass stream held more rows than its buffer of max_rows + %llu rows",
                        (unsigned long long)w->wp.extra_rows);
        e.rows = stream_rows_out(w->pass);   // the rows released before the buffer ran out
    } else if (w->wp.out.image) {
        uint64_t image_n = 0;
        e.status = apt_stream_finish_image(w->pass, rows, cap, &nout, w->h_out.data(), w->h_out.size(), &image_n, &e.info);
        e.rows = stream_rows_out(w->pass);
        if (e.status == APT_OK) {
            e.data = w->h_out.data();
            e.bytes = image_n;
        }
    } else {
        e.status = apt_stream_finish(w->pass, rows, cap, &nout);
        e.rows = stream_rows_out(w->pass);
        if (e.status == APT_OK && e.rows > w->wp.max_rows)
            e.status = fail(APT_ERR_CAPACITY, "the pass has %llu rows, more than max_rows %llu", (unsigned long long)e.rows,
                            (unsigned long long)w->wp.max_rows);
        if (e.status == APT_OK) {
            e.data = w->h_rows;
            e.bytes = e.rows * kPxPerRow * sizeof(float);
        }
    }
    if (e.status == APT_ERR_CUDA || e.status == APT_ERR_NOMEM) return e.status;   // the device failed, not the pass
    ev.pass.start += w->seg_start;
    ev.pass.end += w->seg_start;
    e.ev = ev;
    e.index = w->passes++;
    call(w, e);
    w->active = false;
    return apt_stream_reset(w->pass);
}

int on_event(apt_watch *w, const apt_pass_event &ev) {
    if (ev.kind == APT_PASS_LOS) return los(w, ev);
    apt_watch_event e{};
    e.ev = ev;
    e.ev.pass.start += w->seg_start;
    e.index = w->passes;
    call(w, e);
    return APT_OK;
}

// The start of a step, before its new samples land in the input window: the windows keep only what the first stage, the
// next window and the pass stream can still read.
int prepare(apt_watch *w) {
    // a group that opens in this step starts at or after the next window's first sample, even when the last group's LOS
    // left the pass stream's position past it
    const uint64_t keep_in = std::min<uint64_t>(w->tracker.start_of(w->tracker.next()), w->active ? w->fed : ~0ull);
    return w->win.compact(w->cs, w->wp.p.front, keep_in, w->tracker.next() * w->wp.p.row);
}

// The rest of a step, once its new samples are in the input window and counted in samples_in: the first stage, q of the
// windows whose two rows are final (into q + nq), the rule and the pass stream; when `finish`, the end of the segment.
int advance(apt_watch *w, bool finish, float *q, uint64_t &nq) {
    const WatchPlan &wp = w->wp;
    const Plan &p = wp.p;
    const LaunchCtx c{w->cs, w->sm_count};
    const uint64_t R = p.row;
    if (w->win.samples_in) APT_TRY(w->win.advance(c, p, w->front, finish));
    const uint64_t w0 = w->tracker.next();
    const uint64_t w1 = w->win.work_final / R >= 1 ? w->win.work_final / R - 1 : 0;
    const uint64_t k = w1 > w0 ? w1 - w0 : 0;
    if (k) {
        if (k > wp.q_cap) return fail(APT_ERR_BAD_ARG, "internal: quality buffer overflow");
        APT_TRY(launch_pass_quality(w->cs, w->win.e_origin(), w0, k, static_cast<uint32_t>(R), w->d_q - w0));
        APT_CUDA(cudaMemcpyAsync(w->h_q, w->d_q, k * sizeof(float), cudaMemcpyDeviceToHost, w->cs));
        APT_CUDA(cudaStreamSynchronize(w->cs));
        memcpy(q + nq, w->h_q, k * sizeof(float));
        nq += k;
    }
    // ---- the rule, window by window, and the pass stream ----
    apt_pass_event evs[2];
    int nev = 0;
    auto collect = [&](const apt_pass_event &e) { evs[nev++] = e; };
    for (uint64_t i = 0; i < k; ++i) {
        nev = 0;
        w->tracker.feed(w->h_q[i], collect);
        if (w->tracker.open()) start_pass(w, w->tracker.first());
        for (int j = 0; j < nev; ++j) APT_TRY(on_event(w, evs[j]));
        if (!w->tracker.open() && w->active) {   // a dropped group
            w->active = false;
            APT_TRY(apt_stream_reset(w->pass));
        }
    }
    if (finish) {
        nev = 0;
        w->tracker.finish(w->win.samples_in, collect);
        for (int j = 0; j < nev; ++j) APT_TRY(on_event(w, evs[j]));
        if (w->active) {
            w->active = false;
            APT_TRY(apt_stream_reset(w->pass));
        }
    } else if (w->active) {
        APT_TRY(feed_to(w, w->tracker.end_of(w->tracker.last(), ~0ull)));
    }
    return APT_OK;
}

// One step: n new samples (maybe none) from the host and, when `finish`, the end of the segment.  q receives the new windows.
int step(apt_watch *w, const void *src, int format, uint64_t n, bool finish, float *q, uint64_t &nq) {
    APT_TRY(prepare(w));
    if (n) APT_TRY(w->win.push(LaunchCtx{w->cs, w->sm_count}, src, false, format, n));
    return advance(w, finish, q, nq);
}

// A segment that is long enough ends before the next step: finished as at apt_watch_finish, then a new one starts.
int maybe_roll(apt_watch *w, float *q, uint64_t &nq) {
    const uint64_t nw = w->wp.p.front.work_len(w->win.samples_in);
    // an open group is closed before the step that could take the segment past 2T (T <= 2^31, so work indices stay below
    // 2^32 in the first stage and in the pass stream)
    if (nw < w->T || (w->tracker.open() && nw + w->wp.step_work < 2 * w->T)) return APT_OK;
    APT_TRY(step(w, nullptr, APT_F32, 0, true, q, nq));
    const uint64_t seg_windows = w->wp.p.front.work_len(w->win.samples_in) / w->wp.p.row;
    w->seg_start += w->win.samples_in;
    clear_segment(w);
    apt_watch_event e{};
    e.ev.kind = APT_PASS_SEGMENT;
    e.ev.window = seg_windows >= 1 ? seg_windows - 1 : 0;
    e.ev.pass.start = w->seg_start;
    e.index = w->passes;
    call(w, e);
    return APT_OK;
}

uint64_t q_bound(const apt_watch *w, uint64_t n) {
    const Plan &p = w->wp.p;
    const uint64_t most = p.front.work_len(w->win.samples_in + n) / p.row + 1;
    const uint64_t next = w->tracker.next();
    return (most > next ? most - next : 0) + p.front.work_len(n) / p.row + 2;   // a new segment may start inside the push
}

int reset_feed(apt_watch *w) {
    w->seg_start = 0;
    w->passes = 0;
    w->finished = false;
    clear_segment(w);
    APT_TRY(apt_stream_reset(w->pass));
    APT_TRY(w->win.zero_input(w->cs));
    APT_CUDA(cudaStreamSynchronize(w->cs));
    return APT_OK;
}

}  // namespace

extern "C" int apt_watch_geometry(uint32_t input_rate, const apt_settings *s, const apt_watch_settings *ws, apt_watch_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    WatchPlan wp;
    APT_TRY(make_watch_plan(input_rate, s, ws, wp));
    *info = apt_watch_info{};
    info->device_bytes = wp.own_bytes + wp.stream_bytes;
    info->max_push = wp.max_push;
    info->latency_windows = wp.latency;
    return APT_OK;
}

extern "C" int apt_watch_create(int device, uint32_t input_rate, const apt_settings *s, const apt_watch_settings *ws,
                                apt_watch_cb cb, void *user, apt_watch **out) {
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    std::unique_ptr<apt_watch> w(new (std::nothrow) apt_watch);
    if (!w) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(make_watch_plan(input_rate, s, ws, w->wp));
    const WatchPlan &wp = w->wp;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device; this library has no CPU fallback");
    }
    w->device = device;
    w->cb = cb;
    w->user = user;
    w->T = segment_length();
    struct Rollback {
        apt_watch *w;
        bool armed = true;
        ~Rollback() {
            if (armed) free_watch(w);
        }
    } rollback{w.get()};
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaDeviceGetAttribute(&w->sm_count, cudaDevAttrMultiProcessorCount, device));
    APT_TRY(apt_stream_create(device, input_rate, s, wp.sync, wp.max_push, &w->pass));
    if (wp.out.image) APT_TRY(apt_stream_set_process_mode(w->pass, &wp.ps, wp.max_rows));
    if (wp.out.png) APT_TRY(apt_stream_set_png_mode(w->pass, &wp.out.png_s));
    w->cs = stream_cuda(w->pass);
    APT_TRY(w->front.upload(wp.p.front));
    APT_TRY(w->win.alloc(wp.p.front, wp.cap_in, wp.cap_e, wp.max_push));
    APT_CUDA(cudaMalloc(&w->d_q, wp.q_cap * sizeof(float)));
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&w->h_q), wp.q_cap * sizeof(float), cudaHostAllocDefault));
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&w->h_rows), wp.rows_cap * sizeof(float), cudaHostAllocDefault));
    try {
        w->h_out.resize(std::max<uint64_t>(wp.out_bytes, 1));
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    APT_TRY(reset_feed(w.get()));
    rollback.armed = false;
    *out = w.release();
    return APT_OK;
}

extern "C" void apt_watch_destroy(apt_watch *w) {
    if (!w || w->in_cb) return;
    free_watch(w);
    delete w;
}

extern "C" int apt_watch_push_bound(apt_watch *w, uint64_t n, uint64_t *cap_q) {
    if (!w || !cap_q) return fail(APT_ERR_BAD_ARG, "null argument");
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "a watcher's callback may not call into its own watcher");
    *cap_q = q_bound(w, n);
    return APT_OK;
}

extern "C" int apt_watch_push(apt_watch *w, const void *samples, int format, uint64_t n, float *q, uint64_t cap, uint64_t *nq) {
    if (nq) *nq = 0;
    if (!w || !nq) return fail(APT_ERR_BAD_ARG, "null argument");
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "a watcher's callback may not call into its own watcher");
    if (w->finished) return fail(APT_ERR_BAD_ARG, "push after finish: call apt_watch_reset to start a new feed");
    if (format != APT_F32 && format != APT_PCM16) return fail(APT_ERR_BAD_ARG, "sample format %d is not APT_F32 or APT_PCM16", format);
    if (n == 0) return APT_OK;
    if (!samples) return fail(APT_ERR_BAD_ARG, "null samples");
    const uint64_t need = q_bound(w, n);
    if (!q || cap < need) return fail(APT_ERR_CAPACITY, "q needs room for %llu floats", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(w->device));
    const size_t sb = format == APT_PCM16 ? 2 : 4;
    uint64_t got = 0;
    try {   // the rule's gap buffer is the only host allocation of a step; no exception leaves the C ABI
        for (uint64_t done = 0; done < n;) {
            APT_TRY(maybe_roll(w, q, got));
            const uint64_t k = std::min(w->wp.max_push, n - done);
            APT_TRY(step(w, static_cast<const char *>(samples) + done * sb, format, k, false, q, got));
            done += k;
        }
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    *nq = got;
    return APT_OK;
}

extern "C" int apt_watch_finish(apt_watch *w, float *q, uint64_t cap, uint64_t *nq) {
    if (nq) *nq = 0;
    if (!w || !nq) return fail(APT_ERR_BAD_ARG, "null argument");
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "a watcher's callback may not call into its own watcher");
    if (w->finished) return fail(APT_ERR_BAD_ARG, "the watcher is already finished");
    const uint64_t need = q_bound(w, 0);
    if (!q || cap < need) return fail(APT_ERR_CAPACITY, "q needs room for %llu floats", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(w->device));
    uint64_t got = 0;
    try {
        APT_TRY(step(w, nullptr, APT_F32, 0, true, q, got));
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    w->finished = true;
    *nq = got;
    return APT_OK;
}

extern "C" int apt_watch_reset(apt_watch *w) {
    if (!w) return fail(APT_ERR_BAD_ARG, "null argument");
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "a watcher's callback may not call into its own watcher");
    APT_CUDA(cudaSetDevice(w->device));
    return reset_feed(w);
}

extern "C" int apt_watch_get_info(apt_watch *w, apt_watch_info *info) {
    if (!w || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "a watcher's callback may not call into its own watcher");
    apt_stream_info si{};
    APT_TRY(apt_stream_get_info(w->pass, &si));
    *info = apt_watch_info{};
    info->samples_in = w->seg_start + w->win.samples_in;
    info->segment_start = w->seg_start;
    info->windows = w->tracker.next();
    info->passes = w->passes;
    info->open = w->tracker.open() ? 1 : 0;
    info->device_bytes = w->wp.own_bytes + si.device_bytes;
    info->max_push = w->wp.max_push;
    info->latency_windows = w->wp.latency;
    return APT_OK;
}

// ------------------------------------------------------------------------------------------------------- the I/Q watcher

namespace {

// Everything apt_watch_iq_create derives from its arguments, on the host.
struct WatchIqPlan {
    IqPlan q[APT_WATCH_IQ_MAX_CHANNELS];
    int count = 0;
    uint32_t audio_rate = 0;
    uint64_t max_push = 0;             // I/Q samples per step
    apt_watch_settings wsc{};          // each channel's: max_push = max_push / D + 1 audio samples
    uint64_t shared_bytes = 0, channel_bytes = 0, latency = 0;
};

int make_watch_iq_plan(const apt_iq_settings *iq, const int32_t *offsets, int count, const apt_settings *s,
                       const apt_watch_settings *ws, WatchIqPlan &w) {
    if (!iq || !offsets || !s || !ws) return fail(APT_ERR_BAD_ARG, "null argument");
    if (count < 1 || count > APT_WATCH_IQ_MAX_CHANNELS)
        return fail(APT_ERR_BAD_ARG, "channel count %d outside 1..%d", count, APT_WATCH_IQ_MAX_CHANNELS);
    for (int c = 0; c < count; ++c) {
        apt_iq_settings sc = *iq;
        sc.offset_hz = offsets[c];
        APT_TRY(make_iq(sc, w.q[c]));
    }
    w.count = count;
    w.audio_rate = iq->audio_rate;
    w.max_push = ws->max_push ? ws->max_push : iq->iq_rate;
    if (w.max_push > (1ull << 28)) return fail(APT_ERR_BAD_ARG, "max_push %llu outside [1, 2^28]", (unsigned long long)w.max_push);
    w.wsc = *ws;
    w.wsc.max_push = w.max_push / w.q[0].D + 1;   // the most audio one step of max_push I/Q samples completes
    WatchPlan cp;
    APT_TRY(make_watch_plan(w.audio_rate, s, &w.wsc, cp));
    w.channel_bytes = cp.own_bytes + cp.stream_bytes;
    w.latency = cp.latency;
    w.shared_bytes = IqFeed::bytes(w.q[0], w.max_push) + (w.q[0].hp.size() + count * w.q[0].W.size()) * sizeof(float);
    return APT_OK;
}

}  // namespace

struct apt_watch_iq {
    WatchIqPlan wp;
    int device = 0, sm_count = 0;
    apt_watch_iq_cb cb = nullptr;
    void *user = nullptr;
    cudaStream_t cs = nullptr;         // the shared window's upload, conversion and demodulation
    cudaEvent_t ready[APT_WATCH_IQ_MAX_CHANNELS] = {}, audio = nullptr;
    IqTables t[APT_WATCH_IQ_MAX_CHANNELS];   // t[0] holds the taps, every t[c] its channel's phasors
    IqFeed feed;
    apt_watch *ch[APT_WATCH_IQ_MAX_CHANNELS] = {};
    struct Hop {                       // a channel watcher's callback user data
        apt_watch_iq *w;
        int c;
    } hop[APT_WATCH_IQ_MAX_CHANNELS];
    uint64_t m_done = 0;               // audio samples of every channel since create / reset
    bool finished = false, in_cb = false;
};

namespace {

void iq_event(const apt_watch_event *e, void *user) {
    const apt_watch_iq::Hop *h = static_cast<const apt_watch_iq::Hop *>(user);
    apt_watch_iq *w = h->w;
    if (!w->cb) return;
    w->in_cb = true;
    w->cb(h->c, e, w->user);
    w->in_cb = false;
}

void free_watch_iq(apt_watch_iq *w) {
    cudaSetDevice(w->device);
    if (w->cs) cudaStreamSynchronize(w->cs);
    for (apt_watch *c : w->ch)
        if (c) apt_watch_destroy(c);
    w->feed.release();
    for (IqTables &t : w->t) t.release();
    for (cudaEvent_t e : w->ready)
        if (e) cudaEventDestroy(e);
    if (w->audio) cudaEventDestroy(w->audio);
    if (w->cs) cudaStreamDestroy(w->cs);
    cudaGetLastError();
}

// One step of n I/Q samples (at most max_push): every channel's segment roll first, then the channels' compaction, one upload
// and conversion into the shared window, one demodulation launch into every channel's input window, and each channel's
// advance() in channel order.  Channel c's q go to q + c * cap from got[c] on.
int iq_step(apt_watch_iq *w, const void *src, int format, uint64_t n, float *q, uint64_t cap, uint64_t *got) {
    const int C = w->wp.count;
    for (int c = 0; c < C; ++c) APT_TRY(maybe_roll(w->ch[c], q + c * cap, got[c]));
    for (int c = 0; c < C; ++c) {
        APT_TRY(prepare(w->ch[c]));
        APT_CUDA(cudaEventRecord(w->ready[c], w->ch[c]->cs));
        APT_CUDA(cudaStreamWaitEvent(w->cs, w->ready[c], 0));
    }
    const LaunchCtx lc{w->cs, w->sm_count};
    const IqPlan &p = w->wp.q[0];
    APT_TRY(w->feed.push(lc, p, w->m_done, src, format, n));
    const uint64_t m1 = p.out_len(w->feed.in), added = m1 - w->m_done;
    const IqPlan *pl[APT_WATCH_IQ_MAX_CHANNELS];
    const IqTables *tb[APT_WATCH_IQ_MAX_CHANNELS];
    float *outs[APT_WATCH_IQ_MAX_CHANNELS];
    for (int c = 0; c < C; ++c) {
        apt_watch *a = w->ch[c];
        APT_TRY(a->win.room(added));
        pl[c] = &w->wp.q[c];
        tb[c] = &w->t[c];
        outs[c] = a->win.in_origin() - a->seg_start;   // audio indices are absolute in the kernel, of the segment here
    }
    APT_TRY(iq_launch_channels(lc, pl, tb, C, w->feed.origin(), w->feed.base, w->feed.in, APT_CF32, w->m_done, m1, outs));
    APT_CUDA(cudaEventRecord(w->audio, w->cs));
    w->m_done = m1;
    for (int c = 0; c < C; ++c) {
        apt_watch *a = w->ch[c];
        APT_CUDA(cudaStreamWaitEvent(a->cs, w->audio, 0));
        a->win.commit(added);
        APT_TRY(advance(a, false, q + c * cap, got[c]));
    }
    return APT_OK;
}

uint64_t iq_q_bound(const apt_watch_iq *w, uint64_t n) {
    const uint64_t na = w->wp.q[0].out_len(w->feed.in + n) - w->m_done;
    uint64_t b = 0;
    for (int c = 0; c < w->wp.count; ++c) b = std::max(b, q_bound(w->ch[c], na));
    return b;
}

int iq_guard(const apt_watch_iq *w) {
    if (w->in_cb) return fail(APT_ERR_BAD_ARG, "an I/Q watcher's callback may not call into its own watcher");
    return APT_OK;
}

}  // namespace

extern "C" int apt_watch_iq_geometry(const apt_iq_settings *iq, const int32_t *offsets, int count, const apt_settings *s,
                                     const apt_watch_settings *ws, apt_watch_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    std::unique_ptr<WatchIqPlan> wp(new (std::nothrow) WatchIqPlan);
    if (!wp) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(make_watch_iq_plan(iq, offsets, count, s, ws, *wp));
    *info = apt_watch_info{};
    info->device_bytes = wp->shared_bytes + static_cast<uint64_t>(count) * wp->channel_bytes;
    info->max_push = wp->max_push;
    info->latency_windows = wp->latency;
    return APT_OK;
}

extern "C" int apt_watch_iq_create(int device, const apt_iq_settings *iq, const int32_t *offsets, int count,
                                   const apt_settings *s, const apt_watch_settings *ws, apt_watch_iq_cb cb, void *user,
                                   apt_watch_iq **out) {
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    std::unique_ptr<apt_watch_iq> w(new (std::nothrow) apt_watch_iq);
    if (!w) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(make_watch_iq_plan(iq, offsets, count, s, ws, w->wp));
    const WatchIqPlan &wp = w->wp;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device; this library has no CPU fallback");
    }
    w->device = device;
    w->cb = cb;
    w->user = user;
    struct Rollback {
        apt_watch_iq *w;
        bool armed = true;
        ~Rollback() {
            if (armed) free_watch_iq(w);
        }
    } rollback{w.get()};
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaDeviceGetAttribute(&w->sm_count, cudaDevAttrMultiProcessorCount, device));
    APT_CUDA(cudaStreamCreateWithFlags(&w->cs, cudaStreamNonBlocking));
    APT_CUDA(cudaEventCreateWithFlags(&w->audio, cudaEventDisableTiming));
    for (int c = 0; c < count; ++c) {
        APT_CUDA(cudaEventCreateWithFlags(&w->ready[c], cudaEventDisableTiming));
        APT_TRY(w->t[c].upload(wp.q[c], c == 0));
    }
    APT_TRY(w->feed.alloc(wp.q[0], wp.max_push));
    for (int c = 0; c < count; ++c) {
        w->hop[c] = apt_watch_iq::Hop{w.get(), c};
        APT_TRY(apt_watch_create(device, wp.audio_rate, s, &wp.wsc, iq_event, &w->hop[c], &w->ch[c]));
    }
    rollback.armed = false;
    *out = w.release();
    return APT_OK;
}

extern "C" void apt_watch_iq_destroy(apt_watch_iq *w) {
    if (!w || w->in_cb) return;
    free_watch_iq(w);
    delete w;
}

extern "C" int apt_watch_iq_push_bound(apt_watch_iq *w, uint64_t n, uint64_t *cap_q) {
    if (!w || !cap_q) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(iq_guard(w));
    *cap_q = iq_q_bound(w, n);
    return APT_OK;
}

extern "C" int apt_watch_iq_push(apt_watch_iq *w, const void *iq, int format, uint64_t n, float *q, uint64_t cap, uint64_t *nq) {
    if (!w || !nq) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(iq_guard(w));
    for (int c = 0; c < w->wp.count; ++c) nq[c] = 0;
    if (w->finished) return fail(APT_ERR_BAD_ARG, "push after finish: call apt_watch_iq_reset to start a new feed");
    const size_t sb = iq_sample_bytes(format);
    if (!sb) return fail(APT_ERR_BAD_ARG, "sample format %d is not APT_CU8, APT_CS16 or APT_CF32", format);
    if (n == 0) return APT_OK;
    if (!iq) return fail(APT_ERR_BAD_ARG, "null samples");
    const uint64_t need = iq_q_bound(w, n);
    if (!q || cap < need) return fail(APT_ERR_CAPACITY, "q needs room for %llu floats per channel", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(w->device));
    uint64_t got[APT_WATCH_IQ_MAX_CHANNELS] = {};
    try {   // the rules' gap buffers are the only host allocations of a step; no exception leaves the C ABI
        for (uint64_t done = 0; done < n;) {
            const uint64_t k = std::min(w->wp.max_push, n - done);
            APT_TRY(iq_step(w, static_cast<const char *>(iq) + done * sb, format, k, q, cap, got));
            done += k;
        }
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    for (int c = 0; c < w->wp.count; ++c) nq[c] = got[c];
    return APT_OK;
}

extern "C" int apt_watch_iq_finish(apt_watch_iq *w, float *q, uint64_t cap, uint64_t *nq) {
    if (!w || !nq) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(iq_guard(w));
    for (int c = 0; c < w->wp.count; ++c) nq[c] = 0;
    if (w->finished) return fail(APT_ERR_BAD_ARG, "the I/Q watcher is already finished");
    const uint64_t need = iq_q_bound(w, 0);
    if (!q || cap < need) return fail(APT_ERR_CAPACITY, "q needs room for %llu floats per channel", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(w->device));
    uint64_t got[APT_WATCH_IQ_MAX_CHANNELS] = {};
    try {
        for (int c = 0; c < w->wp.count; ++c) {
            APT_TRY(step(w->ch[c], nullptr, APT_F32, 0, true, q + c * cap, got[c]));
            w->ch[c]->finished = true;
        }
    } catch (const std::bad_alloc &) {
        return fail(APT_ERR_NOMEM, "out of host memory");
    }
    w->finished = true;
    for (int c = 0; c < w->wp.count; ++c) nq[c] = got[c];
    return APT_OK;
}

extern "C" int apt_watch_iq_reset(apt_watch_iq *w) {
    if (!w) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(iq_guard(w));
    APT_CUDA(cudaSetDevice(w->device));
    APT_CUDA(cudaStreamSynchronize(w->cs));
    for (int c = 0; c < w->wp.count; ++c) APT_TRY(reset_feed(w->ch[c]));
    w->feed.in = w->feed.base = 0;
    w->m_done = 0;
    w->finished = false;
    return APT_OK;
}

extern "C" int apt_watch_iq_get_info(apt_watch_iq *w, int channel, apt_watch_info *info) {
    if (!w || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    APT_TRY(iq_guard(w));
    if (channel < 0 || channel >= w->wp.count)
        return fail(APT_ERR_BAD_ARG, "channel %d outside 0..%d", channel, w->wp.count - 1);
    uint64_t bytes = w->wp.shared_bytes;
    for (int c = 0; c < w->wp.count; ++c) {
        apt_watch_info ci{};
        APT_TRY(apt_watch_get_info(w->ch[c], &ci));
        bytes += ci.device_bytes;
    }
    APT_TRY(apt_watch_get_info(w->ch[channel], info));
    info->samples_in = w->feed.in;
    info->device_bytes = bytes;
    info->max_push = w->wp.max_push;
    return APT_OK;
}
