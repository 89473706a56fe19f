// Streaming decoder (include/aptb200.h apt_stream_*, DESIGN.md §9): decode() carried across pushes of audio.
//
// Every step (one slice of at most max_push samples) runs on the stream's own CUDA stream:
//   upload -> resample + envelope of the first-stage units whose input is complete -> low-pass + correlation of the newly
//   final range -> k_stream_sync (roots, seed, orbit walk, rows to gather) -> k_gather_rows_lp -> one copy back.
// The input, envelope and correlation live in windows that keep only what a later step can still read; a window is
// compacted by moving its tail to the front when the tail is shorter than the part dropped (so the move never overlaps).
// With image output (apt_stream_set_process_mode) every round's new rows are also copied into an image buffer on the device,
// and apt_stream_finish_image runs the image stage (post.hpp) and the PNG encoder (png.hpp) on it.
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "aptb200.h"
#include "common.hpp"
#include "decoder.hpp"
#include "filters_host.hpp"
#include "launch.hpp"
#include "stream.hpp"

using namespace aptb200;

namespace {

constexpr uint64_t kHalo = 80;      // envelope samples in front of a low-pass output: 60 taps + the gather's 4-alignment
constexpr uint32_t kRunRing = 256;  // pending peaks as (position, count) runs: a handful are pending in practice

inline uint64_t floor16(uint64_t x) { return x & ~static_cast<uint64_t>(15); }

// Everything the buffers depend on: (plan, sync, max_push).
struct Geom {
    uint64_t G = 0, D = 0, row = 0;
    uint64_t cap_in = 0, cap_e = 0, cap_c = 0, root_cap = 0, gather_cap = 0;
    uint64_t latency = 0, bytes = 0;
};

int check_stream_args(uint32_t input_rate, const apt_settings *s, int sync, uint64_t max_push, Plan &p) {
    if (!s) return fail(APT_ERR_BAD_ARG, "null settings");
    if (max_push == 0 || max_push > (1ull << 28)) return fail(APT_ERR_BAD_ARG, "max_push %llu outside [1, 2^28]", (unsigned long long)max_push);
    APT_TRY(make_plan(input_rate, *s, p));
    if (!p.work_multiple) {
        if (sync) return fail(APT_ERR_WORK_RATE, "work_rate is not multiple of FINAL_RATE");   // decode.rs:172-176
        return fail(APT_ERR_BAD_ARG, "the stream needs a work rate that is a multiple of 4160 (the final NoFilter resample is "
                                     "not streamed)");
    }
    if (!back_fused(p))
        return fail(APT_ERR_BAD_ARG, "the stream supports the standard, fast and slow demodulation low-pass (37/43/61 taps), "
                                     "not %zu taps at %u samples per pixel", p.lp.size(), p.dec);
    if (sync && p.dist > 16384)
        return fail(APT_ERR_BAD_ARG, "work_rate %u is too high for the sync picker (min_distance %u > 16384)", p.st.work_rate, p.dist);
    return APT_OK;
}

Geom make_geom(const Plan &p, int sync, uint64_t max_push) {
    const FrontPlan &f = p.front;
    Geom g;
    g.G = p.guard.size();
    g.D = p.dist;
    g.row = p.row;
    // input tail: from the next unit's first sample to the end of what was pushed (less than one unit span)
    const uint64_t t_in = f.tail();
    const uint64_t w_new = FrontWindow::step_outputs(f, max_push);
    // envelope tail: a pending row (< row + 1 before work_final) or a pending peak (>= decided >= c_end - D), plus the
    // low-pass halo and the 16-sample alignment of the window start
    const uint64_t t_e = g.row + g.D + g.G + kHalo + 64;
    const uint64_t t_c = g.D + 64;
    g.cap_in = 2 * t_in + max_push + 64;
    g.cap_e = 2 * t_e + w_new + 64;
    g.cap_c = sync ? 2 * t_c + w_new + 64 : 0;
    g.root_cap = sync ? w_new + 2 * g.D + 1024 : 0;
    g.gather_cap = w_new / g.row + 4;
    g.latency = sync ? g.D + 1 : 0;
    const uint64_t rows_floats = (g.gather_cap + 1) * kPxPerRow;
    g.bytes = plan_table_bytes(p) + FrontWindow::bytes(f, g.cap_in, g.cap_e, max_push) +
              (sync ? g.cap_c * 4 + g.root_cap * 4 + kRunRing * 8 + sizeof(StreamCarry) : sizeof(StreamCarry)) +
              g.gather_cap * 4 + rows_floats * 4;
    return g;
}

}  // namespace

struct apt_stream {
    apt_decoder dec;                // plan, device, CUDA stream and filter tables (the other members stay unused)
    int sync = 0;
    Geom g;
    FrontWindow win;                // input and envelope windows and the first stage's progress (max_push audio samples)
    float *d_corr = nullptr, *d_rows = nullptr;
    u32 *d_roots = nullptr, *d_gpos = nullptr;
    char *d_carry = nullptr;        // StreamCarry, then the run ring (kRunRing positions, kRunRing counts)
    char *h_carry = nullptr;        // pinned copy of the same
    float *h_rows = nullptr;        // pinned rows of one round
    // recording state
    uint64_t c_base = 0, c_end = 0;
    uint64_t rows_out = 0, gathered = 0, held_slot = 0;
    bool finished = false;
    std::vector<uint64_t> positions;
    uint64_t runs_seen = 0;         // runs whose peaks are in `positions`

    const StreamCarry &carry() const { return *reinterpret_cast<const StreamCarry *>(h_carry); }
    const u32 *run_pos() const { return reinterpret_cast<const u32 *>(h_carry + sizeof(StreamCarry)); }
    const u32 *run_cnt() const { return run_pos() + kRunRing; }

    // I/Q stream (apt_stream_create_iq): every push is converted into the cf32 window `feed`, which keeps the halo the next
    // audio output reads, and k_fm_demod writes the new audio into the input window, whose counters then count audio samples
    bool iq = false;
    uint64_t iq_max_push = 0;       // I/Q samples one step takes
    IqPlan iqp;
    IqTables iqt;
    IqFeed feed;

    // image output (apt_stream_set_process_mode), on when img_rows is set: the rows of the pass (f32, up to img_max_rows, row
    // r at r * 2080) and what becomes of them, allocated when the mode is set so that push and finish allocate nothing
    float *img_rows = nullptr;
    uint64_t img_max_rows = 0;
    ImageOut img;
};

namespace {

void release_image(apt_stream *st) {
    st->img.release();
    st->img.plan = OutPlan{};
    if (st->img_rows) cudaFree(st->img_rows);
    st->img_rows = nullptr;
    st->img_max_rows = 0;
}

void free_stream(apt_stream *st) {
    cudaSetDevice(st->dec.device);
    if (st->dec.stream) cudaStreamSynchronize(st->dec.stream);
    st->win.release();
    for (void *p : {(void *)st->d_corr, (void *)st->d_rows, (void *)st->d_roots, (void *)st->d_gpos, (void *)st->d_carry})
        if (p) cudaFree(p);
    if (st->h_carry) cudaFreeHost(st->h_carry);
    if (st->h_rows) cudaFreeHost(st->h_rows);
    st->feed.release();
    st->iqt.release();
    release_image(st);
    free_decoder_buffers(&st->dec);
}

int reset_state(apt_stream *st) {
    st->win.clear();
    st->c_base = st->c_end = st->rows_out = st->gathered = st->held_slot = st->runs_seen = 0;
    st->feed.in = st->feed.base = 0;
    st->finished = false;
    st->positions.clear();
    APT_CUDA(cudaSetDevice(st->dec.device));
    APT_CUDA(cudaMemsetAsync(st->d_carry, 0, sizeof(StreamCarry), st->dec.stream));
    APT_TRY(st->win.zero_input(st->dec.stream));
    APT_CUDA(cudaStreamSynchronize(st->dec.stream));
    memset(st->h_carry, 0, sizeof(StreamCarry));
    return APT_OK;
}

// First envelope sample a later step can still read.
uint64_t envelope_keep(const apt_stream *st) {
    if (!st->sync) return st->rows_out * st->g.row;
    const StreamCarry &cy = st->carry();
    uint64_t row_lb;
    if (cy.run_head < cy.run_tail) row_lb = st->run_pos()[cy.run_head % kRunRing];   // known peak, envelope not final yet
    else if (cy.seed_state < 2) row_lb = 0;
    else row_lb = cy.s >= st->c_end ? cy.s : std::max<uint64_t>(cy.s, cy.decided);   // the next peak is >= this
    return std::min(row_lb, floor16(st->c_end));   // the next low-pass / correlation run starts at floor16(c_end)
}

int compact_all(apt_stream *st) {
    const uint64_t ek = envelope_keep(st);
    APT_TRY(st->win.compact(st->dec.stream, st->dec.plan.front, ~0ull, ek > kHalo ? ek - kHalo : 0));
    if (st->sync) {
        const StreamCarry &cy = st->carry();
        APT_TRY(window_compact(st->dec.stream, st->d_corr, st->c_base, cy.seed_state == 0 ? 0 : cy.decided, st->c_end));
    }
    return APT_OK;
}

// Copies rows [rows_out, rel_hi) out of the pinned round buffer (slot 0 = row rows_out) and remembers a row that was
// gathered but is not released yet (its peak is the last one).
void take_rows(apt_stream *st, uint64_t rel_hi, float *rows, uint64_t &nout) {
    const uint64_t n = rel_hi - st->rows_out;
    if (n) memcpy(rows + nout, st->h_rows, n * kPxPerRow * sizeof(float));
    nout += n * kPxPerRow;
    st->held_slot = st->gathered > rel_hi ? st->gathered - 1 - st->rows_out : 0;
    st->rows_out = rel_hi;
}

// Image output: rows [first, end) of the pass, at `src` on the device, into the image buffer.  Rows past max_rows are left
// out; finish_image then refuses the image (the pass has more rows than the buffer).
int keep_rows(apt_stream *st, uint64_t first, uint64_t end, const float *src) {
    end = std::min(end, st->img_max_rows);
    if (first >= end) return APT_OK;
    APT_CUDA(cudaMemcpyAsync(st->img_rows + first * kPxPerRow, src, (end - first) * kPxPerRow * sizeof(float),
                             cudaMemcpyDeviceToDevice, st->dec.stream));
    return APT_OK;
}

// The new audio of one step into the input window: audio pushes from the host or (`on_device`, stream_push_device) from
// the device; I/Q pushes are converted into the cf32 window and every audio sample they complete is demodulated into it.
int upload(apt_stream *st, const void *src, bool on_device, int format, uint64_t n) {
    const LaunchCtx c{st->dec.stream, st->dec.sm_count};
    if (!st->iq) return st->win.push(c, src, on_device, format, n);
    const IqPlan &q = st->iqp;
    APT_TRY(st->feed.push(c, q, st->win.samples_in, src, format, n));
    const uint64_t m1 = q.out_len(st->feed.in), added = m1 - st->win.samples_in;
    APT_TRY(st->win.room(added));
    APT_TRY(iq_launch(c, q, st->iqt, st->feed.origin(), st->feed.base, st->feed.in, APT_CF32, st->win.samples_in, m1,
                      st->win.in_origin()));
    st->win.commit(added);
    return APT_OK;
}

// One step: `n` new samples (maybe none) and, when `finish`, the end of the recording.
int step(apt_stream *st, const void *src, bool on_device, int format, uint64_t n, bool finish, float *rows, uint64_t &nout,
         int &status) {
    apt_decoder &d = st->dec;
    const Plan &p = d.plan;
    const Geom &g = st->g;
    const LaunchCtx c{d.stream, d.sm_count};
    APT_TRY(compact_all(st));
    if (n) APT_TRY(upload(st, src, on_device, format, n));
    const uint64_t nw = p.front.work_len(st->win.samples_in);
    if (finish && nw < 10ull * p.row) {    // decode.rs:79-83
        status = fail(APT_ERR_TOO_SHORT, "Got less than 10 rows of samples, audio file is too short");
        return APT_OK;
    }
    // ---- first stage: the units whose input span is complete (all of them at the end) ----
    const uint64_t work_before = st->win.work_final;
    APT_TRY(st->win.advance(c, p, d.front, finish));
    const uint64_t work_final = st->win.work_final;
    const u32 ntaps = static_cast<u32>(p.lp.size());
    const float *e = st->win.e_origin();
    if (!st->sync) {   // rows r with (r+1)*row <= work_final (decode.rs:141-147)
        const uint64_t r_hi = work_final / p.row;
        while (st->rows_out < r_hi) {
            const uint64_t cnt = std::min<uint64_t>(r_hi - st->rows_out, g.gather_cap);
            APT_TRY(launch_gather_lp(c, e, work_final, nullptr, nullptr, static_cast<u32>(cnt), static_cast<u32>(cnt), p.row, kPxPerRow,
                                     p.dec, p.lp.data(), ntaps, st->d_rows, static_cast<u32>(st->rows_out)));
            if (st->img_rows) APT_TRY(keep_rows(st, st->rows_out, st->rows_out + cnt, st->d_rows));
            APT_CUDA(cudaMemcpyAsync(st->h_rows, st->d_rows, cnt * kPxPerRow * sizeof(float), cudaMemcpyDeviceToHost, d.stream));
            APT_CUDA(cudaStreamSynchronize(d.stream));
            st->gathered = st->rows_out + cnt;
            take_rows(st, st->rows_out + cnt, rows, nout);
        }
        return APT_OK;
    }
    // ---- low-pass + correlation of the newly final range ----
    const uint64_t c_new = finish ? nw - g.G : (work_final > g.G ? work_final - g.G : 0);
    if (!finish && c_new <= st->c_end && work_final == work_before) return APT_OK;   // nothing became final
    if (c_new > st->c_end) {
        const uint64_t lp_base = floor16(st->c_end);
        if (c_new - st->c_base > g.cap_c || (lp_base >= kHalo && lp_base - kHalo < st->win.e_base))
            return fail(APT_ERR_BAD_ARG, "internal: correlation window overflow");
        APT_TRY(launch_lowpass_corr(c, e, work_final, p.lp.data(), ntaps, p.dec, nullptr, st->d_corr - st->c_base, lp_base));
        st->c_end = c_new;
    }
    // ---- picker + gather, in rounds until the walk has gone as far as the final data allow ----
    const size_t carry_bytes = sizeof(StreamCarry) + 2 * kRunRing * sizeof(u32);
    StreamCarry *dcy = reinterpret_cast<StreamCarry *>(st->d_carry);
    for (;;) {
        if (st->held_slot)
            APT_CUDA(cudaMemcpyAsync(st->d_rows, st->d_rows + st->held_slot * kPxPerRow, kPxPerRow * sizeof(float),
                                     cudaMemcpyDeviceToDevice, d.stream));
        st->held_slot = 0;
        const uint64_t held = st->gathered - st->rows_out;
        const StreamCarry before = st->carry();
        StreamSyncArgs a{};
        a.corr = st->d_corr - st->c_base;
        a.c_end = st->c_end;
        a.ncorr = st->c_end;
        a.work_final = work_final;
        a.finish = finish ? 1 : 0;
        a.row = p.row;
        a.dist = p.dist;
        a.run_cap = kRunRing;
        a.gather_cap = static_cast<u32>(g.gather_cap);
        a.root_cap = static_cast<u32>(g.root_cap);
        a.roots = st->d_roots;
        a.run_pos = reinterpret_cast<u32 *>(st->d_carry + sizeof(StreamCarry));
        a.run_cnt = a.run_pos + kRunRing;
        a.gpos = st->d_gpos;
        a.carry = dcy;
        APT_TRY(launch_stream_sync(c, a));
        APT_TRY(launch_gather_lp(c, e, work_final, st->d_gpos, &dcy->gres, 0, static_cast<u32>(g.gather_cap), p.row, kPxPerRow,
                                 p.dec, p.lp.data(), ntaps, st->d_rows + held * kPxPerRow, static_cast<u32>(st->gathered)));
        APT_CUDA(cudaMemcpyAsync(st->h_carry, st->d_carry, carry_bytes, cudaMemcpyDeviceToHost, d.stream));
        APT_CUDA(cudaMemcpyAsync(st->h_rows, st->d_rows, (held + g.gather_cap) * kPxPerRow * sizeof(float), cudaMemcpyDeviceToHost,
                                 d.stream));
        APT_CUDA(cudaStreamSynchronize(d.stream));
        const StreamCarry &cy = st->carry();
        if (cy.status != 0) return fail(APT_ERR_BAD_ARG, "internal: root ring overflow");
        // runs pushed by this launch: their ring entries cannot have been reused yet (a launch pushes at most
        // kRunRing - pending runs, and the pending ones start at or after runs_seen)
        for (; st->runs_seen < cy.run_tail; ++st->runs_seen)
            st->positions.insert(st->positions.end(), st->run_cnt()[st->runs_seen % kRunRing], st->run_pos()[st->runs_seen % kRunRing]);
        if (st->positions.size() != cy.len) return fail(APT_ERR_BAD_ARG, "internal: peak runs and peak count disagree");
        // the round's new rows sit behind the held ones; the copy runs on the stream ahead of the next round's gather
        if (st->img_rows) APT_TRY(keep_rows(st, st->gathered, cy.gathered, st->d_rows + held * kPxPerRow));
        st->gathered = cy.gathered;
        // released: rows whose next peak exists; a failed decode (fewer than 5 peaks at the end) releases nothing more
        const bool failed = finish && cy.len < 5;
        const uint64_t rel_hi = failed ? st->rows_out : std::min<uint64_t>(st->gathered, cy.len > 0 ? cy.len - 1 : 0);
        take_rows(st, std::max(rel_hi, st->rows_out), rows, nout);
        if (!cy.more) break;
        if (cy.len == before.len && cy.gathered == before.gathered && cy.run_head == before.run_head)
            return fail(APT_ERR_BAD_ARG, "internal: the picker made no progress");   // never loop on an unchanged carry
    }
    if (finish && st->carry().len < 5)   // decode.rs:112-118
        status = fail(APT_ERR_FEW_SYNC_FRAMES, "Found less than 5 sync frames, audio file is too short or too noisy");
    return APT_OK;
}

// audio samples a push of n samples adds
uint64_t audio_of(const apt_stream *st, uint64_t n) { return st->iq ? st->iqp.out_len(st->feed.in + n) - st->win.samples_in : n; }

uint64_t rows_bound(const apt_stream *st, uint64_t n) {
    const uint64_t nw = st->dec.plan.front.work_len(st->win.samples_in + audio_of(st, n));
    const uint64_t most = nw / st->g.row + 1;
    return most > st->rows_out ? (most - st->rows_out) * kPxPerRow : 0;
}

}  // namespace

extern "C" int apt_stream_geometry(uint32_t input_rate, const apt_settings *s, int sync, uint64_t max_push, apt_stream_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    Plan p;
    APT_TRY(check_stream_args(input_rate, s, sync, max_push, p));
    const Geom g = make_geom(p, sync, max_push);
    *info = apt_stream_info{};
    info->latency_work = g.latency;
    info->max_push = max_push;
    info->device_bytes = g.bytes;
    return APT_OK;
}

namespace {

// The I/Q stream's geometry: its audio stream takes at most max_push / D + 1 audio samples per step; the cf32 window holds
// one step, the halo of the next output (N - 1 + D samples) and the same again so that compaction never overlaps.
int check_iq_stream_args(const apt_iq_settings *is, const apt_settings *s, int sync, uint64_t max_push, IqPlan &q, Plan &p,
                         uint64_t &audio_push) {
    if (!is) return fail(APT_ERR_BAD_ARG, "null I/Q settings");
    if (max_push == 0 || max_push > (1ull << 28)) return fail(APT_ERR_BAD_ARG, "max_push %llu outside [1, 2^28]", (unsigned long long)max_push);
    APT_TRY(make_iq(*is, q));
    audio_push = max_push / q.D + 1;
    return check_stream_args(is->audio_rate, s, sync, audio_push, p);
}

uint64_t iq_bytes(const IqPlan &q, uint64_t max_push) {
    return IqFeed::bytes(q, max_push) + (q.hp.size() + q.W.size()) * sizeof(float);
}

int create(int device, uint32_t input_rate, int sync, uint64_t max_push, std::unique_ptr<apt_stream> &st);

}  // namespace

extern "C" int apt_stream_geometry_iq(const apt_iq_settings *is, const apt_settings *s, int sync, uint64_t max_push,
                                      apt_stream_info *info) {
    if (!info) return fail(APT_ERR_BAD_ARG, "null argument");
    IqPlan q;
    Plan p;
    uint64_t audio_push = 0;
    APT_TRY(check_iq_stream_args(is, s, sync, max_push, q, p, audio_push));
    const Geom g = make_geom(p, sync, audio_push);
    *info = apt_stream_info{};
    info->latency_work = g.latency;
    info->max_push = max_push;
    info->device_bytes = g.bytes + iq_bytes(q, max_push);
    return APT_OK;
}

extern "C" int apt_stream_create(int device, uint32_t input_rate, const apt_settings *s, int sync, uint64_t max_push, apt_stream **out) {
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    std::unique_ptr<apt_stream> st(new (std::nothrow) apt_stream);
    if (!st) return fail(APT_ERR_NOMEM, "out of host memory");
    APT_TRY(check_stream_args(input_rate, s, sync, max_push, st->dec.plan));
    APT_TRY(create(device, input_rate, sync, max_push, st));
    *out = st.release();
    return APT_OK;
}

extern "C" int apt_stream_create_iq(int device, const apt_iq_settings *is, const apt_settings *s, int sync, uint64_t max_push,
                                    apt_stream **out) {
    if (!out) return fail(APT_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    std::unique_ptr<apt_stream> st(new (std::nothrow) apt_stream);
    if (!st) return fail(APT_ERR_NOMEM, "out of host memory");
    uint64_t audio_push = 0;
    APT_TRY(check_iq_stream_args(is, s, sync, max_push, st->iqp, st->dec.plan, audio_push));
    st->iq = true;
    st->iq_max_push = max_push;
    APT_TRY(create(device, is->audio_rate, sync, audio_push, st));
    apt_stream *raw = st.get();
    struct Rollback {
        apt_stream *st;
        bool armed = true;
        ~Rollback() {
            if (armed) free_stream(st);
        }
    } rollback{raw};
    APT_TRY(raw->iqt.upload(raw->iqp));
    APT_TRY(raw->feed.alloc(raw->iqp, max_push));
    raw->g.bytes += iq_bytes(raw->iqp, max_push);
    rollback.armed = false;
    *out = st.release();
    return APT_OK;
}

namespace {

// Device side of apt_stream_create once the plan is checked: `max_push` counts audio samples.
int create(int device, uint32_t input_rate, int sync, uint64_t max_push, std::unique_ptr<apt_stream> &st) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device; this library has no CPU fallback");
    }
    const Plan &p = st->dec.plan;
    st->sync = sync ? 1 : 0;
    st->g = make_geom(p, st->sync, max_push);
    const Geom &g = st->g;
    apt_decoder &d = st->dec;
    d.device = device;
    APT_CUDA(cudaSetDevice(device));
    APT_CUDA(cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, device));
    struct Rollback {
        apt_stream *st;
        bool armed = true;
        ~Rollback() {
            if (armed) free_stream(st);
        }
    } rollback{st.get()};
    APT_CUDA(cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking));
    APT_TRY(upload_plan(&d));
    const uint64_t rows_floats = (g.gather_cap + 1) * kPxPerRow;
    APT_TRY(st->win.alloc(p.front, g.cap_in, g.cap_e, max_push));
    const size_t carry_bytes = sizeof(StreamCarry) + (st->sync ? 2 * kRunRing * sizeof(u32) : 0);
    APT_CUDA(cudaMalloc(&st->d_carry, carry_bytes));
    if (st->sync) {
        APT_CUDA(cudaMalloc(&st->d_corr, g.cap_c * sizeof(float)));
        APT_CUDA(cudaMalloc(&st->d_roots, g.root_cap * sizeof(u32)));
    }
    APT_CUDA(cudaMalloc(&st->d_gpos, g.gather_cap * sizeof(u32)));
    APT_CUDA(cudaMalloc(&st->d_rows, rows_floats * sizeof(float)));
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&st->h_carry), sizeof(StreamCarry) + 2 * kRunRing * sizeof(u32), cudaHostAllocDefault));
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&st->h_rows), rows_floats * sizeof(float), cudaHostAllocDefault));
    APT_TRY(reset_state(st.get()));
    rollback.armed = false;
    return APT_OK;
}

}  // namespace

extern "C" void apt_stream_destroy(apt_stream *st) {
    if (!st) return;
    free_stream(st);
    delete st;
}

extern "C" int apt_stream_push_bound(apt_stream *st, uint64_t n, uint64_t *cap_floats) {
    if (!st || !cap_floats) return fail(APT_ERR_BAD_ARG, "null argument");
    *cap_floats = rows_bound(st, n);
    return APT_OK;
}

extern "C" int apt_stream_push(apt_stream *st, const void *samples, int format, uint64_t n, float *rows, uint64_t cap, uint64_t *nout) {
    if (nout) *nout = 0;
    if (!st) return fail(APT_ERR_BAD_ARG, "null stream");
    if (st->finished) return fail(APT_ERR_BAD_ARG, "push after finish: call apt_stream_reset to start a new recording");
    if (st->iq ? !iq_sample_bytes(format) : format != APT_F32 && format != APT_PCM16)
        return fail(APT_ERR_BAD_ARG, "sample format %d is not one this stream takes (%s)", format,
                    st->iq ? "APT_CU8, APT_CS16 or APT_CF32" : "APT_F32 or APT_PCM16");
    if (n == 0) return APT_OK;
    if (!samples) return fail(APT_ERR_BAD_ARG, "null samples");
    if (st->dec.plan.front.work_len(st->win.samples_in + audio_of(st, n)) >= (1ull << 32))
        return fail(APT_ERR_BAD_ARG, "recording too long: the work-rate index would pass 2^32-1");
    const uint64_t need = rows_bound(st, n);
    if (need && (!rows || cap < need)) return fail(APT_ERR_CAPACITY, "rows needs room for %llu floats", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(st->dec.device));
    uint64_t got = 0;
    const size_t sb = st->iq ? iq_sample_bytes(format) : format == APT_PCM16 ? 2 : 4;
    const uint64_t per_step = st->iq ? st->iq_max_push : st->win.max_push;
    int status = APT_OK;
    for (uint64_t done = 0; done < n;) {
        const uint64_t k = std::min(per_step, n - done);
        APT_TRY(step(st, static_cast<const char *>(samples) + done * sb, false, format, k, false, rows, got, status));
        done += k;
    }
    if (nout) *nout = got;
    return status;
}

extern "C" int apt_stream_finish(apt_stream *st, float *rows, uint64_t cap, uint64_t *nout) {
    if (nout) *nout = 0;
    if (!st) return fail(APT_ERR_BAD_ARG, "null stream");
    if (st->finished) return fail(APT_ERR_BAD_ARG, "the stream is already finished");
    if (st->win.samples_in == 0) return fail(APT_ERR_BAD_ARG, "empty signal");   // signal[0] panics in demodulate, dsp.rs:367
    const uint64_t need = rows_bound(st, 0);
    if (need && (!rows || cap < need)) return fail(APT_ERR_CAPACITY, "rows needs room for %llu floats", (unsigned long long)need);
    APT_CUDA(cudaSetDevice(st->dec.device));
    uint64_t got = 0;
    int status = APT_OK;
    APT_TRY(step(st, nullptr, false, APT_F32, 0, true, rows, got, status));
    st->finished = true;
    if (nout) *nout = got;
    return status;
}

namespace {

bool pushed(const apt_stream *st) { return st->win.samples_in || st->feed.in || st->finished; }

// The image of a finished pass from the rows kept on the device: the image stage, in PNG mode the encoder, then the pixels or
// the file to the caller.  One stream synchronisation for pixels, two for a PNG file (its length is read first).
int finish_image(apt_stream *st, uint8_t *image, uint64_t cap, uint64_t *image_n, apt_image_info *info) {
    ImageOut &o = st->img;
    const uint64_t rows = st->rows_out;
    if (rows > st->img_max_rows) {
        if (info) {
            *info = apt_image_info{};
            info->rows = rows;
        }
        return fail(APT_ERR_CAPACITY, "the pass has %llu rows, more than the image output's max_rows %llu", (unsigned long long)rows,
                    (unsigned long long)st->img_max_rows);
    }
    apt_decoder &d = st->dec;
    const LaunchCtx c{d.stream, d.sm_count};
    APT_TRY(o.launch(c, st->img_rows, nullptr, static_cast<u32>(rows), static_cast<u32>(st->img_max_rows), nullptr, nullptr));
    const uint64_t px_bytes = o.plan.px_bytes(rows * kPxPerRow);
    if (o.plan.png) APT_TRY(o.encode_px(c, rows, nullptr));
    else if (image && cap >= px_bytes) APT_CUDA(cudaMemcpyAsync(image, o.px, px_bytes, cudaMemcpyDeviceToHost, d.stream));
    APT_CUDA(cudaStreamSynchronize(d.stream));
    APT_TRY(post_result(*o.post.head, info));
    if (!o.plan.png) {
        *image_n = px_bytes;
        return check_room(image, px_bytes, cap);
    }
    *image_n = o.length(0);
    APT_TRY(o.copy_out(0, image, cap, cudaMemcpyDeviceToHost, d.stream));
    APT_CUDA(cudaStreamSynchronize(d.stream));
    return APT_OK;
}

}  // namespace

extern "C" int apt_stream_set_process_mode(apt_stream *st, const apt_process_settings *ps, uint64_t max_rows) {
    if (!st) return fail(APT_ERR_BAD_ARG, "null stream");
    if (pushed(st)) return fail(APT_ERR_BAD_ARG, "image output is set before the first push (after create or reset)");
    OutPlan plan;
    APT_TRY(make_out_plan(ps, nullptr, plan));
    if (ps) {
        if (max_rows == 0) return fail(APT_ERR_BAD_ARG, "max_rows must be at least 1");
        if (max_rows >= (1ull << 32) / kPxPerRow) return fail(APT_ERR_BAD_ARG, "max_rows %llu: image too large", (unsigned long long)max_rows);
    }
    APT_CUDA(cudaSetDevice(st->dec.device));
    APT_CUDA(cudaStreamSynchronize(st->dec.stream));
    release_image(st);   // a new process mode also leaves PNG mode
    if (!ps) return APT_OK;
    struct Rollback {
        apt_stream *st;
        bool armed = true;
        ~Rollback() {
            if (armed) release_image(st);
        }
    } rollback{st};
    ImageOut &o = st->img;
    o.plan = plan;
    st->img_max_rows = max_rows;
    APT_TRY(o.post.alloc(plan.post, static_cast<u32>(max_rows)));
    if (plan.post.palette) APT_TRY(o.post.upload_palette(ps->palette, st->dec.stream));
    APT_CUDA(cudaMalloc(&st->img_rows, max_rows * kPxPerRow * sizeof(float)));
    APT_TRY(o.reserve_px(plan.px_bytes(max_rows * kPxPerRow)));
    APT_TRY(o.reserve_ctl(1));
    rollback.armed = false;
    return APT_OK;
}

extern "C" int apt_stream_set_png_mode(apt_stream *st, const apt_png_settings *png) {
    if (!st) return fail(APT_ERR_BAD_ARG, "null stream");
    if (pushed(st)) return fail(APT_ERR_BAD_ARG, "PNG output is set before the first push (after create or reset)");
    ImageOut &o = st->img;
    OutPlan plan = o.plan;
    PngPlan pp;
    if (png) {
        if (!st->img_rows) return fail(APT_ERR_BAD_ARG, "PNG output needs process mode (apt_stream_set_process_mode)");
        APT_TRY(plan.set_png(png));
        APT_TRY(plan.png_plan(st->img_max_rows, pp));
    }
    APT_CUDA(cudaSetDevice(st->dec.device));
    APT_CUDA(cudaStreamSynchronize(st->dec.stream));
    o.work.release();
    o.plan.png = false;
    if (!png) return APT_OK;
    PngLayout lay;
    int rc = png_layout(&pp, nullptr, 1, lay);
    if (rc == APT_OK) rc = o.work.reserve(lay);
    if (rc != APT_OK) {
        o.work.release();
        return rc;
    }
    o.plan = plan;
    return APT_OK;
}

extern "C" int apt_stream_finish_image(apt_stream *st, float *rows, uint64_t cap, uint64_t *nout, uint8_t *image,
                                       uint64_t image_cap, uint64_t *image_n, apt_image_info *info) {
    if (nout) *nout = 0;
    if (image_n) *image_n = 0;
    if (!st || !image_n) return fail(APT_ERR_BAD_ARG, "null argument");
    if (!st->img_rows) return fail(APT_ERR_BAD_ARG, "the stream has no image output (apt_stream_set_process_mode)");
    APT_TRY(apt_stream_finish(st, rows, cap, nout));
    return finish_image(st, image, image_cap, image_n, info);
}

extern "C" int apt_stream_reset(apt_stream *st) {
    if (!st) return fail(APT_ERR_BAD_ARG, "null stream");
    return reset_state(st);
}

extern "C" int apt_stream_sync_positions(apt_stream *st, uint64_t *positions, size_t cap, size_t *n) {
    if (!st || !n) return fail(APT_ERR_BAD_ARG, "null argument");
    *n = st->positions.size();
    if (!positions) return APT_OK;
    std::copy_n(st->positions.begin(), std::min(cap, st->positions.size()), positions);
    if (cap < st->positions.size()) return fail(APT_ERR_CAPACITY, "positions needs %zu entries", st->positions.size());
    return APT_OK;
}

extern "C" int apt_stream_get_info(apt_stream *st, apt_stream_info *info) {
    if (!st || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    info->samples_in = st->iq ? st->feed.in : st->win.samples_in;
    info->work_final = st->win.work_final;
    info->rows_out = st->rows_out;
    info->peaks = st->positions.size();
    info->latency_work = st->g.latency;
    info->max_push = st->iq ? st->iq_max_push : st->win.max_push;
    info->device_bytes = st->g.bytes + (st->img_rows ? stream_image_bytes(st->img.plan, st->img_max_rows) : 0);
    return APT_OK;
}

// ---- used by the watcher (stream.hpp) ----

int aptb200::stream_push_device(apt_stream *st, const float *d_src, uint64_t n, float *rows, uint64_t cap, uint64_t *nout) {
    *nout = 0;
    if (st->iq || st->finished) return fail(APT_ERR_BAD_ARG, "internal: device push into an I/Q or finished stream");
    if (n == 0) return APT_OK;
    if (st->dec.plan.front.work_len(st->win.samples_in + n) >= (1ull << 32))
        return fail(APT_ERR_BAD_ARG, "recording too long: the work-rate index would pass 2^32-1");
    const uint64_t need = rows_bound(st, n);
    if (need && (!rows || cap < need)) return fail(APT_ERR_CAPACITY, "rows needs room for %llu floats", (unsigned long long)need);
    uint64_t got = 0;
    int status = APT_OK;
    for (uint64_t done = 0; done < n;) {
        const uint64_t k = std::min(st->win.max_push, n - done);
        APT_TRY(step(st, d_src + done, true, APT_F32, k, false, rows, got, status));
        done += k;
    }
    *nout = got;
    return status;
}

cudaStream_t aptb200::stream_cuda(const apt_stream *st) { return st->dec.stream; }

uint64_t aptb200::stream_rows_out(const apt_stream *st) { return st->rows_out; }

uint64_t aptb200::stream_image_bytes(const OutPlan &plan, uint64_t max_rows) {
    return max_rows * kPxPerRow * sizeof(float) + ImageOut::device_bytes(plan, max_rows);
}
