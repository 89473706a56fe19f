// First stage of decode(): kernel choice, device tables, unit geometry and launch, and its streamed windows (front.hpp).
#include "front.hpp"

#include <algorithm>
#include <cstdlib>

#include "common.hpp"
#include "decoder.hpp"

namespace aptb200 {

namespace {

template <typename P, typename T>
int upload_vec(P *&dst, const std::vector<T> &src) {   // dst is set before the copy: release() frees it on failure
    APT_CUDA(cudaMalloc(&dst, src.size() * sizeof(T)));
    APT_CUDA(cudaMemcpy(dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    return APT_OK;
}

}  // namespace

FrontPlan make_front(Ratio r, std::vector<float> taps) {
    const uint64_t l = r.l, m = r.m, off2 = 2 * ((static_cast<uint64_t>(taps.size()) - 1) / 2);
    const FrontPlan f{l == 1 ? FrontKind::Decimate : FrontKind::Generic, r, std::move(taps), off2};
    if (l == 1 || getenv("APTB200_GENERIC_RESAMPLER")) return f;
    FrontPlan t = f;   // every attempt starts from f: a shape that does not fit may leave partial tables behind
    auto chosen = [&t](FrontKind k, uint64_t unit_in, uint64_t unit_out, uint64_t before, uint64_t after) {
        t.kind = k, t.unit_in = unit_in, t.unit_out = unit_out, t.before = before, t.after = after;
        return t;
    };
    if (make_tile_plan(r.l, r.m, t.h, t.tile, t.tile_taps, t.tile_xs)) {   // before: the halo row, one super-period back
        const uint64_t qt = t.tile.qt, p_in = t.tile.p_in;
        return chosen(FrontKind::Tiled, qt * p_in, qt * t.tile.p_out, p_in - t.tile_xs.back(), (qt - 1) * p_in + t.tile.row_len);
    }
    // the uniform-tap kernel only where the tiled one does not fit: without a packed fp32 FMA (sm_90) its one uniform
    // tap load per FMA pair makes it the slower of the two (48 kHz x 900 s: 214 us against 125 us on an H100 SXM at 700 W)
    t = f;
    if (make_ut_plan(r.l, r.m, t.h, t.ut, t.ut_stream))                 // after: a block's span beyond its first row
        return chosen(FrontKind::UniformTap, t.ut.rb * m, t.ut.rb * l, t.ut.back, t.ut.slot_floats - t.ut.back);
    t = f;
    if (make_ph_plan(r.l, r.m, t.h, t.ph, t.ph_table, t.ph_xs))         // a tile: 32 periods, +4 samples of alignment
        return chosen(FrontKind::PhaseMajor, kPhTilePeriods * m, kPhTilePeriods * l, m + 4,
                      (kPhTilePeriods - 1) * m + t.ph.row_len);
    return f;
}

void FrontPlan::span(uint64_t u0, uint64_t u1, uint64_t n, uint64_t &xa, uint64_t &xb) const {
    const uint64_t l = r.l, m = r.m;
    if (kind == FrontKind::Decimate) {                  // out[k] = sum_j x[k*m - j] c[j] (k > j), and e[k] reads r[k-1]
        const uint64_t kfirst = u0 == 0 ? 0 : u0 - 1;
        xa = kfirst * m > h.size() ? kfirst * m - h.size() : 0;
        xb = std::min<uint64_t>(n, u1 * m);             // output k exists once (k+1)*m samples do (decimate, dsp.rs:299-301)
    } else if (tiles()) {
        xa = u0 == 0 ? 0 : u0 * unit_in - before;
        xb = std::min<uint64_t>(n, (u1 - 1) * unit_in + after);
    } else {
        const uint64_t kfirst = u0 == 0 ? 0 : u0 - 1;   // the envelope needs r[k0 - 1]
        xa = (kfirst * m + l - 1) / l;
        xa &= ~static_cast<uint64_t>(7);                // keep 16-byte alignment of PCM16 chunks
        xb = std::min<uint64_t>(n, ((u1 - 1) * m + off2) / l + 1);
    }
}

uint64_t FrontPlan::complete(uint64_t n, uint64_t nwork, bool finish) const {
    if (finish || kind == FrontKind::Decimate) return units(nwork);   // decimate: output k needs samples [.., (k+1)m)
    if (tiles()) return std::min(n >= after ? (n - after) / unit_in + 1 : 0, nwork / unit_out);
    return std::min(n * r.l > off2 ? (n * r.l - off2 - 1) / r.m + 1 : 0, nwork);   // (k*m + off2)/l < n
}

uint64_t FrontPlan::tail() const {
    if (kind == FrontKind::Decimate) return h.size() + 2 * uint64_t{r.m} + 32;
    if (tiles()) return before + after + unit_in + 32;
    return (2 * off2 + 2 * uint64_t{r.m}) / r.l + 32;
}

int FrontPlan::chunk_units(uint64_t cap, uint64_t &per_chunk) const {
    if (tiles()) {
        if (cap < before + after + unit_in + 64) return fail(APT_ERR_BAD_ARG, "chunk too small for one tile");
        per_chunk = (cap - before - after - 64) / unit_in + 1;
    } else {
        const uint64_t halo = off2 / r.l + 4;
        if (cap < 2 * halo + 1024) return fail(APT_ERR_BAD_ARG, "chunk too small for the filter");
        per_chunk = (cap - 2 * halo) * r.l / r.m;
    }
    if (per_chunk == 0) return fail(APT_ERR_BAD_ARG, "chunk too small");
    return APT_OK;
}

int FrontTables::upload(const FrontPlan &f) {
    APT_TRY(upload_vec(h, f.h));
    if (f.kind == FrontKind::Tiled) {
        APT_TRY(upload_vec(table, f.tile_taps));
        return upload_vec(xs, f.tile_xs);
    }
    if (f.kind == FrontKind::PhaseMajor) {
        APT_TRY(upload_vec(table, f.ph_table));
        return upload_vec(xs, f.ph_xs);
    }
    return APT_OK;
}

void FrontTables::release() {
    for (void *p : {static_cast<void *>(h), static_cast<void *>(table), xs})
        if (p) cudaFree(p);
    h = table = nullptr;
    xs = nullptr;
}

uint64_t FrontTables::bytes(const FrontPlan &f) {
    return f.h.size() * sizeof(float) + f.tile_taps.size() * sizeof(float) + f.tile_xs.size() * sizeof(u32) +
           f.ph_table.size() * sizeof(float) + f.ph_xs.size() * sizeof(unsigned short);
}

int front_launch(const LaunchCtx &c, const FrontPlan &f, const FrontTables &t, const void *in, int format, const float *conv,
                 uint64_t n, uint64_t nwork, uint64_t u0, uint64_t u1, bool envelope, float cosphi2, float sinphi,
                 float *scratch, float *out, KernelHook *hook) {
    if (f.kind == FrontKind::Decimate) {
        {
            KernelSlot s(hook, "filter_decimate");
            APT_TRY(launch_fir_decimate(c, in, format, t.h, static_cast<u32>(f.h.size()), f.r.m, u1, envelope ? scratch : out, u0));
        }
        if (!envelope) return APT_OK;
        KernelSlot s(hook, "envelope");
        return launch_envelope(c, scratch, u1, cosphi2, sinphi, out, u0);
    }
    KernelSlot s(hook, kFrontSlot);
    const float *fin = format == APT_F32 ? static_cast<const float *>(in) : conv;
    if (f.kind == FrontKind::Tiled && fin)
        return launch_polyphase_tiled(c, fin, n, t.table, static_cast<const u32 *>(t.xs), f.tile, nwork, u0, u1, envelope,
                                      cosphi2, sinphi, out);
    if (f.kind == FrontKind::UniformTap && fin && (reinterpret_cast<uintptr_t>(fin) & 15) == 0)
        return launch_polyphase_ut(c, fin, n, t.h, f.ut, f.ut_stream, nwork, u0, u1, envelope, cosphi2, sinphi, out);
    if (f.kind == FrontKind::PhaseMajor)   // f32 or PCM16 samples (the cast is part of its row staging)
        return launch_polyphase_ph(c, in, format, n, t.table, static_cast<const unsigned short *>(t.xs), f.ph, nwork, u0, u1,
                                   envelope, cosphi2, sinphi, out);
    return launch_polyphase(c, in, format, n, t.h, f.r.l, f.r.m, f.off2, u0 * f.unit_out, std::min(nwork, u1 * f.unit_out),
                            envelope, cosphi2, sinphi, out);
}

int window_compact(cudaStream_t s, float *buf, uint64_t &base, uint64_t keep, uint64_t end) {
    keep = std::min(keep, end) & ~static_cast<uint64_t>(15);
    if (keep <= base) return APT_OK;
    const uint64_t drop = keep - base, tail = end - keep;
    if (tail > drop) return APT_OK;
    if (tail) APT_CUDA(cudaMemcpyAsync(buf, buf + drop, tail * sizeof(float), cudaMemcpyDeviceToDevice, s));
    base = keep;
    return APT_OK;
}

int FrontWindow::alloc(const FrontPlan &f, uint64_t cap_in, uint64_t cap_e, uint64_t max_push) {
    this->cap_in = cap_in, this->cap_e = cap_e, this->max_push = max_push;
    APT_CUDA(cudaMalloc(&d_in, cap_in * sizeof(float)));
    APT_CUDA(cudaMalloc(&d_pcm, max_push * sizeof(int16_t)));
    APT_CUDA(cudaMalloc(&d_conv, max_push * sizeof(float)));
    APT_CUDA(cudaMalloc(&d_e, cap_e * sizeof(float)));
    if (f.needs_scratch()) APT_CUDA(cudaMalloc(&d_r, cap_e * sizeof(float)));
    return APT_OK;
}

void FrontWindow::release() {
    for (void *p : {(void *)d_in, (void *)d_pcm, (void *)d_conv, (void *)d_e, (void *)d_r})
        if (p) cudaFree(p);
    d_in = d_conv = d_e = d_r = nullptr;
    d_pcm = nullptr;
}

int FrontWindow::zero_input(cudaStream_t s) const {
    APT_CUDA(cudaMemsetAsync(d_in, 0, cap_in * sizeof(float), s));
    return APT_OK;
}

int FrontWindow::compact(cudaStream_t s, const FrontPlan &f, uint64_t keep_in, uint64_t keep_e) {
    uint64_t xa, xb, eb = e_base, rb = e_base;
    f.span(units_done, units_done + 1, ~0ull, xa, xb);
    APT_TRY(window_compact(s, d_in, in_base, std::min(keep_in, xa), samples_in));
    APT_TRY(window_compact(s, d_e, eb, keep_e, work_final));
    if (d_r && eb != e_base) APT_TRY(window_compact(s, d_r, rb, keep_e, work_final));
    e_base = eb;
    return APT_OK;
}

int FrontWindow::room(uint64_t n) const {
    if (samples_in - in_base + n > cap_in) return fail(APT_ERR_BAD_ARG, "internal: input window overflow");
    return APT_OK;
}

int FrontWindow::push(const LaunchCtx &c, const void *src, bool on_device, int format, uint64_t n) {
    APT_TRY(room(n));
    float *dst = d_in + (samples_in - in_base);
    if (on_device) {
        APT_CUDA(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, c.stream));
    } else if (format == APT_PCM16) {
        APT_CUDA(cudaMemcpyAsync(d_pcm, src, n * 2, cudaMemcpyHostToDevice, c.stream));
        APT_TRY(launch_pcm16_to_f32(c, d_pcm, n, d_conv));
        APT_CUDA(cudaMemcpyAsync(dst, d_conv, n * 4, cudaMemcpyDeviceToDevice, c.stream));
    } else {
        APT_CUDA(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyHostToDevice, c.stream));
    }
    commit(n);
    return APT_OK;
}

int FrontWindow::advance(const LaunchCtx &c, const Plan &p, const FrontTables &t, bool finish) {
    const uint64_t nw = p.front.work_len(samples_in), u_hi = p.front.complete(samples_in, nw, finish);
    if (u_hi <= units_done) return APT_OK;
    const uint64_t work_hi = finish ? nw : std::min(nw, u_hi * p.front.unit_out);
    if (work_hi - e_base > cap_e) return fail(APT_ERR_BAD_ARG, "internal: envelope window overflow");
    APT_TRY(front_launch(c, p.front, t, in_origin(), APT_F32, nullptr, samples_in, nw, units_done, u_hi, true, p.cosphi2,
                         p.sinphi, d_r ? d_r - e_base : nullptr, d_e - e_base, nullptr));
    units_done = u_hi;
    work_final = work_hi;
    return APT_OK;
}

}  // namespace aptb200
