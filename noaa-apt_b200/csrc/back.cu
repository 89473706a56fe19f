// Back half of decode(): kernel choice, buffers, launch sequence, overflow redo and read-back (back.hpp).
#include "back.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.hpp"
#include "decoder.hpp"

namespace aptb200 {

bool back_fused(const Plan &p) { return p.work_multiple && lowpass_corr_supported(static_cast<u32>(p.lp.size()), p.dec); }

BackPlan make_back(const Plan &p, uint64_t max_work) {
    BackPlan b;
    b.max_work = max_work;
    if (getenv("APTB200_SEQUENTIAL_PICK")) {
        b.walk = Walk::Sequential;
    } else if (const char *e = getenv("APTB200_PICK")) {
        if (!strcmp(e, "cluster")) b.walk = Walk::Cluster;
        else if (!strcmp(e, "grid")) b.walk = Walk::Grid;
    }
    const bool fused = back_fused(p) && !getenv("APTB200_GENERIC_LOWPASS");
    b.kind = fused ? BackKind::Hbm : BackKind::Generic;
    if (!p.work_multiple || max_work <= p.guard.size()) return b;
    if (p.dist > 16384) return b;   // k_roots holds two blocks of min_distance floats in shared memory (work_rate <=
                                    // 9 * 4160): decoding with sync is refused at submit, --no-sync still works
    b.can_sync = true;
    b.max_corr = max_work - p.guard.size();
    b.max_blocks = static_cast<u32>((b.max_corr + p.dist - 1) / p.dist);
    b.max_positions = static_cast<u32>(max_work / p.row + 4);
    if (fused && !getenv("APTB200_LEGACY_SYNC")) {
        b.kind = BackKind::Records;
        b.tile_w = records_tile(p.dec);
        b.max_tiles = static_cast<u32>((b.max_corr + b.tile_w - 1) / b.tile_w);
        // Record pool: every tile owns a region of kRegion records (a noisy recording has ~200 per tile of 1920 positions: a
        // third), tiles with more take theirs from a shared overflow area behind the regions (one atomic, rare).  A
        // recording that does not fit even that (silence, ramps: every position a record) is decoded by the exact-order Hbm
        // kernels (kSyncRedo).  APTB200_RECORD_POOL=<records> shrinks the pool (tests of that path): no regions then.
        constexpr uint64_t kRegion = 640;
        uint64_t region = kRegion;
        if (const char *e = getenv("APTB200_RECORD_REGION")) region = strtoull(e, nullptr, 10);
        uint64_t cap = static_cast<uint64_t>(b.max_tiles) * region + std::max<uint64_t>(b.max_corr / 8, 1u << 16);
        if (const char *e = getenv("APTB200_RECORD_POOL")) {
            cap = std::max<uint64_t>(strtoull(e, nullptr, 10), 64);
            if (static_cast<uint64_t>(b.max_tiles) * region > cap / 2) region = 0;
        }
        if (cap > (1u << 30)) {                  // hours at once: cap the pool, give the regions what is left of it
            cap = 1u << 30;
            region = std::min<uint64_t>(region, cap / 2 / std::max<u32>(b.max_tiles, 1));
        }
        b.pool_cap = static_cast<u32>(cap);
        b.pool_region = static_cast<u32>(region);
    }
    // parallel walks: room for every row-aligned start plus ~63 roots per row (noisy recordings have ~35); beyond that the
    // kernels fall back to the sequential walk by themselves
    b.pick_cap = static_cast<u32>(std::min<uint64_t>(static_cast<uint64_t>(b.max_positions) * 64 + 65536, 1u << 28));
    return b;
}

int BackBuffers::alloc(const Plan &p, const BackPlan &bp) {
    if (bp.can_sync) {
        if (bp.kind == BackKind::Records) {
            APT_CUDA(cudaMalloc(&ctl, sizeof(SyncCtl)));
            APT_CUDA(cudaMemset(ctl, 0, sizeof(SyncCtl)));
            APT_CUDA(cudaMalloc(&desc, static_cast<size_t>(bp.max_tiles) * sizeof(TileDesc)));
            APT_CUDA(cudaMalloc(&pool, static_cast<size_t>(bp.pool_cap) * sizeof(Rec)));
            APT_CUDA(cudaMalloc(&roots, static_cast<size_t>(bp.pool_cap) * sizeof(u32)));
            APT_CUDA(cudaMalloc(&by_id, static_cast<size_t>(bp.pool_cap) * sizeof(u32)));
            APT_CUDA(cudaMalloc(&tile_base, static_cast<size_t>(bp.max_tiles) * sizeof(u32)));
        }
        const u32 count_blocks = std::max(bp.max_blocks, bp.max_tiles);
        APT_CUDA(cudaMalloc(&guard, p.guard.size()));
        APT_CUDA(cudaMemcpy(guard, p.guard.data(), p.guard.size(), cudaMemcpyHostToDevice));
        APT_CUDA(cudaMalloc(&root_count, static_cast<size_t>(count_blocks) * sizeof(u32)));
        APT_CUDA(cudaMalloc(&pos, static_cast<size_t>(bp.max_positions) * sizeof(u32)));
        pos_cap = bp.max_positions;
        APT_CUDA(cudaMalloc(&pick_mem, pick_scratch_bytes(count_blocks, bp.max_positions, bp.pick_cap)));
        pick = pick_scratch_carve(pick_mem, count_blocks, bp.max_positions, bp.pick_cap);
        APT_CUDA(cudaMemset(pick.ticket, 0, 8));
        if (ctl) pick.ticket = &ctl->pad[0];   // zeroed with the control block at the start of every job
    }
    if (bp.kind != BackKind::Records) APT_TRY(ensure_hbm(p, bp));
    APT_CUDA(cudaMalloc(&res, sizeof(SyncResult)));
    APT_CUDA(cudaMemset(res, 0, sizeof(SyncResult)));
    return APT_OK;
}

int BackBuffers::ensure_hbm(const Plan &p, const BackPlan &bp) {
    if (!f) APT_CUDA(cudaMalloc(&f, std::max<uint64_t>(bp.max_work, 1) * sizeof(float)));
    if (p.work_multiple && bp.max_corr) {
        if (!corr) APT_CUDA(cudaMalloc(&corr, bp.max_corr * sizeof(float)));
        if (!root_list) APT_CUDA(cudaMalloc(&root_list, static_cast<size_t>(bp.max_blocks) * p.dist * sizeof(u32)));
    }
    return APT_OK;
}

int BackBuffers::ensure_track(const Plan &p, const BackPlan &bp) {
    if (!f) APT_CUDA(cudaMalloc(&f, std::max<uint64_t>(bp.max_work, 1) * sizeof(float)));
    if (!corr) APT_CUDA(cudaMalloc(&corr, bp.max_corr * sizeof(float)));
    if (!track_back) APT_CUDA(cudaMalloc(&track_back, bp.max_corr));
    if (!track_end) APT_CUDA(cudaMalloc(&track_end, sizeof(u32)));
    const u32 cap = track_positions_cap(bp.max_corr, p.row);
    if (pos_cap < cap) {
        APT_CUDA(cudaFree(pos));
        pos = nullptr;
        pos_cap = 0;
        APT_CUDA(cudaMalloc(&pos, static_cast<size_t>(cap) * sizeof(u32)));
        pos_cap = cap;
    }
    return APT_OK;
}

void BackBuffers::release() {
    for (void *q : {(void *)res, (void *)guard, (void *)pos, (void *)root_count, pick_mem, (void *)ctl, (void *)desc,
                    (void *)pool, (void *)roots, (void *)tile_base, (void *)by_id, (void *)f, (void *)corr, (void *)root_list,
                    (void *)track_back, (void *)track_end})
        if (q) cudaFree(q);
    track_back = nullptr;
    track_end = nullptr;
    pos_cap = 0;
    res = nullptr;
    guard = nullptr;
    pos = root_count = roots = tile_base = by_id = root_list = nullptr;
    pick_mem = nullptr;
    pick = PickScratch{};
    ctl = nullptr;
    desc = nullptr;
    pool = nullptr;
    f = corr = nullptr;
}

namespace {

// Correlation (unless the low-pass kernel wrote it), roots and walk on b.f[0..nwork).
int sync_on_f(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, uint64_t nwork, bool corr_done,
              KernelHook *hook) {
    const u32 glen = static_cast<u32>(p.guard.size());
    const uint64_t ncorr = nwork - glen;
    const u32 nblocks = static_cast<u32>((ncorr + p.dist - 1) / p.dist);
    const Walk walk = bp.walk_for(c);
    if (!corr_done) {
        KernelSlot s(hook, "sync_correlation");
        APT_TRY(launch_corr(c, b.f, ncorr, b.guard, glen, b.corr));
    }
    {
        KernelSlot s(hook, "sync_roots");
        APT_TRY(launch_roots(c, b.corr, ncorr, p.dist, b.root_list, b.root_count, b.res, walk == Walk::Sequential ? nullptr : &b.pick));
    }
    // the walk counts as one launch here, whatever it runs (the Records kind counts each of its kernels)
    KernelSlot s(hook, "sync_pick");
    const u32 *boff = b.pick.block_off;
    const RootIndex ri{b.root_list, b.root_count, boff, nullptr, nullptr, boff + nblocks, p.dist, nblocks};
    return launch_pick(c, ncorr, nwork, p.row, p.dist, ri, b.pos, bp.max_positions, b.res, walk, b.pick);
}

// Hbm and Generic: f (and corr) in HBM.
int launch_hbm(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, BackKind kind, const float *lp,
               const float *one, const float *e, uint64_t nwork, bool sync, float *rows, KernelHook *hook) {
    APT_TRY(b.ensure_hbm(p, bp));
    const u32 ntaps = static_cast<u32>(p.lp.size());
    if (kind == BackKind::Hbm) {
        // low-pass and (when syncing) the sync cross-correlation in one pass over the envelope
        KernelSlot s(hook, sync ? "lowpass_correlation" : "lowpass");
        APT_TRY(launch_lowpass_corr(c, e, nwork, p.lp.data(), ntaps, p.dec, b.f, sync ? b.corr : nullptr));
    } else {
        KernelSlot s(hook, "lowpass");
        APT_TRY(launch_fir_decimate(c, e, APT_F32, lp, ntaps, 1, nwork, b.f));
    }
    if (sync) {
        APT_TRY(sync_on_f(c, p, bp, b, nwork, kind == BackKind::Hbm, hook));
        KernelSlot s(hook, "gather_rows");
        const u32 max_rows = static_cast<u32>(std::min<uint64_t>(nwork / p.row + 1, 1u << 30));
        return launch_gather(c, b.f, b.pos, b.res, 0, max_rows, p.row, kPxPerRow, p.dec, rows);
    }
    const uint64_t nrows = nwork / p.row;                                   // decode.rs:141-147
    if (p.work_multiple) {
        KernelSlot s(hook, "gather_rows");
        return launch_gather(c, b.f, nullptr, b.res, static_cast<u32>(nrows), static_cast<u32>(nrows), p.row, kPxPerRow, p.dec,
                             rows);
    }
    // work_rate is not a multiple of 4160: the final stage is a real L/M resample with the one-tap
    // NoFilter (dsp.rs:79-98), i.e. zero-stuffing then keeping every M-th sample.
    if (p.last.l == 0) return fail(APT_ERR_RESAMPLE_TO_ZERO, "Can't resample to 0Hz");
    if (static_cast<uint64_t>(p.st.work_rate) * p.last.l > UINT32_MAX)
        return fail(APT_ERR_RATE_OVERFLOW, "Can't resample, looks like the sample rates do not have a big divisor "
                                           "in common. input_rate: %u, output_rate: %u", p.st.work_rate, kFinalRate);
    const uint64_t alen = nrows * p.row;
    const uint64_t nout = polyphase_len(alen, p.last.l, p.last.m, 1);
    KernelSlot s(hook, "final_resample");
    return launch_polyphase(c, b.f, APT_F32, alen, one, p.last.l, p.last.m, 0, 0, nout, false, 0.f, 1.f, rows);
}

// Track: f and corr in HBM, the tracked path over corr, rows from f at its positions.
int launch_track(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *lp, const float *e,
                 uint64_t nwork, float *rows, KernelHook *hook) {
    const u32 ntaps = static_cast<u32>(p.lp.size());
    const u32 glen = static_cast<u32>(p.guard.size());
    const uint64_t ncorr = nwork - glen;
    if (bp.kind == BackKind::Generic) {
        {
            KernelSlot s(hook, "lowpass");
            APT_TRY(launch_fir_decimate(c, e, APT_F32, lp, ntaps, 1, nwork, b.f));
        }
        KernelSlot s(hook, "sync_correlation");
        APT_TRY(launch_corr(c, b.f, ncorr, b.guard, glen, b.corr));
    } else {
        KernelSlot s(hook, "lowpass_correlation");
        APT_TRY(launch_lowpass_corr(c, e, nwork, p.lp.data(), ntaps, p.dec, b.f, b.corr));
    }
    {
        KernelSlot s(hook, "sync_track");
        APT_TRY(launch_sync_track(c, b.corr, ncorr, p.row, bp.track->delta, bp.track->lambda, b.track_back, b.track_end));
    }
    {
        KernelSlot s(hook, "sync_backtrack");
        APT_TRY(launch_track_back(c, b.track_back, b.track_end, ncorr, nwork, p.row, bp.track->delta, b.pos, b.pos_cap, b.res));
    }
    KernelSlot s(hook, "gather_rows");
    const u32 max_rows = static_cast<u32>(std::min<uint64_t>(nwork / p.row + 1, 1u << 30));
    return launch_gather(c, b.f, b.pos, b.res, 0, max_rows, p.row, kPxPerRow, p.dec, rows);
}

// Records: f and corr stay on chip; records -> roots -> orbit -> rows straight from the envelope.
int launch_records(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *e, uint64_t nwork,
                   bool sync, float *rows, KernelHook *hook) {
    const u32 ntaps = static_cast<u32>(p.lp.size());
    if (!sync) {
        const u32 nrows = static_cast<u32>(nwork / p.row);                  // decode.rs:141-147
        KernelSlot s(hook, "gather_rows");
        return launch_gather_lp(c, e, nwork, nullptr, b.res, nrows, nrows, p.row, kPxPerRow, p.dec, p.lp.data(), ntaps, rows);
    }
    APT_CUDA(cudaMemsetAsync(b.ctl, 0, sizeof(SyncCtl), c.stream));
    const u64 ncorr = nwork - p.guard.size();
    const u32 ntiles = static_cast<u32>((ncorr + bp.tile_w - 1) / bp.tile_w);
    {
        KernelSlot s(hook, "lowpass_records");
        APT_TRY(launch_lowpass_records(c, e, nwork, ncorr, p.lp.data(), ntaps, p.dec, b.ctl, b.desc, b.pool, bp.pool_cap,
                                       bp.pool_region, ntiles));
    }
    {
        KernelSlot s(hook, "resolve_roots");
        APT_TRY(launch_resolve_roots(c, b.desc, b.pool, ntiles, bp.tile_w, p.dist, ncorr, b.roots, b.root_count, b.tile_base,
                                     b.by_id, b.ctl, b.res));
    }
    {
        KernelSlot s(hook, "sync_pick");
        const RootIndex ri{b.roots, b.root_count, b.tile_base, b.desc, b.by_id, &b.ctl->root_cursor, bp.tile_w, ntiles};
        int nk = 1;
        APT_TRY(launch_pick(c, ncorr, nwork, p.row, p.dist, ri, b.pos, bp.max_positions, b.res, bp.walk_for(c), b.pick, &nk));
        if (hook) hook->extra(nk - 1);
    }
    KernelSlot s(hook, "gather_rows");
    const u32 max_rows = static_cast<u32>(std::min<uint64_t>(nwork / p.row + 1, 1u << 30));
    return launch_gather_lp(c, e, nwork, b.pos, b.res, 0, max_rows, p.row, kPxPerRow, p.dec, p.lp.data(), ntaps, rows);
}

}  // namespace

int back_launch(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *lp, const float *one,
                const float *e, uint64_t nwork, bool sync, float *rows, KernelHook *hook, BackKind &ran) {
    if (sync && bp.track) {
        ran = BackKind::Track;
        return launch_track(c, p, bp, b, lp, e, nwork, rows, hook);
    }
    ran = bp.kind;
    if (bp.kind == BackKind::Records) return launch_records(c, p, bp, b, e, nwork, sync, rows, hook);
    return launch_hbm(c, p, bp, b, bp.kind, lp, one, e, nwork, sync, rows, hook);
}

int back_redo(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *e, uint64_t nwork,
              float *rows, KernelHook *hook, BackKind &ran) {
    ran = BackKind::Hbm;
    APT_CUDA(cudaMemsetAsync(b.res, 0, sizeof(SyncResult), c.stream));
    return launch_hbm(c, p, bp, b, BackKind::Hbm, nullptr, nullptr, e, nwork, true, rows, hook);
}

int track_settings_check(const apt_track_settings &ts) {
    if (ts.delta < 1 || ts.delta > kTrackMaxDelta)
        return fail(APT_ERR_BAD_ARG, "tracked sync: delta %u is outside 1..%u", ts.delta, kTrackMaxDelta);
    if (!std::isfinite(ts.lambda) || ts.lambda < 0.f)
        return fail(APT_ERR_BAD_ARG, "tracked sync: lambda must be finite and >= 0");
    return APT_OK;
}

int back_set_track(const Plan &p, BackPlan &bp, BackBuffers &b, const apt_track_settings *ts) {
    if (!ts) {
        bp.track.reset();
        return APT_OK;
    }
    APT_TRY(b.ensure_track(p, bp));
    bp.track = TrackPlan{ts->delta, ts->lambda};
    return APT_OK;
}

int back_find_sync(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, uint64_t nwork) {
    return sync_on_f(c, p, bp, b, nwork, false, nullptr);
}

int back_materialise(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *e, uint64_t nwork) {
    APT_TRY(b.ensure_hbm(p, bp));
    APT_TRY(launch_lowpass_corr(c, e, nwork, p.lp.data(), static_cast<u32>(p.lp.size()), p.dec, b.f, b.corr));
    APT_CUDA(cudaStreamSynchronize(c.stream));
    return APT_OK;
}

int back_roots(const Plan &p, const BackPlan &bp, const BackBuffers &b, BackKind ran, uint64_t nwork, uint64_t *roots,
               size_t cap, size_t *nroots) {
    *nroots = 0;
    if (!b.root_count || nwork <= p.guard.size()) return APT_OK;
    const uint64_t ncorr = nwork - p.guard.size();
    if (ran == BackKind::Track) return APT_OK;   // the tracked path has no roots
    const bool tiles = ran == BackKind::Records;
    const u32 block = tiles ? bp.tile_w : p.dist;
    const u32 nb = static_cast<u32>((ncorr + block - 1) / block);
    std::vector<u32> counts(nb);
    APT_CUDA(cudaMemcpy(counts.data(), b.root_count, nb * sizeof(u32), cudaMemcpyDeviceToHost));
    std::vector<TileDesc> desc;
    if (tiles) {
        desc.resize(nb);
        APT_CUDA(cudaMemcpy(desc.data(), b.desc, nb * sizeof(TileDesc), cudaMemcpyDeviceToHost));
    }
    size_t total = 0;
    std::vector<u32> tmp;
    for (u32 k = 0; k < nb; ++k) {
        if (roots && counts[k]) {
            tmp.resize(counts[k]);
            const u32 *src = tiles ? b.roots + desc[k].off : b.root_list + static_cast<size_t>(k) * block;
            APT_CUDA(cudaMemcpy(tmp.data(), src, counts[k] * sizeof(u32), cudaMemcpyDeviceToHost));
            for (u32 i = 0; i < counts[k]; ++i)
                if (total + i < cap) roots[total + i] = tmp[i];
        }
        total += counts[k];
    }
    *nroots = total;
    return APT_OK;
}

int back_records(const Plan &p, const BackPlan &bp, const BackBuffers &b, uint64_t nwork, apt_tile_records *tiles,
                 size_t tiles_cap, size_t *ntiles, apt_record *records, size_t records_cap, size_t *nrecords) {
    *ntiles = *nrecords = 0;
    if (!b.desc || nwork <= p.guard.size()) return APT_OK;
    const uint64_t ncorr = nwork - p.guard.size();
    const u32 nt = static_cast<u32>((ncorr + bp.tile_w - 1) / bp.tile_w);
    std::vector<TileDesc> desc(nt);
    APT_CUDA(cudaMemcpy(desc.data(), b.desc, nt * sizeof(TileDesc), cudaMemcpyDeviceToHost));
    size_t total = 0;
    std::vector<Rec> tmp;
    for (u32 k = 0; k < nt; ++k) {
        const u32 cnt = desc[k].ns + desc[k].np;
        if (k < tiles_cap) tiles[k] = apt_tile_records{desc[k].ns, desc[k].np, desc[k].tmax};
        if (records && cnt && total < records_cap) {
            tmp.resize(cnt);
            APT_CUDA(cudaMemcpy(tmp.data(), b.pool + desc[k].off, cnt * sizeof(Rec), cudaMemcpyDeviceToHost));
            for (u32 i = 0; i < cnt && total + i < records_cap; ++i) records[total + i] = apt_record{tmp[i].pos, tmp[i].val};
        }
        total += cnt;
    }
    *ntiles = nt;
    *nrecords = total;
    return APT_OK;
}

}  // namespace aptb200
