// The back half of decode() (decode.rs:93-162): demodulation low-pass, sync correlation, roots, orbit walk and row gather.
// This module alone knows which kernels serve a plan, which buffers they need, how the roots are laid out and what runs
// after a record-pool overflow; the decoder, apt_find_sync and the read-back functions see a BackPlan and BackBuffers.
#pragma once

#include <cstddef>
#include <cstdint>
#include <optional>

#include "aptb200.h"
#include "launch.hpp"

namespace aptb200 {

struct Plan;

enum class BackKind {
    Records,   // low-pass / pixel width 37/3, 43/4, 61/5 (kernels_sync2.cuh), f and corr never reach HBM: k_lowpass_records ->
               // k_resolve_roots -> walk -> k_gather_rows_lp; without sync k_gather_rows_lp alone
    Hbm,       // the same low-passes with f and corr in HBM: k_lowpass_corr -> k_roots -> walk -> k_gather_rows (without sync
               // k_lowpass_corr writes f only); the redo after a record-pool overflow, and every job under APTB200_LEGACY_SYNC=1
    Generic,   // any low-pass in the reference's summation order: k_fir_decimate_generic -> k_corr_generic -> k_roots -> walk ->
               // k_gather_rows, or final_resample when the work rate is not a multiple of 4160; APTB200_GENERIC_LOWPASS=1
    Track,     // a sync job of a decoder in APT_SYNC_TRACK mode: f and corr as Hbm (Generic: as Generic) -> k_sync_track ->
               // k_track_back -> k_gather_rows; no roots
};

// Tracked-sync settings of a decoder (apt_decoder_set_sync_mode), checked by track_settings_check.
struct TrackPlan {
    u32 delta = 2;
    float lambda = 0.25f;
};
int track_settings_check(const apt_track_settings &ts);

// The Records and Hbm kernels exist for the plan's low-pass (the standard, fast and slow profiles).
bool back_fused(const Plan &p);

// The kind and buffer sizes for recordings of up to max_work work-rate samples.
struct BackPlan {
    BackKind kind = BackKind::Generic;
    bool can_sync = false;         // the picker has buffers: work rate a multiple of 4160, min_distance <= 16384
    std::optional<Walk> walk;      // forced by APTB200_SEQUENTIAL_PICK or APTB200_PICK=cluster|grid
    uint64_t max_work = 0, max_corr = 0;
    u32 max_blocks = 0;            // blocks of min_distance correlation positions (Hbm, Generic)
    u32 max_positions = 0;         // sync positions
    u32 tile_w = 0, max_tiles = 0, pool_cap = 0, pool_region = 0;   // Records: tiles and record pool
    u32 pick_cap = 0;              // candidates of the parallel walks
    std::optional<TrackPlan> track;   // sync jobs run the tracked sync (set by back_set_track)

    // Unless forced: the whole-GPU walk when the device is otherwise idle, the 8-SM cluster walk when other jobs are in flight.
    Walk walk_for(const LaunchCtx &c) const { return walk ? *walk : c.busy ? Walk::Cluster : Walk::Grid; }
};

BackPlan make_back(const Plan &p, uint64_t max_work);

// Device buffers of a BackPlan.
struct BackBuffers {
    SyncResult *res = nullptr;
    int8_t *guard = nullptr;                       // the sync template (can_sync)
    u32 *pos = nullptr, *root_count = nullptr;     // sync positions; roots per block / tile
    void *pick_mem = nullptr;
    PickScratch pick{};                            // carved from pick_mem
    SyncCtl *ctl = nullptr;                        // Records
    TileDesc *desc = nullptr;
    Rec *pool = nullptr;
    u32 *roots = nullptr;                          // roots of tile t at roots + desc[t].off
    u32 *tile_base = nullptr, *by_id = nullptr;    // dense root ids: first id of tile t, position by id
    float *f = nullptr, *corr = nullptr;           // Hbm / Generic, allocated on first use when the kind is Records
    u32 *root_list = nullptr;                      // roots of block b at root_list + b * min_distance
    u32 pos_cap = 0;                               // entries of pos
    int8_t *track_back = nullptr;                  // Track: the chosen d of every correlation index
    u32 *track_end = nullptr;                      // Track: the index the walk back starts from

    BackBuffers() = default;
    BackBuffers(const BackBuffers &) = delete;
    ~BackBuffers() { release(); }
    int alloc(const Plan &p, const BackPlan &bp);      // everything but f / corr / root_list of the Records kind
    int ensure_hbm(const Plan &p, const BackPlan &bp); // f, corr and the per-block root lists
    int ensure_track(const Plan &p, const BackPlan &bp);   // f, corr, back, end and room for the tracked positions
    void release();
};

// The sync mode of later sync jobs: the reference's picker (ts == nullptr) or tracked sync with *ts (already checked);
// tracked sync allocates its buffers here.  Needs bp.can_sync.
int back_set_track(const Plan &p, BackPlan &bp, BackBuffers &b, const apt_track_settings *ts);

// Enqueues the back half of one job: the envelope e (nwork samples) -> rows, with the plan's kind.  lp and one are the
// device copies of the low-pass taps and of the one-tap NoFilter (Generic).  `ran` is the kind whose buffers now hold the
// job's f / corr / roots.
int back_launch(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *lp, const float *one,
                const float *e, uint64_t nwork, bool sync, float *rows, KernelHook *hook, BackKind &ran);
// The sync decode again with the Hbm kernels, after the record pool of a Records job overflowed (kSyncRedo).
int back_redo(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *e, uint64_t nwork,
              float *rows, KernelHook *hook, BackKind &ran);
// decode::find_sync (decode.rs:204-263) on the low-passed signal in b.f[0..nwork): correlation, roots and walk.
int back_find_sync(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, uint64_t nwork);
// f and corr of a Records job, computed now for apt_decoder_read_stage (returns when they are written).
int back_materialise(const LaunchCtx &c, const Plan &p, const BackPlan &bp, BackBuffers &b, const float *e, uint64_t nwork);
// The roots of the last job, ascending, in the layout of the kind that ran it.
int back_roots(const Plan &p, const BackPlan &bp, const BackBuffers &b, BackKind ran, uint64_t nwork, uint64_t *roots,
               size_t cap, size_t *nroots);
// The per-tile output of k_lowpass_records of the last job (a Records sync job whose pool did not overflow): counts and
// maximum of every tile, then its records, suffix list then prefix list, in tile order (apt_decoder_last_records).
int back_records(const Plan &p, const BackPlan &bp, const BackBuffers &b, uint64_t nwork, apt_tile_records *tiles,
                 size_t tiles_cap, size_t *ntiles, apt_record *records, size_t records_cap, size_t *nrecords);

}  // namespace aptb200
