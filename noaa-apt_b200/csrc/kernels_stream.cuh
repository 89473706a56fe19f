// Streamed peak picker (apt_stream, DESIGN.md §9): find_sync (decode.rs:204-263) continued from a device-resident carry
// over the correlation values that became final since the last step.
//
// Each launch is one CTA.  It
//   1. decides the roots (kernels_sync.cuh: p is a root iff no corr[j] > corr[p] for j in (p, p+D]) of every position p whose
//      window is final: p + D < c_end, or p < ncorr at the end of the recording.  Positions are taken in blocks of D
//      aligned to absolute multiples of D; for p in block b the window is the rest of block b (suffix maximum) plus a prefix
//      of block b+1 (prefix maximum), the van Herk / Gil-Werman split of k_roots.  A block that was decided only in part
//      is loaded again by the next step; the work per step is O(new values + 2D).  New roots are appended, ascending, to
//      a ring.
//   2. decides the seed (first i <= D with corr[i] > 0) once corr[0..D] is final, and pushes peak 0.
//   3. walks the orbit of F(s) = max(firstroot(s) + D + 1, row*(s/row + 1)) as pick_sequential does, duplicates at s
//      included, for as long as the start and its first root are decided.  firstroot is a binary search over the live
//      roots, so the walk touches only roots.
//   4. lists the rows whose peak is known and whose envelope is final (p + row < work_final) for k_gather_rows_lp.
// Pending peaks are kept as runs (position, count), so the duplicate pushes of a long rootless stretch take one entry.  When
// the row list is full, or the run ring was full and this launch freed entries, carry.more = 1 and the host runs another
// round; a full ring whose first row is not final yet waits for a later step (no round could make progress).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "kernels_sync.cuh"
#include "launch.hpp"

namespace aptb200 {

constexpr int kStreamThreads = 1024;
constexpr int kStreamChunk = 16;          // positions per thread and block: D <= 16384 (as k_roots)

template <int CHUNK>
__global__ void __launch_bounds__(kStreamThreads, 1) k_stream_sync(const StreamSyncArgs a) {
    extern __shared__ float sm[];          // 2*D floats: block b, block b+1
    __shared__ float s_wf[kStreamThreads / 32];
    __shared__ u32 s_wu[kStreamThreads / 32];
    __shared__ float s_pre[kStreamThreads], s_suf[kStreamThreads];   // inclusive prefix / suffix maxima of the chunks
    __shared__ u32 s_seed, s_total;
    StreamCarry *cy = a.carry;
    const u32 tid = threadIdx.x;
    const float NEG = -INFINITY;
    const u64 D = a.dist;
    const u64 lim = a.finish ? a.ncorr : a.c_end;                // correlation indices that exist / are final
    const u64 dec_hi = a.finish ? a.ncorr : (a.c_end > D ? a.c_end - D : 0);
    u64 decided = cy->decided;
    u64 tail = cy->root_tail;
    const u64 head0 = cy->root_head;

    // ---- 1. roots of [decided, dec_hi) ----
    for (u64 b = decided / D; decided < dec_hi; ++b) {
        const u64 base = b * D;
        for (u32 i = tid; i < 2 * D; i += kStreamThreads) {
            const u64 g = base + i;
            sm[i] = g >= decided && g < lim ? __ldg(a.corr + g) : NEG;   // below `decided`: never read by a pending window
        }
        __syncthreads();
        // chunk [lo, lo + CHUNK) of each block: its maxima go through the CTA scans, the values are read again from the tile
        const u32 lo = tid * CHUNK;
        float cmax_a = NEG, cmax_b = NEG;
#pragma unroll
        for (int c = 0; c < CHUNK; ++c) {
            const u32 i = lo + c;
            cmax_a = fmaxf(cmax_a, i < D ? sm[i] : NEG);
            cmax_b = fmaxf(cmax_b, i < D ? sm[D + i] : NEG);
        }
        auto fmx = [](float x, float y) { return fmaxf(x, y); };
        const float pre_incl = block_scan_incl<kStreamThreads>(cmax_b, NEG, fmx, s_wf);
        const float suf_incl = block_scan_incl_rev<kStreamThreads>(cmax_a, NEG, fmx, s_wf);
        s_pre[tid] = pre_incl;
        s_suf[tid] = suf_incl;
        __syncthreads();
        float pm[CHUNK];                                    // prefix maxima of block b+1 up to lo + c
        float run_b = tid > 0 ? s_pre[tid - 1] : NEG;
#pragma unroll
        for (int c = 0; c < CHUNK; ++c) {
            run_b = fmaxf(run_b, lo + c < D ? sm[D + lo + c] : NEG);
            pm[c] = run_b;
        }
        const u64 p_end = min(base + D, dec_hi);
        u32 flags = 0;
        float run = tid + 1 < kStreamThreads ? s_suf[tid + 1] : NEG;
#pragma unroll
        for (int c = CHUNK - 1; c >= 0; --c) {
            const u64 p = base + lo + c;
            if (lo + c < D) {
                const float v = sm[lo + c];
                const float wmax = fmaxf(run, pm[c]);       // max of corr over (p, p+D]
                if (p >= decided && p < p_end && !(wmax > v)) flags |= 1u << c;
                run = fmaxf(run, v);
            }
        }
        const u32 cnt = __popc(flags);
        const u32 incl = block_scan_incl<kStreamThreads>(cnt, 0u, [](u32 x, u32 y) { return x + y; }, s_wu);
        u64 w = tail + incl - cnt;
#pragma unroll
        for (int c = 0; c < CHUNK; ++c)
            if (flags & (1u << c)) a.roots[w++ % a.root_cap] = static_cast<u32>(base + lo + c);
        if (tid == kStreamThreads - 1) s_total = incl;
        __syncthreads();
        tail += s_total;
        decided = p_end;
        __syncthreads();
    }

    // ---- 2. seed: first i <= D with corr[i] > 0 (decode.rs:208-209, the else-if at :250 while i <= D) ----
    if (cy->seed_state == 0 && (a.finish || a.c_end > D)) {
        if (tid == 0) s_seed = kNoSeed;
        __syncthreads();
        const u64 n = min(D + 1, lim);
        for (u32 i = tid; i < n; i += kStreamThreads)
            if (__ldg(a.corr + i) > 0.f) { atomicMin(&s_seed, i); break; }
        __syncthreads();
        if (tid == 0) {
            cy->seed = s_seed;
            cy->seed_state = 1;
        }
    }
    __syncthreads();
    if (tid != 0) return;

    // ---- 3. the walk (thread 0) ----
    if (head0 + a.root_cap < tail) cy->status = 1;   // ring overflow: roots were overwritten
    u64 head = head0;
    // smallest decided root >= s, or ~0 when none is decided yet; drops the roots below s (s only grows)
    auto first_root = [&](u64 s) -> u64 {
        u64 lo = head, hi = tail;
        while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if (a.roots[mid % a.root_cap] < s) lo = mid + 1; else hi = mid;
        }
        head = lo;
        return lo < tail ? a.roots[lo % a.root_cap] : ~0ull;
    };
    // Pending peaks (pushed, row not listed yet) are runs (position, count): the duplicate pushes at one start are one run,
    // however long the rootless stretch before them was.  A run is never changed once written.
    u32 len = cy->len;
    u64 run_tail = cy->run_tail;
    u64 s = cy->s;
    bool ring_full = false;
    auto push = [&](u64 p, u64 count) -> bool {
        if (run_tail - cy->run_head >= a.run_cap) { ring_full = true; return false; }
        a.run_pos[run_tail % a.run_cap] = static_cast<u32>(p);
        a.run_cnt[run_tail % a.run_cap] = static_cast<u32>(count);
        ++run_tail;
        len += static_cast<u32>(count);
        return true;
    };
    const u64 row = a.row;
    if (cy->seed_state == 1) {
        const u64 p = cy->seed == kNoSeed ? 0 : first_root(cy->seed);
        if (p != ~0ull && push(p, 1)) {
            s = max(p + D + 1, 2 * row);
            cy->seed_state = 2;
        }
    }
    if (cy->seed_state == 2) {
        while (s < lim) {
            const u64 target = s / row;                      // peaks.len() after the pushes at s
            if (len + 1 < target && !push(s, target - 1 - len)) break;
            const u64 p = first_root(s);
            if (p == ~0ull || !push(p, 1)) break;
            s = max(p + D + 1, row * (s / row + 1));
        }
    }

    // ---- 4. rows to gather: known peak, final envelope (decode.rs:125-127); at the end only k < len - 1, and none
    //         when fewer than 5 peaks were found (decode.rs:112) ----
    u32 ng = 0;
    u64 gathered = cy->gathered, run_head = cy->run_head;
    u32 used = cy->head_used;                                // rows of the head run listed already
    const bool failed = a.finish && len < 5;
    const u64 k_end = a.finish ? (len > 0 ? len - 1 : 0) : len;
    bool list_full = false;
    while (!failed && gathered < k_end && run_head < run_tail) {
        const u64 p = a.run_pos[run_head % a.run_cap];
        if (p + row >= a.work_final) break;
        if (ng == a.gather_cap) { list_full = true; break; }
        a.gpos[ng++] = static_cast<u32>(p);
        ++gathered;
        if (++used == a.run_cnt[run_head % a.run_cap]) { ++run_head; used = 0; }
    }
    // At the end a peak whose row does not fit (p + row >= N_w) never gets one, nor does any later peak: a full ring
    // drops those runs so that the walk can go on (their positions reach the host with this launch's copy).
    bool dropped = false;
    if (a.finish && ring_full && run_head < run_tail && a.run_pos[run_head % a.run_cap] + row >= a.work_final) {
        run_head = run_tail;
        used = 0;
        dropped = true;
    }
    cy->gres.n_rows = ng;
    cy->gres.status = 0;
    cy->first_gather = cy->gathered;
    cy->gathered = gathered;
    cy->run_head = run_head;
    cy->run_tail = run_tail;
    cy->head_used = used;
    cy->len = len;
    cy->s = s;
    cy->decided = decided;
    cy->root_head = head;
    cy->root_tail = tail;
    // another round makes progress only if this one freed ring entries or filled the row list; a full ring whose head
    // row is not final yet waits for a later step instead
    cy->more = list_full || (ring_full && (ng > 0 || dropped)) ? 1u : 0u;
}

}  // namespace aptb200
