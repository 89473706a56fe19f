// Tracked sync (DESIGN.md "Tracked sync"): the row period followed through the whole pass by dynamic programming over the
// sync correlation c[0 .. ncorr).  P = row, block k = [kP, min((k+1)P, ncorr)).
//
//   z[i] = (c[i] - m_k) / s_k                        m_k, s_k: mean and population deviation of block k (double, rounded once)
//   S[i] = z[i]                                      i < P + delta
//   S[i] = z[i] + max_{d = -delta..delta} (S[i-P-d] - pen[d])   otherwise, candidates in the order 0, -1, +1, -2, +2, ...,
//                                                    the first strictly larger one wins; back[i] = the winning d
//   before block k >= 2 is evaluated, the maximum S of block k-1 is subtracted from every S of blocks k-1 and k-2
//
// Every float operation is a single IEEE operation (__fsub_rn etc.: nothing contracts), in the order tests/_track_oracle.py
// restates.  k_sync_track: one cluster of CS CTAs walks the blocks in order, CTA r owns the columns [rW, min((r+1)W, P))
// of every block (W = ceil(P / CS)); S of blocks k-2, k-1, k stays in shared memory, only back reaches HBM.
// k_track_back: the end (argmax of S over the last P indices, written by k_sync_track) walked back to the positions.
#pragma once

#include <cooperative_groups.h>

#include "launch.hpp"

namespace aptb200 {

constexpr u32 kTrackThreads = 256;
constexpr u32 kTrackWarps = kTrackThreads / 32;
constexpr u32 kTrackMaxRow = 20480;    // can_sync: min_distance = 0.8 row <= 16384
constexpr u32 kTrackWalkSteps = 32;    // k_track_back: steps resolved per staged window

struct TrackArgs {
    const float *corr;
    u64 ncorr;
    u32 row, delta;
    float pen[2 * kTrackMaxDelta + 1];   // pen[delta + d] = float(lambda * d^2)
    int8_t *back;                        // [ncorr]
    u32 *end;                            // argmax of S over [max(0, ncorr - P), ncorr), first index on ties
};

// Shared partial sums of one block: per warp (entry r * kTrackWarps + w of the cluster), double-buffered by block parity.
struct TrackPartials {
    double s1[2][kTrackWarps], s2[2][kTrackWarps];
    float mx[2][kTrackWarps];            // maximum S of the previous block over the warp's columns
    float ev[kTrackWarps];               // end argmax: value and index per warp
    u32 ei[kTrackWarps];
};

__device__ __forceinline__ float track_z(float c, float m, float s, bool ok) {
    return ok ? __fdiv_rn(__fsub_rn(c, m), s) : 0.f;
}

template <u32 CS>
__global__ void __launch_bounds__(kTrackThreads, 1) k_sync_track(const TrackArgs a) {
    namespace cg = cooperative_groups;
    constexpr u32 Q = (kTrackMaxRow + CS * kTrackThreads - 1) / (CS * kTrackThreads);   // columns per thread
    cg::cluster_group cluster = cg::this_cluster();
    const u32 r = cluster.block_rank();
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 P = a.row, D = a.delta;
    const u32 W = (P + CS - 1) / CS;
    const u32 c0 = r * W;
    const u32 wr = c0 < P ? min(W, P - c0) : 0u;           // columns of this CTA
    const u64 ncorr = a.ncorr;
    const u64 K = (ncorr + P - 1) / P;

    extern __shared__ float smem[];
    auto slot = [&](u64 k) { return smem + (k % 3) * W; };   // raw S of block k
    float *ext = smem + 3 * W;                             // [wr + 2D]: candidates of columns c0 - D .. c0 + wr + D
    __shared__ TrackPartials part;
    __shared__ float head[kTrackMaxDelta];
    __shared__ float pen[2 * kTrackMaxDelta + 1];
    if (tid < 2 * D + 1) pen[tid] = a.pen[tid];   // published by the first cluster barrier

    float cur[Q], nxt[Q];
    auto load = [&](u64 k, float *v) {
#pragma unroll
        for (u32 q = 0; q < Q; ++q) {
            const u32 j = tid + q * kTrackThreads;
            const u64 i = k * P + c0 + j;
            v[q] = (k < K && j < wr && i < ncorr) ? __ldg(a.corr + i) : 0.f;
        }
    };
    // partial sums of block k over this thread's columns (ascending), warp tree, one entry per warp
    auto stats = [&](const float *v, u32 par, float smax) {
        double s1 = 0.0, s2 = 0.0;
#pragma unroll
        for (u32 q = 0; q < Q; ++q) {
            const double x = static_cast<double>(v[q]);
            s1 = __dadd_rn(s1, x);
            s2 = __dadd_rn(s2, __dmul_rn(x, x));
        }
#pragma unroll
        for (u32 off = 16; off; off >>= 1) {
            s1 = __dadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, off));
            s2 = __dadd_rn(s2, __shfl_xor_sync(0xffffffffu, s2, off));
            smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, off));
        }
        if (lane == 0) {
            part.s1[par][warp] = s1;
            part.s2[par][warp] = s2;
            part.mx[par][warp] = smax;
        }
    };

    load(0, cur);
    load(1, nxt);
    stats(cur, 0, -INFINITY);
    cluster.sync();

    float sh = 0.f, sh_prev = 0.f;      // shifts applied before blocks k and k-1 (valid for k >= 2, k-1 >= 2)
    for (u64 k = 0; k < K; ++k) {
        const u32 par = static_cast<u32>(k & 1);
        const u64 base = k * P;
        const u32 blen = static_cast<u32>(min(static_cast<u64>(P), ncorr - base));
        // m_k, s_k and the maximum of block k-1: entries e = lane, lane + 32, ... of the cluster, then the xor tree
        double s1 = 0.0, s2 = 0.0;
        float mx = -INFINITY;
        for (u32 e = lane; e < CS * kTrackWarps; e += 32) {
            const TrackPartials *rp = cluster.map_shared_rank(&part, e / kTrackWarps);
            s1 = __dadd_rn(s1, rp->s1[par][e % kTrackWarps]);
            s2 = __dadd_rn(s2, rp->s2[par][e % kTrackWarps]);
            mx = fmaxf(mx, rp->mx[par][e % kTrackWarps]);
        }
#pragma unroll
        for (u32 off = 16; off; off >>= 1) {
            s1 = __dadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, off));
            s2 = __dadd_rn(s2, __shfl_xor_sync(0xffffffffu, s2, off));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        }
        const double n = static_cast<double>(blen);
        const double md = __ddiv_rn(s1, n);
        double var = __dsub_rn(__ddiv_rn(s2, n), __dmul_rn(md, md));
        if (!(var > 0.0)) var = 0.0;
        const float m = __double2float_rn(md);
        const float s = __double2float_rn(__dsqrt_rn(var));
        const bool ok = s != 0.f && isfinite(s) && isfinite(m);
        sh_prev = sh;
        sh = mx;
        const bool shift1 = k >= 2, shift2 = k >= 3;
        // a candidate of block k-1 (rel 1) or k-2 (rel 2) in the frame of block k
        auto cand = [&](u32 rel, u32 col) {
            const u32 owner = col / W;
            const float *src = cluster.map_shared_rank(slot(k + 3 - rel), owner);
            float v = src[col - owner * W];
            if (rel == 2 && shift2) v = __fsub_rn(v, sh_prev);
            if (shift1) v = __fsub_rn(v, sh);
            return v;
        };
        // one step of the recurrence at column j; cv(x) is the candidate at column j + x of block k-1 (d = -x)
        auto step = [&](float z, auto cv, int8_t &bd) {
            float best = __fsub_rn(cv(0), pen[D]);
            int b = 0;
            for (u32 u = 1; u <= D; ++u) {
                const float tn = __fsub_rn(cv(static_cast<int>(u)), pen[D - u]);    // d = -u: column j + u
                if (tn > best) best = tn, b = -static_cast<int>(u);
                const float tp = __fsub_rn(cv(-static_cast<int>(u)), pen[D + u]);   // d = +u: column j - u
                if (tp > best) best = tp, b = static_cast<int>(u);
            }
            bd = static_cast<int8_t>(b);
            return __fadd_rn(z, best);
        };
        if (k >= 1 && wr) {
            // the first D columns of block k, which the last CTA's columns P - D .. P - 1 read: computed there again, in
            // the same operations as CTA 0 computes them
            if (r == CS - 1 && tid < D && tid >= blen) {
                head[tid] = 0.f;   // a last block of fewer than D columns: no column here, and none reads it
            } else if (r == CS - 1 && tid < D) {
                const float z = track_z(__ldg(a.corr + base + tid), m, s, ok);
                if (k == 1) {
                    head[tid] = z;
                } else {
                    int8_t bd;
                    head[tid] = step(z, [&](int x) {
                        const int col = static_cast<int>(tid) + x;
                        return col < 0 ? cand(2, static_cast<u32>(col + static_cast<int>(P))) : cand(1, static_cast<u32>(col));
                    }, bd);
                }
            }
            for (u32 x = tid; x < wr + 2 * D; x += kTrackThreads) {
                const int col = static_cast<int>(c0 + x) - static_cast<int>(D);
                float v = 0.f;
                if (col < 0) {
                    if (k >= 2) v = cand(2, static_cast<u32>(col + static_cast<int>(P)));
                } else if (col < static_cast<int>(P)) {
                    v = cand(1, static_cast<u32>(col));
                }
                ext[x] = v;
            }
            __syncthreads();
            if (r == CS - 1 && tid < D) ext[wr + D + tid] = head[tid];
            __syncthreads();
        }
        float *out = slot(k);
        float tmax = -INFINITY;
#pragma unroll
        for (u32 q = 0; q < Q; ++q) {
            const u32 j = tid + q * kTrackThreads;
            const u64 i = base + c0 + j;
            if (j < wr && i < ncorr) {
                const float z = track_z(cur[q], m, s, ok);
                float v;
                int8_t bd = 0;
                if (i < static_cast<u64>(P) + D) v = z;
                else v = step(z, [&](int x) { return ext[static_cast<int>(j + D) + x]; }, bd);
                out[j] = v;
                a.back[i] = bd;
                tmax = fmaxf(tmax, v);
            }
        }
#pragma unroll
        for (u32 q = 0; q < Q; ++q) cur[q] = nxt[q];
        if (k + 1 < K) stats(cur, par ^ 1u, tmax);
        load(k + 2, nxt);
        cluster.sync();
    }

    // the end: argmax of S over [max(0, ncorr - P), ncorr) in the frame of the last block, first index on ties
    const u64 lo = ncorr > P ? ncorr - P : 0;
    float bv = -INFINITY;
    u32 bi = 0xFFFFFFFFu;
    for (u32 rel = (K >= 2 ? 1u : 0u) + 1; rel-- > 0;) {
        const u64 k = K - 1 - rel;
        const float *src = slot(k);
        for (u32 j = tid; j < wr; j += kTrackThreads) {
            const u64 i = k * P + c0 + j;
            if (i < lo || i >= ncorr) continue;
            float v = src[j];
            if (rel == 1 && K - 1 >= 2) v = __fsub_rn(v, sh);
            if (v > bv || bi == 0xFFFFFFFFu) bv = v, bi = static_cast<u32>(i);
        }
    }
#pragma unroll
    for (u32 off = 16; off; off >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const u32 oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (oi != 0xFFFFFFFFu && (bi == 0xFFFFFFFFu || ov > bv || (ov == bv && oi < bi))) bv = ov, bi = oi;
    }
    if (lane == 0) part.ev[warp] = bv, part.ei[warp] = bi;
    cluster.sync();
    if (r == 0 && tid == 0) {
        float v = -INFINITY;
        u32 idx = 0xFFFFFFFFu;
        for (u32 e = 0; e < CS * kTrackWarps; ++e) {
            const TrackPartials *rp = cluster.map_shared_rank(&part, e / kTrackWarps);
            const float ov = rp->ev[e % kTrackWarps];
            const u32 oi = rp->ei[e % kTrackWarps];
            if (oi != 0xFFFFFFFFu && (idx == 0xFFFFFFFFu || ov > v || (ov == v && oi < idx))) v = ov, idx = oi;
        }
        *a.end = idx;
    }
    cluster.sync();   // no CTA leaves while CTA 0 reads its shared memory
}

// Backtrack: i <- i - P - back[i] from the end while i >= P + delta; the positions ascending, then the rows of decode.rs:
// 120-132 (every position but the last with p + row < N_w), at most floor(N_w / row) of them (the decoder's output bound).
// One CTA: the windows the next kTrackWalkSteps steps can reach are staged in shared memory, thread 0 walks them.
__global__ void __launch_bounds__(kTrackThreads) k_track_back(const int8_t *__restrict__ back, const u32 *__restrict__ end,
                                                             u64 ncorr, u64 nwork, u32 row, u32 delta,
                                                             u32 *__restrict__ positions, u32 cap,
                                                             SyncResult *__restrict__ result) {
    constexpr u32 kWin = kTrackWalkSteps + kTrackWalkSteps * (kTrackWalkSteps - 1) * kTrackMaxDelta;
    __shared__ int8_t win[kWin];
    __shared__ u32 s_cur, s_n, s_done, s_rows;
    const u32 tid = threadIdx.x;
    const u64 stop = static_cast<u64>(row) + delta;
    if (tid == 0) {
        const u32 e = *end;
        s_cur = e;
        positions[0] = e;
        s_n = 1;
        s_done = e < stop;
        s_rows = 0;
    }
    __syncthreads();
    while (!s_done) {
        const u64 cur = s_cur;
        // window s: the indices s steps back can reach, [cur - s(P + delta), cur - s(P - delta)]
        u32 off = 0;
        for (u32 st = 0; st < kTrackWalkSteps; ++st) {
            const u32 width = 2 * st * delta + 1;
            const long long lo = static_cast<long long>(cur) - static_cast<long long>(st) * (row + delta);
            for (u32 u = tid; u < width; u += blockDim.x) {
                const long long x = lo + u;
                win[off + u] = (x >= 0 && static_cast<u64>(x) < ncorr) ? back[x] : 0;
            }
            off += width;
        }
        __syncthreads();
        if (tid == 0) {
            u64 i = cur;
            u32 n = s_n, o = 0;
            bool done = false;
            for (u32 st = 0; st < kTrackWalkSteps; ++st) {
                if (i < stop) { done = true; break; }
                const long long lo = static_cast<long long>(cur) - static_cast<long long>(st) * (row + delta);
                i = i - row - static_cast<long long>(win[o + (static_cast<long long>(i) - lo)]);
                if (n < cap) positions[n] = static_cast<u32>(i);
                ++n;
                o += 2 * st * delta + 1;
            }
            s_cur = static_cast<u32>(i);
            s_n = n;
            s_done = done || i < stop;
        }
        __syncthreads();
    }
    const u32 n = min(s_n, cap);
    for (u32 x = tid; x < n / 2; x += blockDim.x) {
        const u32 t = positions[x];
        positions[x] = positions[n - 1 - x];
        positions[n - 1 - x] = t;
    }
    __syncthreads();
    u32 cnt = 0;
    for (u32 x = tid; x + 1 < n; x += blockDim.x) cnt += static_cast<u64>(positions[x]) + row < nwork ? 1u : 0u;
    atomicAdd(&s_rows, cnt);
    __syncthreads();
    if (tid == 0) {
        result->n_peaks = n;
        result->n_rows = static_cast<u32>(min(static_cast<u64>(s_rows), nwork / row));
        result->status = n < 5 ? 3u /* APT_ERR_FEW_SYNC_FRAMES */ : 0u;
        result->seed_index = 0;
        result->n_roots = 0;
    }
}

}  // namespace aptb200
