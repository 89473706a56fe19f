"""The fused back half of decode() restated in float32, operation by operation in the kernels' order, so that the device's
low-passed signal, correlation, per-tile records, roots, positions and rows can be compared bit for bit.

The restatement starts from the device's own envelope (Decoder.read_stage("demodulated")), so it does not depend on the
first stage's rounding.  Every step is the one the kernels of kernels_sync2.cuh and kernels_lpsync.cuh take:

- low-pass (dsp.rs:386-410): f[o] = fma(c[NT-1], e[o-NT+1], ... fma(c[1], e[o-1], fma(c[0], e[o], 0))), one chain per
  output, tap 0 first, e[k] = 0 for k < 1 (dsp.rs:399: signal[0] is never read);
- box sums through pair sums P[k] = f[2k] + f[2k+1]: B[2u] = P[u] + S_u, B[2u+1] = (f[2u+1] + S_u) + f[2u+BOX] with
  S_u = P[u+1] + ... + P[u+PW-1] left to right (BOX = 2*PW; pairs start at even indices of the whole signal);
- correlation: 0, then +-B[i + BOX*b] for b = 0..18 in order, signs '-', (-,+) x 7, '-' x 4 (decode.rs:188-198);
- records: per tile of W positions the maximum, the weak suffix records (>= everything later in the tile) and the strict
  prefix records (> everything earlier in the tile);
- roots by their definition, positions by the picker's walk (carried_walk), rows f[pos_j + PW*c] with pixel 0 of row 0
  set to zero (decode.rs:158-159).

numpy has no fused multiply-add: fma32 forms the exact product in float64, adds the addend by TwoSum and rounds the sum
to odd before the final rounding to float32, which gives the correctly rounded float32 FMA.  No other step leaves
float32.
"""
import ctypes as C

import numpy as np

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib
from noaa_apt_b200.decode import RECORD, TILE_RECORDS

FINAL_RATE = 4160
PX = 2080
REC_TB = 64                      # kRecTB (kernels_sync2.cuh): rows of 32 low-passed samples staged per tile


def fma32(a, b, c):
    """Correctly rounded float32 a*b + c, elementwise (numpy broadcasting)."""
    a = np.asarray(a, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    p = a * b                                        # exact: 24 + 24 significant bits
    s = p + c
    bp = s - p                                       # TwoSum: s + err == p + c exactly
    err = (p - (s - bp)) + (c - bp)
    even = (s.view(np.int64) & 1) == 0
    toward = np.where(err > 0, np.inf, -np.inf)
    s = np.where((err != 0) & even, np.nextafter(s, toward), s)   # round to odd: the float32 rounding sees the sticky bit
    return s.astype(np.float32)


def pixel_width(work_rate):
    return work_rate // FINAL_RATE


def tile_width(pw):
    """rec_tile_outputs: correlation positions per tile, the largest multiple of 32 whose f values (plus the 18 runs of
    the template ahead and the box sum's own width) fit the 32 x kRecTB samples a tile stages."""
    return (32 * REC_TB - 18 * 2 * pw - (2 * pw - 1)) // 32 * 32


def lowpass_taps(work_rate, atten=25.0):
    """The demodulation low-pass of decode.rs:95-102 as the library designs it."""
    c = np.float32(FINAL_RATE) / np.float32(work_rate)
    return na.filters.Lowpass(na.Freq(float(c)), atten, na.Freq(float(np.float32(c) / np.float32(5.0)))).design()


def lowpass(e, taps):
    """f[o] for o < e.size: one FMA chain per output, tap 0 first."""
    e = np.asarray(e, np.float32)
    n = e.size
    f = np.zeros(n, np.float32)
    for t, c in enumerate(np.asarray(taps, np.float32)):
        x = np.zeros(n, np.float32)
        if n > t + 1:
            x[t + 1:] = e[1:n - t]                   # x[o] = e[o - t] for o - t >= 1, else 0
        f = fma32(c, x, f)
    return f


def box_sums(f, pw, count):
    """B[0 .. count) of f, in the kernels' order (f is read as zero beyond its end)."""
    box = 2 * pw
    half = (count + 1) // 2
    fp = np.zeros(2 * (half + pw) + 2, np.float32)
    k = min(f.size, fp.size)
    fp[:k] = f[:k]
    P = fp[0::2] + fp[1::2]
    u = np.arange(half)
    s = P[u + 1].copy()
    for k in range(2, pw):
        s = s + P[u + k]
    b = np.empty(2 * half, np.float32)
    b[0::2] = P[u] + s
    b[1::2] = (fp[2 * u + 1] + s) + fp[2 * u + box]
    return b[:count]


def correlation_signs():
    """Sign of run b = 0..18 of the sync template."""
    return [-1] + [(-1 if b % 2 else 1) for b in range(1, 15)] + [-1] * 4


def correlation(f, pw):
    """corr[i] for i < f.size - 38*PW (decode.rs:225)."""
    box = 2 * pw
    ncorr = max(f.size - 38 * pw, 0)
    b = box_sums(f, pw, ncorr + 18 * box)
    corr = np.zeros(ncorr, np.float32)
    for k, sign in enumerate(correlation_signs()):
        seg = b[k * box: k * box + ncorr]
        corr = corr + seg if sign > 0 else corr - seg
    return corr


def tile_records(corr, w):
    """Per tile of w positions: (n_suffix, n_prefix, max) and the records (pos, val), suffix list then prefix list, in tile
    order -- the layout of Decoder.last_records()."""
    n = corr.size
    nt = (n + w - 1) // w
    tiles = np.zeros(nt, dtype=TILE_RECORDS)
    pos, val = [], []
    for t in range(nt):
        c = corr[t * w: min((t + 1) * w, n)]
        later = np.concatenate([np.maximum.accumulate(c[::-1])[::-1][1:], [-np.inf]]).astype(np.float32)
        earlier = np.concatenate([[-np.inf], np.maximum.accumulate(c)[:-1]]).astype(np.float32)
        suf = np.nonzero(~(later > c))[0]
        pre = np.nonzero(c > earlier)[0]
        tiles[t] = (suf.size, pre.size, c.max())
        for idx in (suf, pre):
            pos.append(t * w + idx)
            val.append(c[idx])
    recs = np.zeros(sum(p.size for p in pos), dtype=RECORD)
    if recs.size:
        recs["pos"] = np.concatenate(pos)
        recs["val"] = np.concatenate(val)
    return tiles, recs


def roots_direct(corr, dist):
    """Definition of a root: no corr[j] > corr[p] for j in (p, p + dist]."""
    n = corr.size
    pad = np.concatenate([corr, np.full(dist, -np.inf, np.float32)])
    w = np.lib.stride_tricks.sliding_window_view(pad[1:], dist).max(axis=1)[:n]
    return np.nonzero(~(w > corr))[0].astype(np.uint64)


def min_distance(work_rate):
    return (PX * work_rate // FINAL_RATE) * 8 // 10


def rows(f, positions, pw):
    """decode.rs:122-134,158-159: rows f[pos_j + PW*c] of every position but the last whose row ends inside f; positions
    None: the rows j*row without sync (decode.rs:141-147)."""
    row = PX * pw
    if positions is None:
        starts = np.arange(f.size // row, dtype=np.int64) * row
    else:
        p = np.asarray(positions, np.int64)[:-1]
        starts = p[p + row < f.size]
    out = f[starts[:, None] + pw * np.arange(PX)[None, :]].astype(np.float32) if starts.size else np.zeros((0, PX), np.float32)
    if out.size:
        out[0, 0] = 0.0
    return out.ravel()


def window_max(c, d):
    """w[p] = max(c[p+1 .. p+d]) over the given values (-inf beyond), by the van Herk / Gil-Werman block split."""
    n = c.size
    x = np.full(((n + 2 * d) // d + 1) * d, -np.inf, dtype=np.float32)
    x[: n - 1] = c[1:]
    blocks = x.reshape(-1, d)
    g = np.maximum.accumulate(blocks, axis=1).ravel()
    h = np.maximum.accumulate(blocks[:, ::-1], axis=1)[:, ::-1].ravel()
    p = np.arange(n)
    return np.maximum(h[p], g[p + d - 1])


def carried_walk(corr, work_rate, splits, on_step=None, run_cap=256, gather_cap=8):
    """Positions the stream decides when corr becomes final on [0, c) for c in splits, then at the end.

    Pending peaks are (position, count) runs in a ring of run_cap entries; each round walks as far as it can, lists at
    most gather_cap rows whose envelope is final, and another round follows only if it can make progress (as in
    k_stream_sync).  on_step(c_end, peaks, state) sees the state after each step."""
    pw = work_rate // FINAL_RATE
    row = PX * pw
    D = row * 8 // 10
    G = 38 * pw
    ncorr = corr.size
    st = dict(decided=0, seed_state=0, seed=None, s=0, length=0, gathered=0, used=0, rounds=0)
    roots = []
    runs = []            # pending runs [position, count], oldest first
    peaks = []           # every peak pushed, expanded

    def first_root(x):
        i = int(np.searchsorted(roots, x, side="left"))
        return roots[i] if i < len(roots) else None

    for c_end in list(splits) + [None]:
        finish = c_end is None
        lim = ncorr if finish else c_end
        dec_hi = ncorr if finish else max(c_end - D, 0)
        wf = ncorr + G if finish else c_end + G
        if dec_hi > st["decided"]:
            d0 = st["decided"]
            vis = corr[d0:lim]                                 # the windows of [d0, dec_hi), clipped at lim
            w = window_max(vis, D)
            p = np.arange(dec_hi - d0)
            roots.extend((d0 + p[~(w[p] > vis[p])]).tolist())
            st["decided"] = dec_hi
        if st["seed_state"] == 0 and (finish or c_end > D):
            hit = np.nonzero(corr[: min(D + 1, lim)] > 0)[0]
            st["seed"] = int(hit[0]) if hit.size else None
            st["seed_state"] = 1
        while True:
            st["rounds"] += 1
            ring_full = False

            def push(pos, count):
                nonlocal ring_full
                if len(runs) >= run_cap:
                    ring_full = True
                    return False
                runs.append([pos, count])
                peaks.extend([pos] * count)
                st["length"] += count
                return True

            if st["seed_state"] == 1:
                p0 = 0 if st["seed"] is None else first_root(st["seed"])
                if p0 is not None and push(p0, 1):
                    st["s"] = max(p0 + D + 1, 2 * row)
                    st["seed_state"] = 2
            if st["seed_state"] == 2:
                s = st["s"]
                while s < lim:
                    target = s // row
                    if st["length"] + 1 < target and not push(s, target - 1 - st["length"]):
                        break
                    r = first_root(s)
                    if r is None or not push(r, 1):
                        break
                    s = max(r + D + 1, row * (s // row + 1))
                st["s"] = s
            n = st["length"]
            k_end = (n - 1 if n else 0) if finish else n
            failed = finish and n < 5
            ng, list_full = 0, False
            while not failed and st["gathered"] < k_end and runs:
                if runs[0][0] + row >= wf:
                    break
                if ng == gather_cap:
                    list_full = True
                    break
                ng += 1
                st["gathered"] += 1
                st["used"] += 1
                if st["used"] == runs[0][1]:
                    runs.pop(0)
                    st["used"] = 0
            dropped = False
            if finish and ring_full and runs and runs[0][0] + row >= wf:
                runs.clear()
                st["used"] = 0
                dropped = True
            if not (list_full or (ring_full and (ng > 0 or dropped))):
                break
        st["pending_runs"] = len(runs)
        st["first_pending"] = runs[0][0] if runs else None
        if on_step is not None and not finish:
            on_step(c_end, list(peaks), dict(st))
    return np.array(peaks, dtype=np.uint64)


def positions(corr, work_rate):
    """find_sync's positions on a given correlation (decode.rs:204-263)."""
    return carried_walk(corr, work_rate, [])


def back_half(e, work_rate, atten=25.0, sync=True):
    """Everything the fused back half computes from the envelope e: f, corr, tiles/records, roots, positions, rows."""
    pw = pixel_width(work_rate)
    f = lowpass(e, lowpass_taps(work_rate, atten))
    out = {"f": f}
    if not sync:
        out["rows"] = rows(f, None, pw)
        return out
    corr = correlation(f, pw)
    out["corr"] = corr
    out["tiles"], out["records"] = tile_records(corr, tile_width(pw))
    out["roots"] = roots_direct(corr, min_distance(work_rate))
    out["positions"] = positions(corr, work_rate)
    out["rows"] = rows(f, out["positions"], pw)
    return out


def work_len(n, rate, settings):
    """N_w: envelope samples of a decode of n input samples (the first stage's output length, apt_resample_len)."""
    filt = na.filters.LowpassDcRemoval(na.Freq.hz(settings.resample_cutout, rate), settings.resample_atten,
                                       na.Freq.hz(settings.resample_delta_freq, rate))
    cf = filt.to_c()
    got = C.c_uint64(0)
    na.err.raise_for(_lib.load().apt_resample_len(int(n), int(rate), int(settings.work_rate), C.byref(cf), C.byref(got)))
    return got.value


def input_len_for(nwork, rate, settings):
    """The smallest input length whose envelope has nwork samples, or None when no length gives exactly nwork."""
    lo, hi = 1, int(nwork * rate / settings.work_rate) + 64
    while work_len(hi, rate, settings) < nwork:
        hi *= 2
    while lo < hi:                                   # first n with work_len(n) >= nwork
        mid = (lo + hi) // 2
        if work_len(mid, rate, settings) >= nwork:
            hi = mid
        else:
            lo = mid + 1
    return lo if work_len(lo, rate, settings) == nwork else None
