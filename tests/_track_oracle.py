"""Tracked sync (DESIGN.md "Tracked sync") restated on the host.

`track_f32` repeats the float32 operations of k_sync_track in its order: the block statistics in double (per-thread
sums over the CTA's columns, the warp xor tree, the cluster's warp entries, then the xor tree again), z, the recurrence
with the candidates in the order 0, -1, +1, -2, +2, ..., the per-block shift and the end argmax.  `track_f64` is the
plain float64 statement of the rule (numpy mean / std, no shift) that the float32 one is checked against.
`rows_from_positions` is step 4: decode.rs:120-132 on the tracked positions, at most floor(N_w / row) rows."""
import numpy as np

THREADS = 256
WARPS = THREADS // 32
CLUSTER = 8      # k_sync_track's cluster size (track_cluster())


def _xor_tree(v):
    """v[..., 32] -> lane 0 after `v += shfl_xor(v, off)` for off = 16 .. 1."""
    v = v.copy()
    idx = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ off]
    return v[..., 0]


def block_stats(c, row, cs=CLUSTER):
    """m_k, s_k (float32) of every block, in k_sync_track's order of double operations."""
    c = np.asarray(c, dtype=np.float32)
    ncorr = c.size
    P = row
    K = -(-ncorr // P)
    W = -(-P // cs)
    Q = -(-20480 // (cs * THREADS))
    cp = np.zeros(K * P, dtype=np.float64)
    cp[:ncorr] = c
    blocks = cp.reshape(K, P)
    s1 = np.zeros((K, cs, THREADS))
    s2 = np.zeros((K, cs, THREADS))
    for q in range(Q):
        # column r*W + t + THREADS*q of each block (0 outside the CTA's slice), added in q order
        x = np.zeros((K, cs, THREADS))
        for r in range(cs):
            j = np.arange(THREADS) + q * THREADS
            col = r * W + j
            ok = (j < W) & (col < P)
            x[:, r, ok] = blocks[:, col[ok]]
        s1 = s1 + x
        s2 = s2 + x * x
    # warp tree -> entries e = r * WARPS + w
    s1 = _xor_tree(s1.reshape(K, cs, WARPS, 32)).reshape(K, cs * WARPS)
    s2 = _xor_tree(s2.reshape(K, cs, WARPS, 32)).reshape(K, cs * WARPS)
    E = cs * WARPS
    a1 = np.zeros((K, 32))
    a2 = np.zeros((K, 32))
    for e0 in range(0, E, 32):
        n = min(32, E - e0)
        a1[:, :n] = a1[:, :n] + s1[:, e0:e0 + n]
        a2[:, :n] = a2[:, :n] + s2[:, e0:e0 + n]
    t1 = _xor_tree(a1)
    t2 = _xor_tree(a2)
    blen = np.minimum(P, ncorr - np.arange(K) * P).astype(np.float64)
    md = t1 / blen
    var = t2 / blen - md * md
    var = np.where(var > 0.0, var, 0.0)
    return md.astype(np.float32), np.sqrt(var).astype(np.float32)


def _z(c, m, s):
    ok = (s != 0) & np.isfinite(s) & np.isfinite(m)
    with np.errstate(all="ignore"):
        z = ((c - m) / s).astype(np.float32)
    return np.where(ok, z, np.float32(0)).astype(np.float32)


def _pen(delta, lam):
    return {d: np.float32(np.float32(lam) * np.float32(d * d)) for d in range(-delta, delta + 1)}


def _order(delta):
    out = [0]
    for u in range(1, delta + 1):
        out += [-u, u]
    return out


def track_f32(c, row, delta=2, lam=0.25, cs=CLUSTER):
    """(positions ascending, back, end) of the tracked path, bit for bit as k_sync_track + k_track_back compute it."""
    c = np.asarray(c, dtype=np.float32)
    ncorr = c.size
    P = row
    K = -(-ncorr // P)
    m, s = block_stats(c, row, cs)
    pen = _pen(delta, lam)
    order = _order(delta)
    S = np.zeros(ncorr, dtype=np.float32)
    back = np.zeros(ncorr, dtype=np.int8)
    for k in range(K):
        lo, hi = k * P, min((k + 1) * P, ncorr)
        if k >= 2:
            M = S[(k - 1) * P:k * P].max()
            S[(k - 2) * P:k * P] = S[(k - 2) * P:k * P] - M
        z = _z(c[lo:hi], m[k], s[k])
        i_all = np.arange(lo, hi)
        # the first delta columns, then the rest (which may read them)
        for part in (slice(0, min(delta, hi - lo)), slice(min(delta, hi - lo), hi - lo)):
            i = i_all[part]
            zz = z[part]
            rec = i >= P + delta
            v = zz.copy()
            if rec.any():
                ii = i[rec]
                best = (S[ii - P] - pen[0]).astype(np.float32)
                bd = np.zeros(ii.size, dtype=np.int8)
                for d in order[1:]:
                    t = (S[ii - P - d] - pen[d]).astype(np.float32)
                    better = t > best
                    best = np.where(better, t, best)
                    bd = np.where(better, np.int8(d), bd)
                v[rec] = (zz[rec] + best).astype(np.float32)
                back[ii] = bd
            S[i] = v
    lo = max(0, ncorr - P)
    end = lo + int(np.argmax(S[lo:]))
    pos = [end]
    i = end
    while i >= P + delta:
        i = i - P - int(back[i])
        pos.append(i)
    return np.array(pos[::-1], dtype=np.int64), back, end


def track_f64(c, row, delta=2, lam=0.25):
    """The rule in float64 with numpy's mean and std and no shift: positions ascending."""
    c = np.asarray(c, dtype=np.float64)
    ncorr = c.size
    P = row
    z = np.zeros(ncorr)
    for k in range(-(-ncorr // P)):
        b = c[k * P:(k + 1) * P]
        sd = b.std()
        if sd > 0 and np.isfinite(sd):
            z[k * P:(k + 1) * P] = (b - b.mean()) / sd
    S = z.copy()
    back = np.zeros(ncorr, dtype=np.int64)
    order = _order(delta)
    pen = {d: lam * d * d for d in order}
    for i0 in range(P + delta, ncorr, P):
        # rows are independent within [i0, i0 + P - delta); the last delta columns read the first ones
        for a, b in ((i0, min(i0 + P - delta, ncorr)), (min(i0 + P - delta, ncorr), min(i0 + P, ncorr))):
            if a >= b:
                continue
            ii = np.arange(a, b)
            best = S[ii - P] - pen[0]
            bd = np.zeros(ii.size, dtype=np.int64)
            for d in order[1:]:
                t = S[ii - P - d] - pen[d]
                better = t > best
                best = np.where(better, t, best)
                bd = np.where(better, d, bd)
            S[ii] = z[ii] + best
            back[ii] = bd
    lo = max(0, ncorr - P)
    i = lo + int(np.argmax(S[lo:]))
    pos = [i]
    while i >= P + delta:
        i = i - P - int(back[i])
        pos.append(i)
    return np.array(pos[::-1], dtype=np.int64)


def rows_from_positions(f, pos, row, dec, nwork):
    """decode.rs:120-132 on the positions, at most floor(N_w / row) rows, then the NoFilter decimation by dec (element 0
    of the output is 0, decode.rs:158-159)."""
    rows = []
    for p in pos[:-1]:
        if p + row < nwork:
            rows.append(np.asarray(f[p:p + row:dec], dtype=np.float32)[: row // dec])
        else:
            break
    rows = rows[: nwork // row]
    out = np.concatenate(rows) if rows else np.zeros(0, dtype=np.float32)
    if out.size:
        out[0] = 0.0   # dsp::filter with NoFilter never reads signal[0] (dsp.rs:399)
    return out


def score(pos, truth, tol=2):
    """Fraction of the true positions with a tracked position within tol samples."""
    pos = np.sort(np.asarray(pos, dtype=np.int64))
    truth = np.asarray(truth, dtype=np.int64)
    if pos.size == 0 or truth.size == 0:
        return 0.0
    j = np.searchsorted(pos, truth)
    a = pos[np.clip(j, 0, pos.size - 1)]
    b = pos[np.clip(j - 1, 0, pos.size - 1)]
    near = np.minimum(np.abs(a - truth), np.abs(b - truth))
    return float(np.mean(near <= tol))
