"""Plain-numpy restatement of the pass search (DESIGN.md §12): the window quality q in float64 and the pass rule."""
import math

import numpy as np

ENTER, EXIT, MAX_GAP_S, MIN_LENGTH_S = 0.30, 0.15, 30.0, 60.0


def quality(e, row):
    """q[w] for w < W = max(0, floor(len(e) / row) - 1): the Pearson correlation of row w with row w + 1, centred sums in
    float64; 0 where the denominator is 0 or not finite."""
    rows = len(e) // row
    w_count = max(rows - 1, 0)
    if w_count == 0:
        return np.zeros(0, dtype=np.float64)
    m = np.asarray(e[: rows * row], dtype=np.float64).reshape(rows, row)
    c = m - m.mean(axis=1, keepdims=True)
    ss = np.einsum("ij,ij->i", c, c)
    cross = np.einsum("ij,ij->i", c[:-1], c[1:])
    den = np.sqrt(ss[:-1] * ss[1:])
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where((den > 0) & np.isfinite(den), cross / np.where(den > 0, den, 1.0), 0.0)
    return q


def windows_of(seconds):
    return int(math.floor(2.0 * float(np.float32(seconds))))


def find_passes(q, n, rate, enter=ENTER, exit=EXIT, max_gap_s=MAX_GAP_S, min_length_s=MIN_LENGTH_S):
    """The pass rule: list of dicts with the fields of apt_pass (mean and peak as float32, the mean summed in float64 in
    window order)."""
    q = np.asarray(q, dtype=np.float32)
    enter, exit = np.float32(enter), np.float32(exit)
    max_gap, min_length = windows_of(max_gap_s), windows_of(min_length_s)
    groups = []
    for w in np.nonzero(q >= exit)[0].tolist():
        if groups and w - groups[-1][1] - 1 < max_gap:
            groups[-1][1] = w
        else:
            groups.append([w, w])
    out = []
    for a, b in groups:
        seg = q[a:b + 1]
        if not (seg >= enter).any() or b - a + 1 < min_length:
            continue
        total = 0.0
        for v in seg.tolist():
            total += v
        out.append({"start": a * rate // 2, "end": min(n, -((-(b + 2) * rate) // 2)), "first_window": a,
                    "windows": b - a + 1, "mean_quality": float(np.float32(total / (b - a + 1))),
                    "peak_quality": float(seg.max())})
    return out
