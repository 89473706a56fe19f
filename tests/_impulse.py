"""Exact inputs for the first stage (front.hpp): impulse trains whose resampled values every correct kernel must return
bit for bit, the restatement of fast_resampling that gives those values, and a per-element bound for the envelope.

An impulse train is zero except for +-2^e samples (e in 0..14; PCM16 trains also use -32768), spaced so that no output
window x*L in [k*M, k*M + off2] holds more than two of them.  Then every product tap * sample is exact, adding zeros is
exact, and two non-zero terms round once whatever their order and whether or not they are fused: any summation order,
slice split, halo dot product or shuffle reduction gives the value exact_resample computes with index arithmetic alone.
A dropped tap, a tap of the neighbouring phase or a wrong window start changes at least one output, however small the
tap is.

No GPU here: the kernel choice is restated from the host-side plan entry points (apt_tile_plan, apt_ut_plan,
apt_ph_plan), in make_front's order (front.cu).
"""
import ctypes as C
import math

import numpy as np

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib
import oracle

CARRIER_HZ = 2400
PH_TILE_PERIODS = 32                                     # kPhTilePeriods (launch.hpp): periods per phase-major tile
ENVELOPE_REL = 2.0 ** -19                                # envelope bound, relative to sqrt(r[k-1]^2 + r[k]^2) / sin(phi)


# One (rate, profile) per input-rate family the first stage treats differently, with make_front's choice for it:
# kind, tiled loop shape (iterations, first iteration of half B, end of half A, halves), groups G and rows per bulk copy.
REPRESENTATIVES = [
    (48000, "standard", "tiled", (7, 1, 6, 2), 13, 2),      # fixed loop shapes (launch.cu)
    (96000, "standard", "tiled", (11, 11, 11, 1), 13, 2),
    (48000, "fast", "tiled", (3, 0, 3, 2), 13, 2),
    (32000, "fast", "tiled", (3, 0, 3, 2), 13, 1),          # fixed shape, one row per copy
    (8000, "slow", "tiled", (3, 0, 3, 2), 13, 1),
    (20800, "standard", "tiled", (3, 0, 3, 2), 3, 1),       # G = 3
    (12000, "standard", "tiled", (2, 0, 2, 2), 13, 2),      # runtime loop, two halves
    (24000, "standard", "tiled", (4, 0, 4, 2), 13, 1),
    (64000, "fast", "tiled", (4, 1, 3, 2), 13, 2),          # runtime: A only, both halves, B only
    (24960, "fast", "tiled", (2, 0, 2, 2), 1, 2),           # G = 1
    (24960, "slow", "tiled", (8, 0, 8, 2), 5, 2),           # G = 5
    (48000, "slow", "tiled", (14, 14, 14, 1), 13, 1),       # runtime loop, one half
    (96000, "slow", "tiled", (28, 28, 28, 1), 13, 2),
    (120000, "standard", "tiled", (14, 14, 14, 1), 13, 2),
    (192000, "standard", "uniform-tap", None, None, None),
    (144000, "standard", "uniform-tap", None, None, None),
    (11025, "standard", "phase-major", None, None, None),
    (37500, "standard", "phase-major", None, None, None),
    (8000, "fast", "phase-major", None, None, None),
    (8000, "standard", "generic", None, None, None),
    (16000, "standard", "generic", None, None, None),
    (32000, "standard", "generic", None, None, None),
    (64000, "standard", "generic", None, None, None),
    (24960, "standard", "decimate", None, None, None),
    (20800, "slow", "decimate", None, None, None),
]


def settings(profile):
    return na.Settings() if profile == "standard" else na.Settings.profile(profile)


def ratio(rate, s):
    g = math.gcd(rate, s.work_rate)
    return s.work_rate // g, rate // g


def front_filter(rate, s):
    """The first stage's filter at the input rate (decode.rs:65-77), as Decoder and resample_with_filter build it."""
    return na.filters.LowpassDcRemoval(na.Freq.hz(s.resample_cutout, rate), s.resample_atten,
                                       na.Freq.hz(s.resample_delta_freq, rate))


def front_taps(rate, s):
    """The taps the first stage runs: designed at the interpolated rate for L > 1 (dsp.rs:93), else at the input rate."""
    l, _ = ratio(rate, s)
    f = front_filter(rate, s)
    if l > 1:
        f.resample(rate, rate * l)
    return f.design()


def front_choice(rate, s):
    """make_front's choice for (rate, settings): tiled, then uniform-tap, then phase-major, then generic; L = 1 decimates.

    Returns a dict: kind, l, m, taps, the plan info of the chosen kind, shape (the tiled loop shape (iterations, first
    iteration of half B, end of half A, halves) launch.cu dispatches on, else None), unit_in / unit_out (input samples
    and outputs of one unit; 0 / 1 where a unit is one output), p_out and R (outputs of one row of a unit and of one
    group of it; one period of L outputs for the uniform-tap and phase-major kernels)."""
    lib = _lib.load()
    l, m = ratio(rate, s)
    h = np.ascontiguousarray(front_taps(rate, s), dtype=np.float32)
    c = dict(rate=rate, l=l, m=m, taps=h, info=None, shape=None, unit_in=0, unit_out=1, p_out=1, R=1)
    if l == 1:
        return dict(c, kind="decimate")
    t = _lib.CTileInfo()
    assert lib.apt_tile_plan(l, m, h.ctypes.data, h.size, C.byref(t), None, 0, None, 0) == 0
    if t.usable:
        bb = t.shift // 16 if t.halves == 2 else t.iters
        return dict(c, kind="tiled", info=t, shape=(t.iters, bb, t.half_taps // 16, t.halves),
                    unit_in=t.rows_per_tile * t.p_in, unit_out=t.rows_per_tile * t.p_out, p_out=t.p_out, R=4 * t.halves)
    u = _lib.CUtInfo()
    assert lib.apt_ut_plan(l, m, h.ctypes.data, h.size, C.byref(u), None, 0) == 0
    if u.usable:
        return dict(c, kind="uniform-tap", info=u, unit_in=u.rows_per_block * m, unit_out=u.rows_per_block * l, p_out=l, R=l)
    p = _lib.CPhInfo()
    assert lib.apt_ph_plan(l, m, h.ctypes.data, h.size, C.byref(p), None, 0, None, 0) == 0
    if p.usable:
        return dict(c, kind="phase-major", info=p, unit_in=PH_TILE_PERIODS * m, unit_out=PH_TILE_PERIODS * l, p_out=l, R=l)
    return dict(c, kind="generic")


def window(l, m, ntaps):
    """Most input samples one output window can hold."""
    if l == 1:
        return ntaps                                     # filter + decimate: x in (k*m - ntaps, k*m]
    return 2 * ((ntaps - 1) // 2) // l + 1               # x*l in [k*m, k*m + off2]


def impulse_train(n, l, m, ntaps, seed, dtype=np.float32, force=()):
    """n samples, zero but for +-2^e impulses (e in 0..14; int16 also -32768) with at most two in any output window.

    Impulses always sit at samples 0 and 1 (both in the first window), at n - 1 and at one of n - 4 .. n - 2 (which one
    depends on the seed: four impulses in the last window would break the two-term rule; a train shorter than two
    windows has only the first two), and at every position in `force`; the rest are random, any three consecutive ones
    spanning at least a window."""
    w = window(l, m, ntaps)
    rng = np.random.default_rng(seed)
    ends = (n - 2 - seed % 3, n - 1) if n - 4 > w else ()        # a train shorter than two windows starts with two
    fixed = sorted({p for p in (0, 1, *ends, *force) if 0 <= p < n})
    for a, b in zip(fixed, fixed[2:]):
        if b - a < w:
            raise ValueError(f"forced impulses {a} .. {b} put three in one window of {w} samples")
    cand = np.cumsum(rng.integers(1, w + 1, n // 2 + 2))
    cand = cand[cand < n]
    # left to right: every fixed impulse, and each random one that keeps any three consecutive impulses -- counting the
    # fixed ones ahead of it -- more than a window apart
    pos, fi = [], 0
    for p in np.union1d(cand, fixed).tolist():
        if fi < len(fixed) and p == fixed[fi]:
            pos.append(p)
            fi += 1
            continue
        ahead = fixed[fi:fi + 2]
        if len(pos) >= 2 and p - pos[-2] < w:
            continue
        if ahead and pos and ahead[0] - pos[-1] < w:
            continue
        if len(ahead) == 2 and ahead[1] - p < w:
            continue
        pos.append(p)
    pos = np.unique(np.asarray(pos, dtype=np.int64))
    mag = 2.0 ** rng.integers(0, 15, pos.size)
    val = np.where(rng.integers(0, 2, pos.size) == 1, mag, -mag)
    if np.dtype(dtype) == np.int16:
        val[rng.integers(0, 8, pos.size) == 0] = -32768.0
    x = np.zeros(n, dtype=dtype)
    x[pos] = val.astype(dtype)
    return x


def contributions(nx, x_pos, l, m, ntaps):
    """(output, tap index, impulse position) of every non-zero term of a train of nx samples with impulses at x_pos."""
    x_pos = np.asarray(x_pos, dtype=np.int64)
    if l == 1:                                           # filtered[i] = sum_{j < ntaps, j < i} x[i-j] c[j]; out[k] = filtered[k*m]
        count = nx // m
        lo = x_pos // m + (x_pos % m != 0)               # k*m >= x
        hi = np.minimum((x_pos + ntaps - 1) // m, count - 1)
        hi = np.where(x_pos > 0, hi, lo - 1)             # x[0] never enters the filter (strict i > j, dsp.rs:399)
    else:
        off, off2 = (ntaps - 1) // 2, 2 * ((ntaps - 1) // 2)
        count = (nx * l - off + m - 1) // m if nx * l > off else 0
        lo = np.maximum(-(-(x_pos * l - off2) // m), 0)
        hi = np.minimum(x_pos * l // m, count - 1)
    cnt = np.maximum(hi - lo + 1, 0)
    xs = np.repeat(x_pos, cnt)
    ks = np.repeat(lo, cnt) + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    taps = ks * m - xs if l == 1 else xs * l - ks * m
    return ks, taps, xs, count


def exact_resample(x, l, m, h):
    """fast_resampling (dsp.rs:186-289; L = 1: filter + decimate, dsp.rs:105-123) of an impulse train, in float32, by
    index arithmetic: out[k] = sum of h[x*L - k*M] * x[x] over the (at most two) impulses of output k's window."""
    x = np.asarray(x)
    xf = x.astype(np.float32)                            # PCM16: the `as f32` cast of wav.rs:37
    h = np.asarray(h, dtype=np.float32)
    ks, taps, xs, count = contributions(x.size, np.flatnonzero(xf), l, m, h.size)
    out = np.zeros(count, dtype=np.float32)
    assert np.bincount(ks, minlength=count).max(initial=0) <= 2, "more than two impulses in one output window"
    np.add.at(out, ks, h[taps] * xf[xs])                 # float32: 0 + a, then a + b rounded once
    return out


def used_taps(x, l, m, ntaps):
    """Tap indices some output of the train multiplies by a non-zero sample."""
    ks, taps, _, _ = contributions(x.size, np.flatnonzero(x), l, m, ntaps)
    return np.unique(taps)


def sin_phi(work_rate):
    phi = np.float32(2.0) * np.float32(oracle.freq_get_rad(oracle.freq_hz(CARRIER_HZ, work_rate)))
    return float(np.sin(np.float64(phi)))


def envelope_misses(e, r, work_rate):
    """Indices where the envelope e of the exact resampled signal r leaves its bound: e[0] must be 0 and, for k >= 1,
    |e[k] - demodulate(r)[k]| <= 2^-19 * sqrt(r[k-1]^2 + r[k]^2) / sin(phi).  The argument of the square root cannot
    cancel (|2 cos(phi)| < 2 at every work rate), so a few ulp of that scale cover the device's sqrt.approx and its multiply
    by 1/sin(phi); a wrong previous sample moves e[k] by about the scale itself."""
    e = np.asarray(e, dtype=np.float32)
    r = np.asarray(r, dtype=np.float32)
    assert e.shape == r.shape, (e.shape, r.shape)
    ref = oracle.demodulate(r, oracle.freq_hz(CARRIER_HZ, work_rate)).astype(np.float64)
    r64 = r.astype(np.float64)
    scale = np.zeros_like(r64)
    scale[1:] = np.sqrt(r64[:-1] ** 2 + r64[1:] ** 2) / sin_phi(work_rate)
    bad = ~(np.abs(e.astype(np.float64) - ref) <= ENVELOPE_REL * scale)    # NaN fails
    bad[0] = not (e[0] == 0)
    return np.flatnonzero(bad)


def describe(idx, unit_out, what="outputs"):
    """First few failing indices with the unit each falls in."""
    idx = np.asarray(idx)
    head = ", ".join(f"{int(k)} (unit {int(k) // unit_out}, +{int(k) % unit_out})" for k in idx[:8])
    return f"{idx.size} {what} differ: {head}"


def train_len(c):
    """Length of a representative's impulse train: three and a half units, and enough impulses that every residue of
    x mod M, hence every tap, meets one (checked by the CPU suite)."""
    return max(3 * c["unit_in"] + c["unit_in"] // 2 + 37, 8 * c["m"] * window(c["l"], c["m"], c["taps"].size), 4000)


def unit_force(n, unit_in, w, extra=()):
    """Impulses on both sides of every unit boundary (and of the boundaries in `extra`) of an n-sample train whose output
    windows hold w samples, leaving out boundaries within a window of the impulses every train starts and ends with."""
    b = {*range(unit_in, n, unit_in), *extra} if unit_in else set(extra)
    return [p for q in sorted(b) if w + 1 <= q <= n - w - 4 for p in (q - 1, q)]


def representative_train(c, dtype=np.float32, seed=0):
    n = train_len(c)
    return impulse_train(n, c["l"], c["m"], c["taps"].size, seed=c["rate"] % 97 + seed, dtype=dtype,
                         force=unit_force(n, c["unit_in"], window(c["l"], c["m"], c["taps"].size)))


CHUNK_FLOOR = 1 << 16                                    # the decoder raises APTB200_CHUNK_SAMPLES to at least this


def front_span(c):
    """(before, after): input samples in front of a run's first unit and beyond the start of its last one (front.cu)."""
    t = c["info"]
    if c["kind"] == "tiled":
        h = c["taps"]
        tt = np.zeros(t.groups * t.group_stride, np.float32)
        xs = np.zeros(t.groups, np.uint32)
        assert _lib.load().apt_tile_plan(c["l"], c["m"], h.ctypes.data, h.size, C.byref(_lib.CTileInfo()), tt.ctypes.data,
                                         tt.size, xs.ctypes.data, xs.size) == 0
        return t.p_in - int(xs[-1]), (t.rows_per_tile - 1) * t.p_in + t.row_len
    if c["kind"] == "uniform-tap":
        return t.back, t.slot_floats - t.back
    if c["kind"] == "phase-major":
        return c["m"] + 4, (PH_TILE_PERIODS - 1) * c["m"] + t.row_len
    return None


def chunk_units(c, cap):
    """Units one chunk of `cap` staged samples serves in the chunked upload (FrontPlan::chunk_units)."""
    cap &= ~7
    span = front_span(c)
    if span:
        return (cap - span[0] - span[1] - 64) // c["unit_in"] + 1
    halo = 2 * ((c["taps"].size - 1) // 2) // c["l"] + 4
    return (cap - 2 * halo) * c["l"] // c["m"]


def seam_caps(c):
    """APTB200_CHUNK_SAMPLES values for the chunked upload: the smallest the decoder takes, the smallest above it whose
    chunk holds its units with fewer than 8 samples to spare, and 8 samples less (one unit fewer per chunk)."""
    cap = CHUNK_FLOOR + 8
    while chunk_units(c, cap) == chunk_units(c, cap - 8):
        cap += 8
    assert chunk_units(c, cap - 8) < chunk_units(c, cap)
    return sorted({CHUNK_FLOOR, cap, cap - 8})


def seam_inputs(c, n, cap):
    """Input positions of the first output of every chunk after the first one (chunk seams of an n-sample decode)."""
    per = chunk_units(c, cap)
    nwork = exact_len(n, c["l"], c["m"], c["taps"].size)
    units = -(-nwork // c["unit_out"])
    first = [u * c["unit_out"] for u in range(per, units, per)]
    return [-(-k * c["m"] // c["l"]) for k in first]


def exact_len(n, l, m, ntaps):
    """Outputs of n samples: fast_resampling's count, or n // m for filter + decimate."""
    if l == 1:
        return n // m
    off = (ntaps - 1) // 2
    return (n * l - off + m - 1) // m if n * l > off else 0
