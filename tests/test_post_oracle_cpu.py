"""Checks the C oracle's image-stage functions (oracle/apt_oracle.c) and tests/_process_oracle.py on non-finite and tie
inputs before the device tests rely on them.  The oracle was written for finite data; here each function is compared
bit for bit (NaN payloads and the sign of zero included) with a plain-Python transcription of the Rust it restates,
written with numpy float32 scalars in loops, one rounded operation per Rust operation:
    dsp::get_min / get_max        dsp.rs:20-54
    misc::percent                 misc.rs:119-175
    read_telemetry / from_bands   telemetry.rs:125-243, :30-66
    map_signal_u8                 noaa_apt.rs:249-259
    write_wav, 16-bit samples     wav.rs:71-85
    tune_input_values             processing.rs:125-140
    equalisation table            imageext.rs:23-46, :95-119"""
import math

import numpy as np
import pytest

import oracle
import _process_oracle as po
from _post_cases import MINMAX_CASES, NAN, NEG_NAN, NAN_PAYLOAD, INF, NZ, Z, old_rule_minmax, preimages, telemetry_image

F = np.float32


def bits(v):
    return np.asarray(v, dtype=np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


# ------------------------------------------------------------------------------ transcriptions of the Rust functions

def get_max(x):
    m = x[0]
    for s in x:
        if s > m:
            m = s
    return m


def get_min(x):
    m = x[0]
    for s in x:
        if s < m:
            m = s
    return m


def as_uint(v, hi):
    """Rust `as` from f32 to an unsigned integer type of maximum hi: truncation toward zero, saturation, NaN -> 0."""
    if v != v or v <= 0:
        return 0
    return hi if v >= hi else int(math.trunc(float(v)))


def as_i16(v):
    if v != v:
        return 0
    if v >= 32767:
        return 32767
    if v <= -32768:
        return -32768
    return int(math.trunc(float(v)))


def rust_max(a, b):
    """f32::max: the non-NaN operand when one is NaN."""
    if a != a:
        return b
    if b != b:
        return a
    return a if a > b else b


def rust_min(a, b):
    if a != a:
        return b
    if b != b:
        return a
    return a if a < b else b


def rust_round(v):
    """f32::round: half away from zero (exact in f64 for |v| < 2^52)."""
    return F(math.copysign(math.floor(abs(float(v)) + 0.5), float(v)))


def percent(x, p):
    p = F(p)
    remainder = (F(1) - p) / F(2)
    buckets = [0] * 1000
    mn, mx = get_min(x), get_max(x)
    total_range = mx - mn
    for s in x:
        buckets[min(max(as_uint(np.trunc((s - mn) / total_range * F(1000)), 2**64 - 1), 0), 999)] += 1
    accum = 0
    low = high = None
    n = F(len(x))
    for b, count in enumerate(buckets):
        accum += count
        if low is None and F(accum) / n > remainder:
            low = b
        elif high is None and F(accum) / n > F(1) - remainder:
            high = b
    if high is None:
        high = 999
    return F(low) / F(1000) * total_range + mn, F(high) / F(1000) * total_range + mn


def telemetry_rows(x):
    ma, mb, var = [], [], []
    for r in range(x.size // 2080):
        line = x[r * 2080:(r + 1) * 2080]
        a, b = line[994:994 + 44], line[2034:2034 + 44]
        sa = F(0)
        for v in a:
            sa = sa + v
        sb = F(0)
        for v in b:
            sb = sb + v
        cma, cmb = sa / F(44), sb / F(44)
        va = F(0)
        for v in a:
            va = va + (v - cma) * (v - cma)
        vb = F(0)
        for v in b:
            vb = vb + (v - cmb) * (v - cmb)
        ma.append(cma)
        mb.append(cmb)
        var.append((va + vb) / F(88))
    return np.array(ma, F), np.array(mb, F), np.array(var, F)


def read_telemetry(x):
    """-> (wedges_a, wedges_b, best row); raises ValueError where the reference returns an error or panics."""
    sample = [F(v) for v in (31, 63, 95, 127, 159, 191, 224, 255, 0, 0, 0, 0, 0, 0, 0, 0,
                             31, 63, 95, 127, 159, 191, 224, 255, 0) for _ in range(8)]
    ma, mb, var = telemetry_rows(x)
    if ma.size < len(sample):
        raise ValueError("Recording too short for telemetry decoding")
    best = (0, F(0))
    sq = [np.sqrt(v) for v in var]
    for i in range(ma.size - len(sample)):
        s = F(0)
        for j in range(len(sample)):
            s = s + sample[j] * ma[i + j]
            s = s + sample[j] * mb[i + j]
        dev = F(0)
        for j in range(len(sample)):
            dev = dev + sq[i + j]
        q = s / dev
        if q > best[1]:
            best = (i, q)
    row = best[0]

    def chunks(m):
        out = []
        for c in range((m.size - row) // 8):
            t = F(0)
            for v in m[row + 8 * c: row + 8 * c + 8]:
                t = t + v
            out.append(t / F(8))
        return out[:25]
    ca, cb = chunks(ma), chunks(mb)
    if len(ca) < 25:
        raise ValueError("index out of bounds")
    wa = [(ca[w - 1] + ca[w + 15]) / F(2) if w <= 9 else ca[w - 1] for w in range(1, 17)]
    wb = [(cb[w - 1] + cb[w + 15]) / F(2) if w <= 9 else cb[w - 1] for w in range(1, 17)]
    return np.array(wa, F), np.array(wb, F), row


def map_signal_u8(x, low, high):
    low, high = F(low), F(high)
    rng = high - low
    return np.array([as_uint(rust_round(rust_min(rust_max((v - low) / rng * F(255), F(0)), F(255))), 255) for v in x],
                    np.uint8)


def quantize_i16(x):
    mx = get_max(x)
    with np.errstate(all="ignore"):
        return np.array([as_i16(v / mx * F(32767)) for v in x], np.int16)


def tune_value(v, start, end):
    s, e = F(start) * F(0.3), F(end) * F(0.3)
    out = F(v) * (F(1) + e - s) - s * F(255)
    # f32::clamp keeps NaN; `as u32` turns it into 0
    out = F(0) if out < 0 else (F(255) if out > 255 else out)
    return as_uint(out, 2**32 - 1)


def equalize_lut(counts):
    hist = []
    acc = 0
    for c in counts:
        acc = (acc + int(c)) % 2**32
        hist.append(acc)
    total = F(hist[255])
    return np.array([as_uint(F(255) * (F(h) / total), 255) for h in hist], np.uint8)


# ------------------------------------------------------------------------------ min / max

@pytest.mark.parametrize("name,x,differs", MINMAX_CASES, ids=[c[0] for c in MINMAX_CASES])
def test_minmax_is_get_min_get_max(name, x, differs):
    lo, hi = oracle.minmax(x)
    assert same(lo, get_min(x)) and same(hi, get_max(x)), name
    old = old_rule_minmax(x)
    assert (not (same(old[0], lo) and same(old[1], hi))) == differs, (name, bits(old), bits([lo, hi]))


def test_minmax_keeps_nan_payloads_through_the_binding():
    for v in (NAN, NEG_NAN, NAN_PAYLOAD):
        lo, hi = oracle.minmax(np.array([v, 1.0], F))
        assert bits(lo) == bits(v) and bits(hi) == bits(v)


# ------------------------------------------------------------------------------ percent

def _percent_inputs():
    r = np.random.default_rng(7)
    u = r.random(300, dtype=F)
    yield "uniform", u
    yield "bucket_zero_mass", np.concatenate([np.zeros(995, F), np.ones(5, F)])
    yield "quarter_ties", np.array([0.0, 0.0, 0.2, 0.2, 0.3, 0.3, 1.0, 1.0], F)
    exact, below = preimages(np.arange(0, 1001, 7, dtype=F), 0.0, 1.0, 1000.0)
    yield "bucket_edges", np.concatenate([[F(0), F(1)], exact, below])
    yield "constant", np.full(10, 0.3, F)
    yield "top_clamp", np.array([0.0, 0.999, 0.9995, 1.0, 1.0], F)
    for name, x, _ in MINMAX_CASES:
        yield name, x


@pytest.mark.parametrize("p", [0.0, 1e-7, 0.5, 0.98, 1.0])
def test_percent_is_misc_percent(p):
    for name, x in _percent_inputs():
        lo, hi = oracle.percent(x, p)
        with np.errstate(all="ignore"):
            want = percent(x, p)
        assert same(lo, want[0]) and same(hi, want[1]), (name, p, bits([lo, hi]), bits(want))


def test_percent_cases_reach_their_branches():
    # all the mass in bucket 0: low is bucket 0 and the `else if` makes high the next bucket, not bucket 0 again
    lo, hi = oracle.percent(np.concatenate([np.zeros(995, F), np.ones(5, F)]), 0.98)
    assert lo == 0.0 and same(hi, F(1) / F(1000) * F(1))
    # buckets 0, 200, 300 and 999 hold 2 of 8 pixels each: accum / total == remainder (0.25) exactly at bucket 0 and
    # == 1 - remainder at bucket 300, neither of which is "over" it
    lo, hi = oracle.percent(np.array([0.0, 0.0, 0.2, 0.2, 0.3, 0.3, 1.0, 1.0], F), 0.5)
    assert same(lo, F(200) / F(1000)) and same(hi, F(999) / F(1000))


# ------------------------------------------------------------------------------ telemetry

@pytest.mark.parametrize("rows,kw", [(199, {}), (200, {}), (201, {}), (208, {}), (230, dict(nan_row=215)),
                                     (230, dict(negative=True)), (240, dict(zero_var=(0, 240))),
                                     (260, dict(zero_var=(20, 240), seed=3))])
def test_telemetry_is_read_telemetry(rows, kw):
    x = telemetry_image(rows, **kw)
    ra, rb, rv = oracle.telemetry_rows(x)
    with np.errstate(all="ignore"):
        ta, tb, tv = telemetry_rows(x)
    assert same(ra, ta) and same(rb, tb) and same(rv, tv)
    try:
        with np.errstate(all="ignore"):
            want = read_telemetry(x)
    except ValueError:
        with pytest.raises(oracle.OracleError):
            oracle.read_telemetry(x)
        return
    wa, wb, best = oracle.read_telemetry(x)
    assert best == want[2] and same(wa, want[0]) and same(wb, want[1])
    if kw.get("negative"):
        assert best == 0                                          # every quality is below 0: best stays (0, 0.)
    if kw.get("zero_var") == (20, 240):
        assert best == 20                                         # q = +Inf from row 20 on: the first +Inf wins


# ------------------------------------------------------------------------------ map, quantisation, tunes, equalisation

def _map_inputs():
    r = np.random.default_rng(3)
    pix = np.concatenate([r.random(20, dtype=F) * F(1.2) - F(0.1),
                          np.array([NAN, NEG_NAN, INF, -INF, Z, NZ, 0.5, 1.0, 254.5 / 255, 255.5 / 255, -0.5 / 255], F)])
    for lo, hi in ((0.0, 1.0), (1.0, 0.0), (0.5, 0.5), (NAN, 1.0), (0.0, NAN), (-INF, 1.0), (0.0, INF), (NZ, Z)):
        yield pix, lo, hi
    exact, below = preimages(np.arange(-1, 256, dtype=F) + F(0.5), 0.0, 1.0, 255.0)
    yield np.concatenate([exact, below]), 0.0, 1.0


def test_map_signal_u8_is_the_reference_map():
    with np.errstate(all="ignore"):
        for x, lo, hi in _map_inputs():
            assert np.array_equal(oracle.map_signal_u8(x, lo, hi), map_signal_u8(x, lo, hi)), (lo, hi)
    # v exactly k + 0.5 (k = -1 .. 255) rounds away from zero; one ulp below it rounds down
    exact, below = preimages(np.arange(-1, 256, dtype=F) + F(0.5), 0.0, 1.0, 255.0)
    assert exact.size == 257 and below.size == 256
    assert oracle.map_signal_u8(exact, 0.0, 1.0).tolist() == [0] + list(range(1, 256)) + [255]
    v = below * F(255)                                              # k + 0.5 - 1 ulp -> k
    assert np.array_equal(oracle.map_signal_u8(below, 0.0, 1.0), np.clip(np.ceil(v) - 1, 0, 255).astype(np.uint8))


@pytest.mark.parametrize("x", [
    [NZ, -1.0, Z, -2.0], [1.0, Z, NZ, 2.0], [-1.0, NZ, Z, -3.0], [-2.0, Z, NZ, -1.5], [NAN, 1.0, 2.0],
    [0.5, NAN, 1.0, -1.0], [NEG_NAN, 0.5], [0.5, NEG_NAN, -0.25], [1.0, INF, -2.0, NAN], [-3.0, -1.0, -2.0, 0.5, -0.5],
    [1.0, 0.99999994, -1.0, -1.0000001], [3.0, 0.0, -3.0, 2.9999998], [-0.5]])
def test_quantize_i16_is_write_wav(x):
    x = np.array(x, F)
    assert np.array_equal(oracle.quantize_i16(x), quantize_i16(x))


def test_quantize_signed_zero_maximum_is_the_first_zero():
    # get_max keeps the first zero, -0.0: x / -0.0 is +Inf for x < 0 and NaN for x = ±0
    assert oracle.quantize_i16(np.array([NZ, -1.0, Z, -2.0], F)).tolist() == [0, 32767, 0, 32767]
    assert oracle.quantize_i16(np.array([Z, -1.0, NZ, -2.0], F)).tolist() == [0, -32768, 0, -32768]


@pytest.mark.parametrize("start,end", [(0.0, 0.0), (0.4, -0.3), (-5.0, 5.0), (5.0, -5.0), (3.3, 3.3), (NAN, 0.0),
                                       (0.0, NAN), (INF, 0.0), (-INF, 0.0), (0.0, INF), (0.0, -INF)])
def test_tune_values_is_tune_input_values(start, end):
    v = np.arange(256, dtype=np.uint8)
    with np.errstate(all="ignore"):
        want = np.array([tune_value(i, start, end) for i in range(256)], np.uint32)
        assert np.array_equal(po.tune_values(v, start, end), want)


def test_equalize_lut_is_the_reference_table():
    r = np.random.default_rng(5)
    for half in (r.integers(0, 256, (7, 1040), dtype=np.uint8), np.full((3, 1040), 17, np.uint8),
                 r.integers(0, 3, (20000, 1040), dtype=np.uint8)):         # 2.08e7 pixels: counts above 2^24 round
        counts = np.bincount(half.ravel(), minlength=256)
        assert np.array_equal(po.equalize_lut(half), equalize_lut(counts))
