"""The image stage (kernels_post.cuh) bit for bit at its edges: min / max, MinMax and Percent bounds, telemetry, the u8
map, histogram equalisation, false colour, rotation and the 16-bit quantisation, each against the C oracle and
tests/_process_oracle.py applied to the same f32 rows (both checked against the Rust functions in
test_post_oracle_cpu.py).  Floats compare as their u32 bits, images with np.array_equal.

The inputs are the ones where such kernels go wrong: NaN (at pixel 0, in the middle, last, in a row another CTA
reads), NaN payloads, signed zeros tied at the minimum or maximum, infinities, subnormals, bucket and rounding edges,
quality ties on different threads, and row counts at the kernels' grid and stride limits.

A NaN the stage computes (Percent bounds from a NaN minimum, a telemetry mean of a NaN band) is CUDA's canonical NaN,
while the x86 oracle keeps the operand's payload: those values compare as "both NaN".  Min / max and MinMax bounds are
pixels, not results of arithmetic, and compare with their payloads."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth, wav
import oracle
import _process_oracle as po
from _post_cases import (MINMAX_CASES, NAN, NEG_NAN, NAN_PAYLOAD, NEG_NAN_PAYLOAD, INF, SUB, SUB_MAX, NZ, Z, preimages,
                         telemetry_image)

pytestmark = pytest.mark.gpu
F = np.float32
PERCENTS = [0.0, 1e-7, 0.5, 0.98, 1.0]


def bits(v):
    return np.asarray(v, dtype=np.float32).view(np.uint32)


def same(a, b):
    """bit for bit, NaN payloads included"""
    return np.array_equal(bits(a), bits(b))


def same_nan(a, b):
    """bit for bit, except that any two NaNs agree"""
    a, b = np.asarray(a, F), np.asarray(b, F)
    na_, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na_, nb) and np.array_equal(bits(np.where(na_, 0, a)), bits(np.where(nb, 0, b)))


@pytest.fixture(scope="module")
def wide_rows():
    """Rows enough that k_post_stats' CTAs each take more than one row (its grid is sm_count * 8 CTAs)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 + 40


def _rows(n, seed=0, negative=False):
    x = np.random.default_rng(seed).random((n, 2080), dtype=F) * F(0.8) + F(0.1)
    return -x if negative else x


def _check_process(rows, contrast, percent=0.98, **kw):
    img, info = image.process(rows, contrast, percent, **kw)
    kw["rotate_"] = kw.pop("rotate", False)
    want, (lo, hi) = po.process(rows, contrast, percent, **kw)
    assert np.array_equal(img, want)
    exact = same if contrast in (image.MINMAX, image.HISTOGRAM) else same_nan
    assert exact([info["low"], info["high"]], [lo, hi]), (bits([info["low"], info["high"]]), bits([lo, hi]))
    return img


# ------------------------------------------------------------------------------ min / max and the MinMax bounds

@pytest.mark.parametrize("name,x,differs", MINMAX_CASES, ids=[c[0] for c in MINMAX_CASES])
def test_minmax_edge_cases(name, x, differs):
    lo, hi, _ = image.contrast_bounds(x, image.MINMAX)
    assert same([lo, hi], oracle.minmax(x)), (bits([lo, hi]), bits(oracle.minmax(x)))


@pytest.mark.parametrize("name,x,differs", MINMAX_CASES, ids=[c[0] for c in MINMAX_CASES])
def test_percent_on_minmax_edge_cases(name, x, differs):
    for p in PERCENTS:
        lo, hi, _ = image.contrast_bounds(x, image.PERCENT, p)
        assert same_nan([lo, hi], oracle.percent(x, p)), (p, bits([lo, hi]), bits(oracle.percent(x, p)))


def _edit(kind, x):
    last = x.shape[0] - 1
    if kind == "nan_first":
        x[0, 0] = NAN_PAYLOAD
    elif kind == "nan_middle":
        x[x.shape[0] // 2, 1500] = NAN
    elif kind == "nan_last":
        x[last, 2079] = NEG_NAN_PAYLOAD
    elif kind == "nan_far_row":                                      # a row of the last CTAs, not CTA 0's
        x[last - 3, 17] = NEG_NAN
    elif kind in ("min_zeros_neg_first", "min_zeros_pos_first"):
        first, second = (NZ, Z) if kind == "min_zeros_neg_first" else (Z, NZ)
        x[5, 100], x[last - 1, 7] = first, second
    elif kind in ("max_zeros_neg_first", "max_zeros_pos_first"):
        x *= F(-1)
        first, second = (NZ, Z) if kind == "max_zeros_neg_first" else (Z, NZ)
        x[2, 2000], x[last, 3] = first, second
    elif kind == "infinities":
        x[last - 4, 9], x[3, 3] = INF, -INF
    elif kind == "subnormals":
        r = np.random.default_rng(9)
        x[...] = (r.integers(1, 0x7FFFFF, x.shape, dtype=np.uint32) | (r.integers(0, 2, x.shape, dtype=np.uint32) << 31)).view(F)
        x[last, 1], x[1, 5] = SUB_MAX, -SUB_MAX
    elif kind == "min_tie_across_ctas":                              # the same smallest value in three rows
        x[last, 40] = x[1, 30] = x[last // 2, 20] = F(0.0625)
    return x


EDITS = ["nan_first", "nan_middle", "nan_last", "nan_far_row", "min_zeros_neg_first", "min_zeros_pos_first",
         "max_zeros_neg_first", "max_zeros_pos_first", "infinities", "subnormals", "min_tie_across_ctas"]


@pytest.mark.parametrize("kind", EDITS)
def test_bounds_and_images_across_ctas(kind, wide_rows):
    x = _edit(kind, _rows(wide_rows, seed=EDITS.index(kind)))
    lo, hi, info = image.contrast_bounds(x, image.MINMAX)
    assert same([lo, hi], oracle.minmax(x)) and info["rows"] == wide_rows
    for contrast in (image.MINMAX, image.PERCENT, image.HISTOGRAM):
        _check_process(x, contrast)


@pytest.mark.parametrize("x", [np.full((3, 2080), 0.3, F), _rows(1, 4), np.array([0.25], F), _rows(3, 5).ravel()[:2 * 2080 + 5],
                               np.concatenate([[NAN], _rows(2, 6).ravel()[:4000]])],
                         ids=["constant", "one_row", "one_pixel", "not_whole_rows", "not_whole_rows_nan_first"])
def test_small_and_partial_images(x):
    lo, hi, info = image.contrast_bounds(x, image.MINMAX)
    assert same([lo, hi], oracle.minmax(x))
    for p in PERCENTS:
        lo, hi, _ = image.contrast_bounds(x, image.PERCENT, p)
        assert same_nan([lo, hi], oracle.percent(x, p)), p
    if x.size % 2080 == 0:
        for contrast in (image.MINMAX, image.PERCENT, image.HISTOGRAM):
            _check_process(x.reshape(-1, 2080), contrast, rotate=True)


# ------------------------------------------------------------------------------ Percent

def _percent_cases():
    e1, b1 = preimages(np.arange(0, 1001, dtype=F), 0.0, 1.0, 1000.0)   # (x - min) / range * 1000 == k, and 1 ulp below
    e2, b2 = preimages(np.arange(0, 1001, dtype=F), -3.0, 5.0, 1000.0)
    yield "bucket_edges", np.concatenate([[F(0), F(1)], e1, b1])
    yield "bucket_edges_offset", np.concatenate([[F(-3), F(5)], b2, e2])
    yield "top_clamp", np.array([0.0, 0.998, 0.999, 0.99949, 0.9995, 0.99999994, 1.0, 1.0], F)
    yield "bucket_zero_mass", np.concatenate([np.zeros(995, F), np.ones(5, F)])
    yield "quarter_ties", np.array([0.0, 0.0, 0.2, 0.2, 0.3, 0.3, 1.0, 1.0], F)
    yield "range_zero", np.full(4160, -0.7, F)


@pytest.mark.parametrize("name,x", list(_percent_cases()), ids=[c[0] for c in _percent_cases()])
def test_percent_edges(name, x):
    for p in PERCENTS:
        lo, hi, _ = image.contrast_bounds(x, image.PERCENT, p)
        assert same([lo, hi], oracle.percent(x, p)), (p, bits([lo, hi]), bits(oracle.percent(x, p)))
    if name == "bucket_zero_mass":                                    # the `else if`: high is bucket 1, not bucket 0
        assert image.contrast_bounds(x, image.PERCENT, 0.98)[:2] == (0.0, float(F(1) / F(1000)))
    if name == "quarter_ties":                                        # accum / total == 1/4 is not over the remainder
        assert image.contrast_bounds(x, image.PERCENT, 0.5)[:2] == (float(F(0.2)), float(F(0.999)))


def test_percent_rounds_its_counts_above_2_24_pixels():
    r = np.random.default_rng(11)
    x = (r.random((8200, 2080), dtype=F) ** 3).astype(F)             # 17 056 000 pixels: total and accum round to f32
    x[4100, 7] = NAN
    for p in PERCENTS:
        lo, hi, _ = image.contrast_bounds(x, image.PERCENT, p)
        assert same([lo, hi], oracle.percent(x, p)), p


# ------------------------------------------------------------------------------ telemetry

def _telemetry_cases(sm_rows):
    yield "rows_199", telemetry_image(199)
    for n in (200, 201, 208, 1224, 1225, 1226):                    # 1225: the search's 1 024 threads start to stride
        yield f"rows_{n}", telemetry_image(n, seed=n)
    for name, n in (("rows_sm-1", sm_rows - 1), ("rows_sm", sm_rows), ("rows_sm+1", sm_rows + 1)):   # k_post_stats' grid
        yield name, telemetry_image(n, seed=n)
    yield "periodic_100", telemetry_image(1400, seed=2, period=100)
    yield "periodic_1100", telemetry_image(2300, seed=3, period=1100)
    yield "all_negative", telemetry_image(500, negative=True)
    yield "zero_variance_all", telemetry_image(240, zero_var=(0, 240))
    yield "zero_variance_run", telemetry_image(1300, seed=4, zero_var=(1030, 1260))
    yield "nan_band", telemetry_image(400, seed=5, nan_row=150)


@pytest.fixture(scope="module")
def telemetry_cases():
    sm_rows = torch.cuda.get_device_properties(0).multi_processor_count * 8
    return dict(_telemetry_cases(sm_rows))


@pytest.mark.parametrize("case", ["rows_199", "rows_200", "rows_201", "rows_208", "rows_1224", "rows_1225", "rows_1226",
                                  "rows_sm-1", "rows_sm", "rows_sm+1", "periodic_100", "periodic_1100", "all_negative",
                                  "zero_variance_all", "zero_variance_run", "nan_band"])
def test_telemetry(case, telemetry_cases):
    x = telemetry_cases[case]
    a, b, v = image.telemetry_rows(x)
    ra, rb, rv = oracle.telemetry_rows(x)
    assert same_nan(a, ra) and same_nan(b, rb) and same_nan(v, rv)
    if x.size // 2080 < 200:
        with pytest.raises(na.err.Internal) as e:
            image.contrast_bounds(x, image.TELEMETRY)
        assert e.value.code == na._lib.ERR_TOO_SHORT
        with pytest.raises(oracle.OracleError):
            oracle.read_telemetry(x)
        return
    lo, hi, info = image.contrast_bounds(x, image.TELEMETRY)
    wa, wb, best = oracle.read_telemetry(x)
    assert info["telemetry_row"] == best
    assert same(info["wedges_a"], wa) and same(info["wedges_b"], wb)
    assert same([lo, hi], po.bounds(x, po.TELEMETRY))
    # the case does what it is there for: the first of equal qualities, (0, 0.) kept, the first +Inf
    first = {"periodic_100": best < 100, "periodic_1100": best < 1100, "all_negative": best == 0,
             "zero_variance_all": best == 0, "zero_variance_run": best == 1030}
    assert first.get(case, True), best
    if case.startswith("periodic"):
        _check_process(x.reshape(-1, 2080), image.TELEMETRY, rotate=True, rgba=True)


# ------------------------------------------------------------------------------ the u8 map

def _map_pixels(n):
    exact, below = preimages(np.arange(-1, 256, dtype=F) + F(0.5), 0.0, 1.0, 255.0)   # v = k + 0.5, and 1 ulp below
    special = np.array([NAN, NEG_NAN, INF, -INF, Z, NZ, SUB, 0.5, 1.0], F)
    x = np.resize(np.concatenate([special, exact, below]), n)
    if n > 4:
        x[-3:] = exact[100:103]                                      # ties in the scalar tail after the float4 loop too
    return x


@pytest.mark.parametrize("n", [1, 2, 3, 5, 4099])
def test_map_signal_u8_edges(n):
    x = _map_pixels(n)
    for lo, hi in ((0.0, 1.0), (1.0, 0.0), (0.5, 0.5), (NAN, 1.0), (0.0, NAN), (-INF, 1.0), (0.0, INF), (NZ, Z), (Z, NZ),
                   (0.0, 255.0), (-1e-30, 1e30)):
        assert np.array_equal(image.map_signal_u8(x, lo, hi), oracle.map_signal_u8(x, lo, hi)), (n, lo, hi)


def test_map_rounds_half_away_from_zero():
    exact, _ = preimages(np.array([-0.5, 0.5, 1.5, 127.5, 254.5, 255.5], F), 0.0, 1.0, 255.0)
    assert image.map_signal_u8(exact, 0.0, 1.0).tolist() == [0, 1, 2, 128, 255, 255]


# ------------------------------------------------------------------------------ process: equalisation, colour, rotation

_A, _B = np.meshgrid(np.arange(256), np.arange(256))                            # palette[b][a]: 65 536 distinct entries
PALETTE = np.stack([_A, _B, (_A * 7 + _B * 13) & 255], -1).astype(np.uint8)
OUTPUTS = {"grey_minmax": dict(contrast=image.MINMAX), "rgba_percent": dict(contrast=image.PERCENT, rgba=True),
           "hist": dict(contrast=image.HISTOGRAM), "hist_rgba": dict(contrast=image.HISTOGRAM, rgba=True),
           "palette": dict(contrast=image.MINMAX, palette=PALETTE, tune=(0.4, -0.3, -0.6, 0.8))}


@pytest.mark.parametrize("out", list(OUTPUTS))
@pytest.mark.parametrize("rotate", [False, True])
@pytest.mark.parametrize("rows", [1, 2, 3, 301])
def test_process(rows, rotate, out):
    x = _rows(rows, seed=rows)
    x[:, 2000:2079] = np.linspace(0, 1, 79, dtype=F)                 # every grey value present somewhere
    kw = dict(OUTPUTS[out])
    _check_process(x, kw.pop("contrast"), rotate=rotate, **kw)


@pytest.mark.parametrize("rotate", [False, True])
def test_process_channel_half_of_one_grey_value(rotate):
    x = _rows(40, seed=8)
    x[:, 1040:] = F(0.5)
    for contrast in (image.HISTOGRAM, image.MINMAX):
        _check_process(x, contrast, rotate=rotate)


def test_equalisation_counts_above_2_24_pixels():
    # 17 000 rows: channel A's half holds 17 680 000 pixels, the first 17 610 667 of them grey 0 and the rest 255.
    # Neither count is an f32: hist[0] rounds to nearest (up, 17 610 668), and 255 * hist[0] / total truncates to 254;
    # rounded toward zero it would give 253.
    rows, h = 17000, 17610667
    x = np.full((rows, 2080), 0.5, F)
    half = np.ones(rows * 1040, F)
    half[:h] = 0.0
    x[:, :1040] = half.reshape(rows, 1040)
    img = _check_process(x, image.HISTOGRAM)
    assert img[0, 0] == 254


@pytest.mark.parametrize("tune", [(0.16, 0.2, 0.08, -0.77),       # one value of each channel rounds differently under FMA
                                  (-4.0, 4.0, 4.0, -4.0), (3.4, 3.4, -3.4, -3.4), (float("nan"), float("inf"), float("-inf"), 0.0),
                                  (0.0, float("nan"), 1e30, -1e30)])
def test_false_colour_tunes(tune):
    x = _rows(7, seed=9)
    x[:, 86:995] = np.linspace(0, 1, 909, dtype=F)
    x[:, 1126:2035] = np.linspace(1, 0, 909, dtype=F)
    for rotate in (False, True):
        _check_process(x, image.MINMAX, rotate=rotate, palette=PALETTE, tune=tune)


# ------------------------------------------------------------------------------ 16-bit quantisation (wav.rs:71-85)

def _quantize_cases():
    r = np.random.default_rng(13)
    yield "max_zeros_neg_first", np.array([NZ, -1.0, Z, -2.0], F)
    yield "max_zeros_pos_first", np.array([Z, -1.0, NZ, -2.0], F)
    yield "nan_first", np.array([NAN, 1.0, -2.0, 3.0], F)
    yield "nan_middle", np.array([1.0, NAN, -2.0, 0.5], F)
    yield "neg_nan", np.array([0.25, NEG_NAN, 1.0, -1.0], F)
    yield "max_inf", np.array([1.0, INF, -INF, -2.0], F)
    yield "negative_max", np.array([-3.0, -1.0, -2.0, -0.5, -1e-3], F)
    mx = F(0.75)
    near = mx * np.array([1.0, 0.99999994, -1.0, -1.0000305, -1.0000153, -1.0001, 32766.5 / 32767], F)
    yield "near_full_scale", np.concatenate([[mx], near]).astype(F)
    yield "one", np.array([-0.3], F)
    yield "five", np.array([0.1, -0.2, 0.3, -0.4, 0.25], F)
    big = -r.random(2**20 + 3, dtype=F)
    big[100], big[2**20] = NZ, Z
    yield "big_max_zeros", big
    big = r.standard_normal(2**20 + 3).astype(F)
    big[0] = NAN_PAYLOAD
    yield "big_nan_first", big
    big = r.standard_normal(2**20 + 3).astype(F)
    big[2**19 + 1] = NEG_NAN
    yield "big_neg_nan_middle", big


@pytest.mark.parametrize("name,x", list(_quantize_cases()), ids=[c[0] for c in _quantize_cases()])
def test_quantize_i16(name, x):
    assert np.array_equal(wav.quantize_i16(x), oracle.quantize_i16(x))


# ------------------------------------------------------------------------------ through the decoder

@pytest.fixture(scope="module", params=[(11025, "nan"), (11025, "inf"), (48000, "nan"), (48000, "inf")],
                ids=["11025-nan", "11025-inf", "48000-nan", "48000-inf"])
def bad_recording(request):
    rate, kind = request.param
    x = synth.apt_signal(rate, 20, seed=21)
    x[x.size // 2 + 17] = NAN if kind == "nan" else INF
    rows = na.decode(na.Context(), na.Settings(), x, rate, False)
    assert rows.size % 2080 == 0
    return rate, x, rows.reshape(-1, 2080)


@pytest.mark.parametrize("contrast", [image.MINMAX, image.PERCENT, image.HISTOGRAM])
def test_decoder_process_and_png_with_a_non_finite_sample(bad_recording, contrast):
    rate, x, rows = bad_recording
    want, (lo, hi) = po.process(rows, contrast)
    exact = same if contrast != image.PERCENT else same_nan
    img, info = image.decode_image(None, na.Settings(), x, rate, sync=False, contrast=contrast)
    assert np.array_equal(img, want)
    assert exact([info["low"], info["high"]], [lo, hi])
    png, info = image.decode_png(None, na.Settings(), x, rate, sync=False, contrast=contrast)
    with Image.open(io.BytesIO(png)) as im:
        assert np.array_equal(np.asarray(im), want)
    assert exact([info["low"], info["high"]], [lo, hi])
    if contrast == image.MINMAX:
        assert np.isfinite([lo, hi]).all() or np.isnan(rows.ravel()[0])   # one NaN pixel does not blank the image
