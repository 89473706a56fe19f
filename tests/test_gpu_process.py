"""The rest of noaa_apt::process on the device (kernels_post.cuh: histogram equalisation, false colour, rotation) against
the CPU restatement in tests/_process_oracle.py.  Given the same f32 rows the image must be bit-identical; through
decode() the rows differ from the oracle's by <= 1e-5, which moves a few grey values by one level."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth
import oracle
import _process_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TUNES = [(0.0, 0.0, 0.0, 0.0), (0.4, -0.3, -0.6, 0.8)]
CONTRASTS = [(image.MINMAX, 0.98), (image.PERCENT, 0.98), (image.TELEMETRY, 0.98), (image.HISTOGRAM, 0.98)]


@pytest.fixture(scope="module")
def palettes():
    fx = np.load(os.path.join(GOLDEN, "palettes.npz"))
    rnd = np.random.default_rng(99).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    return {"daylight": fx["noaa-apt-daylight"], "wxtoimg": fx["WXtoImg-NO"], "random": rnd}


@pytest.fixture(scope="module")
def recording():
    x = synth.apt_signal(11025, 150, seed=12)       # 300 rows: enough for a telemetry frame (200 rows)
    return x, na.decode(na.Context(), na.Settings(), x, 11025, True)


def _variants(palettes):
    """(palette name, rgba, tune): grey, RGBA grey, and every palette with both tunes."""
    yield None, False, TUNES[0]
    yield None, True, TUNES[0]
    for name in palettes:
        for t in TUNES:
            yield name, True, t


@pytest.mark.parametrize("rotate", [False, True])
@pytest.mark.parametrize("contrast,percent", CONTRASTS)
def test_process_bit_exact_on_the_gpu_rows(recording, palettes, contrast, percent, rotate):
    _, rows = recording
    for name, rgba, tune in _variants(palettes):
        pal = palettes[name] if name else None
        if pal is not None and contrast == image.HISTOGRAM:
            continue                                    # refused: test_errors
        img, info = image.process(rows, contrast, percent, rotate, pal, tune, rgba)
        ref, (low, high) = po.process(rows, contrast, percent, rotate, pal, tune, rgba)
        assert (info["low"], info["high"]) == (low, high) and info["rows"] == rows.size // 2080
        assert img.shape == ref.shape and np.array_equal(img, ref), (name, rgba, tune)


def _synthetic_rows(n_rows, seed):
    """An APT-like image: sync bars, a flat space band, telemetry wedges 8 rows high, noise, clipped pixels."""
    r = np.random.default_rng(seed)
    img = r.normal(0.5, 0.15, (n_rows, 2080)).astype(np.float32)
    for x0 in (0, 1040):
        img[:, x0:x0 + 39] = ((np.arange(39) // 4) % 2).astype(np.float32)
        img[:, x0 + 39:x0 + 86] = np.float32(0.05 if x0 == 0 else 0.9)
        img[:, x0 + 995:x0 + 1040] = ((np.arange(n_rows) // 8) % 16 / 15.0).astype(np.float32)[:, None]
    img[r.random(img.shape) < 0.03] = np.float32(1.5)
    img[r.random(img.shape) < 0.03] = np.float32(-0.5)
    return img


def test_process_20000_rows_bit_exact(palettes):
    # 20 000 rows: 20.8 M pixels per channel half, above 2^24, so the u32 -> f32 conversions of the equalisation round
    rows = _synthetic_rows(20000, 7)
    for contrast, rotate, pal, rgba in ((image.HISTOGRAM, True, None, False), (image.HISTOGRAM, False, None, True),
                                        (image.MINMAX, True, palettes["random"], True)):
        img, _ = image.process(rows, contrast, 0.98, rotate, pal, TUNES[1], rgba)
        ref, _ = po.process(rows, contrast, 0.98, rotate, pal, TUNES[1], rgba)
        assert np.array_equal(img, ref), (contrast, rotate, rgba)


def _grey(rows, contrast, percent=0.98):
    low, high = po.bounds(rows.ravel(), contrast, percent)
    return oracle.map_signal_u8(rows.ravel(), low, high).reshape(-1, 2080)


@pytest.mark.parametrize("sync", [True, False])
def test_decode_image_forms_agree_and_match_the_oracle(recording, palettes, sync):
    x, _ = recording
    pcm = synth.apt_pcm16(11025, 150, seed=12)
    rows = na.decode(na.Context(), na.Settings(), x, 11025, sync)
    cases = [dict(contrast=image.HISTOGRAM, rotate=True),
             dict(contrast=image.TELEMETRY if sync else image.PERCENT, rotate=True, palette=palettes["daylight"], tune=TUNES[1]),
             dict(contrast=image.PERCENT, percent=0.95, rgba=True),
             dict(contrast=image.MINMAX)]
    dec = na.Decoder(11025, na.Settings(), max_samples=x.size)
    for kw in cases:
        img, info = image.decode_image(na.Context(), na.Settings(), x, 11025, sync, **kw)
        img16, info16 = image.decode_image(na.Context(), na.Settings(), pcm, 11025, sync, **kw)
        dec.set_process_mode(**kw)
        img_dec = dec.decode(x, sync)
        img_dec16 = dec.decode(pcm, sync)
        assert np.array_equal(img, img16) and np.array_equal(img, img_dec) and np.array_equal(img, img_dec16), kw
        assert dec.image_info()["low"] == info["low"] and info16["high"] == info["high"]
        # bit-exact against the oracle's process applied to the GPU's own rows
        ref, (low, high) = po.process(rows, kw["contrast"], kw.get("percent", 0.98), kw.get("rotate", False),
                                      kw.get("palette"), kw.get("tune", TUNES[0]), kw.get("rgba"))
        assert (info["low"], info["high"]) == (low, high)
        assert np.array_equal(img, ref), kw
    dec.set_process_mode(None)
    assert np.array_equal(dec.decode(x, sync), rows)                # back to f32 rows
    dec.close()


def test_decode_image_close_to_the_all_oracle_pipeline(recording, palettes):
    """The rows of the device agree with the oracle's to 1e-5, so a grey value can differ by one level where a row value
    sits on a rounding edge of map_signal_u8 (< 0.2 % of the pixels).  Where the two grey images agree the results must
    agree too, up to one level in histogram mode: the cumulative histograms differ by the few moved pixels k, which
    moves 255 * cum / total by 255 * k / total < 1 level."""
    x, _ = recording
    ref_rows = oracle.decode(x, 11025).reshape(-1, 2080)
    pal = palettes["wxtoimg"]
    for contrast, kw in ((image.MINMAX, {}), (image.HISTOGRAM, {}), (image.PERCENT, dict(palette=pal, tune=TUNES[1]))):
        img, _ = image.decode_image(na.Context(), na.Settings(), x, 11025, True, contrast, **kw)
        ref, _ = po.process(ref_rows, contrast, 0.98, False, kw.get("palette"), kw.get("tune", TUNES[0]), kw.get("rgba"))
        gpu_rows = na.decode(na.Context(), na.Settings(), x, 11025, True).reshape(-1, 2080)
        same = _grey(gpu_rows, contrast) == _grey(ref_rows, contrast)
        assert same.mean() > 0.998, contrast
        diff = np.abs(img.astype(np.int16) - ref.astype(np.int16))
        if diff.ndim == 3:
            diff = diff.max(axis=2)
        if "palette" in kw:
            both = same.copy()
            both[:, 86:995] &= same[:, 1126:2035]                   # a coloured pixel reads channel A and channel B
            assert diff[both].max() == 0
        else:
            assert diff[same].max() <= (1 if contrast == image.HISTOGRAM else 0)
            assert diff.max() <= 1 or contrast == image.HISTOGRAM


def test_full_size_48khz_recording(palettes):
    pcm = synth.apt_pcm16(48000, 900, seed=3)
    rows = na.decode(na.Context(), na.Settings(), pcm, 48000, True)
    for contrast, kw in ((image.TELEMETRY, dict(rotate=True, palette=palettes["daylight"], tune=TUNES[1])),
                         (image.HISTOGRAM, dict(rotate=True))):
        img, info = image.decode_image(na.Context(), na.Settings(), pcm, 48000, True, contrast, **kw)
        assert info["rows"] == rows.size // 2080 >= 1700
        ref, _ = po.process(rows, contrast, 0.98, kw["rotate"], kw.get("palette"), kw.get("tune", TUNES[0]), kw.get("rgba"))
        assert np.array_equal(img, ref), contrast


def test_image_mode_launches_are_unchanged_and_process_mode_counts_its_kernels(recording):
    x, _ = recording
    lib = na._lib.load()
    dec = na.Decoder(11025, na.Settings(), max_samples=x.size)
    bound = dec.out_bound(x.size)

    def launches(fn):
        c0 = dec.launch_count
        out = fn()
        return dec.launch_count - c0, out

    dec.decode(x, True)                                             # first job: lazy allocations
    plain, _ = launches(lambda: dec.decode(x, True))
    for contrast, extra in ((image.MINMAX, 3), (image.PERCENT, 4), (image.TELEMETRY, 3)):
        assert lib.apt_decoder_set_image_mode(dec._h, contrast, 0.98) == 0
        n, img = launches(lambda: (dec.submit(x, True, out=np.empty(bound, np.uint8)), dec.wait())[1].copy())
        assert n == plain + extra, contrast                          # stats, (percent histogram), bounds, map
        ref, _ = image.decode_image_u8(na.Context(), na.Settings(), x, 11025, True, contrast, 0.98)
        assert np.array_equal(img, ref.ravel())
    # process mode: + post_map_u8_hist, post_eq_lut and post_finish as needed
    for kw, extra in ((dict(contrast=image.MINMAX), 3), (dict(contrast=image.HISTOGRAM), 5),
                      (dict(contrast=image.MINMAX, rotate=True), 4), (dict(contrast=image.PERCENT, rgba=True), 5)):
        dec.set_process_mode(**kw)
        n, _ = launches(lambda: dec.decode(x, True))
        assert n == plain + extra, kw
    dec.set_process_mode(contrast=image.HISTOGRAM, rotate=True)
    dec.set_profiling(True)
    dec.decode(x, True)
    names = [k for k, _ in dec.kernel_times_ms()]
    assert names[-5:] == ["post_stats", "post_bounds", "post_map_u8_hist", "post_eq_lut", "post_finish"]
    dec.close()


def test_errors(recording, palettes):
    x, _ = recording
    lib = na._lib.load()
    with pytest.raises(na.err.InvalidInput, match="colour histogram equalisation is not available"):
        image.decode_image(na.Context(), na.Settings(), x, 11025, True, image.HISTOGRAM, palette=palettes["daylight"])
    with pytest.raises(na.err.InvalidInput):
        image.decode_image(na.Context(), na.Settings(), x, 11025, True, image.MINMAX, palette=palettes["daylight"], rgba=False)
    dec = na.Decoder(11025, na.Settings(), max_samples=x.size)
    with pytest.raises(na.err.InvalidInput, match="colour histogram"):
        dec.set_process_mode(image.HISTOGRAM, palette=palettes["random"])
    dec.close()
    # a short buffer: the required size counts 4 bytes per pixel for RGBA
    s = na.Settings().to_c()
    out = np.empty(16, np.uint8)
    n = C.c_uint64(0)
    need = {}
    for rgba in (False, True):
        ps, _, _keep = image.process_settings(image.MINMAX, rgba=rgba)
        st = lib.apt_decode_image(x.ctypes.data, na._lib.F32, x.size, 11025, C.byref(s), 1, C.byref(ps), out.ctypes.data,
                                  out.size, C.byref(n), None, na._lib.STATUS_CB(0), None)
        assert st == na._lib.ERR_CAPACITY
        need[rgba] = int(re.search(rb"(\d+) bytes", lib.apt_last_error()).group(1))
    assert need[True] == 4 * need[False] and need[False] % 2080 == 0 and need[False] >= 290 * 2080
    # "Recording too short for telemetry decoding" is still Internal / APT_ERR_TOO_SHORT
    short = synth.apt_signal(11025, 60, seed=4)                     # 120 rows < 200
    with pytest.raises(na.err.Internal, match="too short for telemetry") as e:
        image.decode_image(na.Context(), na.Settings(), short, 11025, True, image.TELEMETRY, rotate=True,
                           palette=palettes["wxtoimg"])
    assert e.value.code == na._lib.ERR_TOO_SHORT
    with pytest.raises(na.err.Internal):
        image.process(na.decode(na.Context(), na.Settings(), short, 11025, True), image.TELEMETRY, rgba=True)
