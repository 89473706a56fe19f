"""Image and PNG output of apt_stream on the GPU: the image, info, status and PNG bytes that finish_image returns equal the
whole-recording entry points (apt_decode_image / apt_decode_png, or apt_process / apt_png_encode of apt_decode_iq's rows)
for any split into pushes, while the rows stay those of apt_decode; the mode rules, the status order, memory accounting
and concurrent streams on one device."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, image, synth
from noaa_apt_b200.err import Error as AptError

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX_PUSH = 24000


def schedules(n, rate, seed=0):
    rng = np.random.default_rng(seed)
    out = {"one": [n]}
    sizes, t = [], 0
    while t < n:
        k = int(min(n - t, rng.integers(1, 3 * MAX_PUSH + 1)))
        sizes.append(k)
        t += k
    out["random"] = sizes
    sizes, t = [], 0
    while t < min(n, 2 * rate):    # 1-7-sample pushes over the first 2 s, then large ones
        k = int(min(n - t, rng.integers(1, 8)))
        sizes.append(k)
        t += k
    while t < n:
        k = min(n - t, 5 * MAX_PUSH)
        sizes.append(k)
        t += k
    out["tiny_then_large"] = sizes
    return out


def split(x, sizes, fmt="f32"):
    pieces, t = [], 0
    for i, k in enumerate(sizes):
        p = x[t:t + k]
        if fmt == "mixed" and i % 2:
            p = p.astype(np.int16)
        pieces.append(p)
        t += k
    return pieces


@pytest.fixture(scope="module")
def palette():
    return np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]


SETTINGS = {
    "grey_minmax": dict(contrast=image.MINMAX),
    "grey_percent": dict(contrast=image.PERCENT, percent=0.98),
    "grey_telemetry": dict(contrast=image.TELEMETRY),
    "grey_histogram_rotate": dict(contrast=image.HISTOGRAM, rotate=True),
    "rgba_false_colour": dict(contrast=image.TELEMETRY, rotate=True, palette="daylight", tune=(0.4, -0.3, -0.6, 0.8),
                              rgba=True),
}


def kw_of(name, palette):
    kw = dict(SETTINGS[name])
    if kw.get("palette") == "daylight":
        kw["palette"] = palette
    return kw


def whole(x, rate, kw, png=False, sync=True):
    """(image or PNG bytes, info, status) of the whole-recording entry point."""
    try:
        if png:
            out, info = image.decode_png(None, na.Settings(), x, rate, sync, **kw)
        else:
            out, info = image.decode_image(None, na.Settings(), x, rate, sync, **kw)
        return out, info, _lib.OK
    except AptError as e:
        return None, None, e.code


def stream_pass(strm, pieces):
    """(rows of the pushes and finish_image, image, info, status)."""
    got = [strm.push(p) for p in pieces]
    try:
        rows, img, info = strm.finish_image()
        got.append(rows)
        st = _lib.OK
    except AptError as e:
        img, info, st = None, None, e.code
    return np.concatenate([g.ravel() for g in got]), img, info, st


def same_info(a, b):
    return (a["rows"] == b["rows"] and a["telemetry_row"] == b["telemetry_row"] and
            np.float32(a["low"]).tobytes() == np.float32(b["low"]).tobytes() and
            np.float32(a["high"]).tobytes() == np.float32(b["high"]).tobytes() and
            np.array_equal(a["wedges_a"].view(np.uint32), b["wedges_a"].view(np.uint32)) and
            np.array_equal(a["wedges_b"].view(np.uint32), b["wedges_b"].view(np.uint32)))


@pytest.mark.parametrize("fmt", ["f32", "mixed"])
@pytest.mark.parametrize("rate", [48000, 11025])
def test_audio_stream_image_and_png_equal_whole_recording(rate, fmt, palette):
    x = synth.apt_pcm16(rate, seconds=120, seed=5).astype(np.float32)
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        want_rows = dec.decode(x)
    scheds = schedules(x.size, rate)
    ok = 0
    with na.Stream(rate, na.Settings(), max_push=MAX_PUSH) as strm:
        for name in SETTINGS:
            kw = kw_of(name, palette)
            want_img, want_info, want_st = whole(x, rate, kw)
            want_png, _, want_png_st = whole(x, rate, kw, png=True)
            assert want_png_st == want_st
            ok += want_st == _lib.OK
            strm.reset()
            strm.set_process_mode(max_rows=300, **kw)
            for sched in ("one", "random", "tiny_then_large"):
                strm.reset()
                rows, img, info, st = stream_pass(strm, split(x, scheds[sched], fmt))
                assert st == want_st, (name, sched, st, want_st)
                if st == _lib.OK:
                    assert np.array_equal(rows.view(np.uint32), want_rows.view(np.uint32)), (name, sched)
                    assert img.dtype == np.uint8 and img.shape == want_img.shape and np.array_equal(img, want_img), (name, sched)
                    assert same_info(info, want_info), (name, sched)
            strm.reset()
            strm.set_png_mode()
            for sched in ("one", "random"):
                strm.reset()
                rows, png, info, st = stream_pass(strm, split(x, scheds[sched], fmt))
                assert st == want_st, (name, sched, st, want_st)
                if st == _lib.OK:
                    assert np.array_equal(rows.view(np.uint32), want_rows.view(np.uint32)), (name, sched)
                    assert isinstance(png, bytes) and png == want_png, (name, sched)
                    assert same_info(info, want_info), (name, sched)
    assert ok == len(SETTINGS)


@pytest.mark.parametrize("iq_rate", [1_024_000, 2_400_000])
def test_iq_stream_image_and_png_equal_process_of_decode_iq(iq_rate, palette):
    s = na.iq.IqSettings(iq_rate, offset_hz=-37_000)
    x = synth.apt_iq(iq_rate, 15.0, seed=11, offset_hz=-37_000, fmt="cu8")
    rows = na.iq.decode_iq(x, s)
    max_push = iq_rate // 5
    rng = np.random.default_rng(2)
    n = x.size // 2
    cuts = np.sort(rng.choice(np.arange(1, n), size=40, replace=False))
    bounds = np.r_[0, cuts, n]
    for kw in (dict(contrast=image.MINMAX),
               dict(contrast=image.PERCENT, rotate=True, palette=palette, tune=(0.1, 0.9, 0.2, 0.7), rgba=True)):
        want_img, want_info = image.process(rows, **kw)
        want_png = image.encode_png(want_img)
        with na.Stream.for_iq(s, max_push=max_push) as strm:
            strm.set_process_mode(max_rows=60, **kw)
            for png in (False, True):
                if png:
                    strm.reset()
                    strm.set_png_mode()
                got = [strm.push(x[2 * a:2 * b]) for a, b in zip(bounds[:-1], bounds[1:])]
                last, img, info = strm.finish_image()
                got = np.concatenate([g.ravel() for g in got + [last]])
                assert np.array_equal(got, rows)
                if png:
                    assert img == want_png
                else:
                    assert np.array_equal(img, want_img)
                assert same_info(info, want_info)


def test_full_pass_in_one_second_pushes(palette):
    rate = 48000
    x = synth.apt_pcm16(rate, seconds=900, seed=21)
    with na.Stream(rate, na.Settings(), max_push=rate) as strm:
        for kw in (dict(contrast=image.MINMAX), dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True)):
            want, want_info = image.decode_png(None, na.Settings(), x, rate, True, **kw)
            strm.reset()
            strm.set_process_mode(max_rows=2400, **kw)
            strm.set_png_mode()
            bytes0 = strm.info()["device_bytes"]
            for at in range(0, x.size, rate):
                strm.push(x[at:at + rate])
                assert strm.info()["device_bytes"] == bytes0
            _, png, info = strm.finish_image()
            assert strm.info()["device_bytes"] == bytes0
            assert png == want and info["rows"] == want_info["rows"] > 1700


def _raw_finish(strm, image_cap):
    """apt_stream_finish_image through ctypes: (status, rows, image bytes, image_n, info)."""
    lib = _lib.load()
    cap = C.c_uint64(0)
    assert lib.apt_stream_push_bound(strm._h, 0, C.byref(cap)) == 0
    rows = np.empty(max(cap.value, 2080), np.float32)
    img = np.empty(max(image_cap, 1), np.uint8)
    nout, image_n = C.c_uint64(0), C.c_uint64(0)
    ci = _lib.CImageInfo()
    st = lib.apt_stream_finish_image(strm._h, rows.ctypes.data, rows.size, C.byref(nout), img.ctypes.data, image_cap,
                                     C.byref(image_n), C.byref(ci))
    return st, rows[: nout.value], img, image_n.value, image._info(ci)


def test_status_cases():
    rate = 48000
    x = synth.apt_signal(rate, 40, seed=3)
    with na.Stream(rate, na.Settings(), max_push=MAX_PUSH) as strm:
        strm.set_process_mode(contrast=image.MINMAX, max_rows=200)
        strm.set_png_mode()
        # the decode's own status (too short), and noise: whatever the whole recording gives
        noise = np.random.default_rng(4).standard_normal(rate * 30).astype(np.float32) * 1000
        for sig in (x[: rate * 4], noise):
            want_png, _, want = whole(sig, rate, dict(contrast=image.MINMAX), png=True)
            strm.reset()
            _, png, _, st = stream_pass(strm, [sig])
            assert st == want and png == want_png
        assert whole(x[: rate * 4], rate, dict(contrast=image.MINMAX))[2] == _lib.ERR_TOO_SHORT
        # the image stage's status: telemetry on a pass too short for a frame
        _, _, want = whole(x, rate, dict(contrast=image.TELEMETRY))
        assert want == _lib.ERR_TOO_SHORT
        strm.reset()
        strm.set_process_mode(contrast=image.TELEMETRY, max_rows=200)
        _, _, _, st = stream_pass(strm, [x])
        assert st == want
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        want_rows = dec.decode(x)
    nrows = want_rows.size // 2080
    # more rows than max_rows: every row still leaves, the image is refused with the pass's row count
    with na.Stream(rate, na.Settings(), max_push=MAX_PUSH) as strm:
        strm.set_process_mode(contrast=image.MINMAX, max_rows=nrows - 7)
        pushed = [strm.push(x[a:a + 30000]) for a in range(0, x.size, 30000)]
        st, last, _, _, info = _raw_finish(strm, 1 << 24)
        assert st == _lib.ERR_CAPACITY and info["rows"] == nrows
        assert np.array_equal(np.concatenate([p.ravel() for p in pushed] + [last]), want_rows)
        assert str(nrows) in _lib.load().apt_last_error().decode()
        strm.reset()                                    # and with the Python binding
        strm.push(x)
        with pytest.raises(na.err.InvalidInput) as e:
            strm.finish_image()
        assert e.value.code == _lib.ERR_CAPACITY and str(nrows) in str(e.value)
    # image_cap too small: the required size comes back, the pass is finished
    want_png, want_info = image.decode_png(None, na.Settings(), x, rate, True, contrast=image.MINMAX)
    want_img, _ = image.decode_image(None, na.Settings(), x, rate, True, contrast=image.MINMAX)
    with na.Stream(rate, na.Settings(), max_push=MAX_PUSH) as strm:
        strm.set_process_mode(contrast=image.MINMAX, max_rows=200)
        strm.push(x)
        st, _, _, need, info = _raw_finish(strm, 1000)
        assert st == _lib.ERR_CAPACITY and need == want_img.size and info["rows"] == nrows
        with pytest.raises(na.err.InvalidInput):
            strm.push(x[:100])                          # finished
        strm.reset()
        strm.set_png_mode()
        strm.push(x)
        st, _, _, need, _ = _raw_finish(strm, 100)
        assert st == _lib.ERR_CAPACITY and need == len(want_png)
        strm.reset()
        strm.push(x)
        st, _, img, n, info = _raw_finish(strm, len(want_png))
        assert st == _lib.OK and n == len(want_png) and img[:n].tobytes() == want_png and same_info(info, want_info)


def test_mode_rules_reset_memory_and_plain_finish(palette):
    rate = 11025
    x = synth.apt_signal(rate, 40, seed=3)
    y = synth.apt_signal(rate, 55, seed=8)
    lib = _lib.load()
    with na.Stream(rate, na.Settings(), max_push=MAX_PUSH) as strm:
        base = strm.info()["device_bytes"]
        bad = [lambda: strm.set_png_mode(),                                                   # PNG without process mode
               lambda: strm.set_process_mode(contrast=image.HISTOGRAM, palette=palette),      # colour histogram
               lambda: strm.set_process_mode(contrast=image.MINMAX, max_rows=0),
               lambda: strm.set_process_mode(contrast=7)]
        for f in bad:
            with pytest.raises(na.err.InvalidInput) as e:
                f()
            assert e.value.code == _lib.ERR_BAD_ARG
        assert strm.info()["device_bytes"] == base
        strm.set_process_mode(contrast=image.MINMAX, max_rows=150)
        grey_bytes = strm.info()["device_bytes"]
        assert grey_bytes > base + 150 * 2080 * 5
        for kw in (dict(rgb_from_rgba=True), dict(block_bytes=1000), dict(filter=5)):
            with pytest.raises(na.err.InvalidInput) as e:
                strm.set_png_mode(**kw)
            assert e.value.code == _lib.ERR_BAD_ARG
        assert strm.info()["device_bytes"] == grey_bytes
        # reset keeps the modes; a second, different pass gives its own image
        strm.set_png_mode()
        for sig in (x, y):
            strm.reset()
            strm.push(sig)
            _, png, _ = strm.finish_image()
            assert png == image.decode_png(None, na.Settings(), sig, rate, True, contrast=image.MINMAX)[0]
        # no mode can change after a push
        strm.reset()
        rows = [strm.push(x[:5000])]
        for f in (lambda: strm.set_process_mode(contrast=image.PERCENT), lambda: strm.set_process_mode(None),
                  lambda: strm.set_png_mode(), lambda: strm.set_png_mode(False)):
            with pytest.raises(na.err.InvalidInput) as e:
                f()
            assert e.value.code == _lib.ERR_BAD_ARG
        # plain finish() in image mode: the rows, no image
        rows.append(strm.push(x[5000:]))
        rows.append(strm.finish())
        assert np.array_equal(np.concatenate([r.ravel() for r in rows]), na.decode(None, None, x, rate))
        # switching off frees the image output's memory
        strm.reset()
        strm.set_process_mode(None)
        assert strm.info()["device_bytes"] == base
        with pytest.raises(na.err.InvalidInput):
            strm.finish_image()
        assert lib.apt_stream_set_png_mode(strm._h, C.byref(image.png_settings())) == _lib.ERR_BAD_ARG
        # an IDAT for max_rows RGBA rows that could pass 2^31 - 1 bytes
        strm.set_process_mode(contrast=image.MINMAX, rgba=True, max_rows=240_000)
        with pytest.raises(na.err.InvalidInput) as e:
            strm.set_png_mode()
        assert e.value.code == _lib.ERR_BAD_ARG
        strm.set_process_mode(None)
        assert strm.info()["device_bytes"] == base


def test_no_sync_stream_image():
    rate = 48000
    x = synth.apt_signal(rate, 30, seed=6)
    kw = dict(contrast=image.PERCENT, rotate=True)
    want, want_info = image.decode_image(None, na.Settings(), x, rate, False, **kw)
    want_png, _ = image.decode_png(None, na.Settings(), x, rate, False, **kw)
    with na.Stream(rate, na.Settings(), sync=False, max_push=MAX_PUSH) as strm:
        strm.set_process_mode(max_rows=100, **kw)
        rows, img, info, st = stream_pass(strm, split(x, schedules(x.size, rate)["random"]))
        assert st == _lib.OK and np.array_equal(img, want) and same_info(info, want_info)
        assert np.array_equal(rows, na.decode(None, None, x, rate, sync=False))
        strm.reset()
        strm.set_png_mode()
        _, png, _, st = stream_pass(strm, [x])
        assert st == _lib.OK and png == want_png


def test_concurrent_png_streams_on_one_device(palette):
    rate = 48000
    jobs = []
    for i, kw in enumerate((dict(contrast=image.MINMAX), dict(contrast=image.PERCENT, rgba=True, palette=palette),
                            dict(contrast=image.HISTOGRAM, rotate=True), dict(contrast=image.MINMAX, rgba=True))):
        x = synth.apt_signal(rate, 90 + 10 * i, seed=30 + i)
        jobs.append((x, kw, image.decode_png(None, na.Settings(), x, rate, True, **kw)[0]))
    results = [None] * len(jobs)

    def run(i):
        x, kw, _ = jobs[i]
        try:
            with na.Stream(rate, na.Settings(), max_push=rate) as strm:
                strm.set_process_mode(max_rows=300, **kw)
                strm.set_png_mode()
                for rep in range(2):
                    strm.reset()
                    for at in range(0, x.size, 20000):
                        strm.push(x[at:at + 20000])
                    results[i] = strm.finish_image()[1]
        except Exception as e:   # noqa: BLE001 -- reported below
            results[i] = e

    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (_, _, want), got in zip(jobs, results):
        assert got == want
