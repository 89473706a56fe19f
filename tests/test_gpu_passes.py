"""Finding passes on the device (DESIGN.md §12): q against a float64 restatement of the decoder's own envelope, the same
bits on every run and for every chunk size, the rule on the device's q, passes found in synthetic multi-pass recordings
and none in real receiver noise or silence, and every decoded range equal to the one-shot decode of the host slice."""
import ctypes as C
import os

import numpy as np
import pytest

import __graft_entry__ as entry
import _passes_oracle as po

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# noise, a pass, noise, a pass, silence, a pass, noise: 1040 s
LAYOUT = [("noise", 100), ("pass", 240, 1), ("noise", 80), ("pass", 240, 2), ("silence", 80), ("pass", 240, 3),
          ("noise", 60)]
SHORT = [("noise", 20), ("pass", 70, 5), ("silence", 15), ("noise", 15)]


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.fail("no CUDA device")
    return noaa_apt_b200


_cache = {}


def recording(rate, layout=LAYOUT, seed=0):
    from noaa_apt_b200 import synth
    key = (rate, id(layout), seed)
    if key not in _cache:
        _cache[key] = synth.apt_passes(rate, layout, seed=seed)
    return _cache[key]


def _env(name, value):
    class Env:
        def __enter__(self):
            self.old = os.environ.get(name)
            os.environ[name] = str(value)

        def __exit__(self, *exc):
            if self.old is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = self.old
    return Env()


@pytest.mark.parametrize("rate", [11025, 48000])
@pytest.mark.parametrize("fmt", ["f32", "pcm16"])
def test_quality_matches_float64_restatement_and_is_bit_stable(na, rate, fmt):
    pcm = recording(rate, SHORT)
    x = pcm if fmt == "pcm16" else pcm.astype(np.float32)
    with na.Decoder(rate, max_samples=x.size) as dec:
        dec.decode(x, sync=False)
        e = dec.read_stage(0)
    row = na.Settings().to_c().work_rate // 2
    want = po.quality(e, row)
    with na.Recording(x, rate) as rec:
        q = rec.quality()
        q2 = rec.quality()
        info = rec.info()
    assert info["windows"] == q.size == want.size == len(e) // row - 1
    assert info["work_samples"] == len(e) and info["row_samples"] == row
    assert np.max(np.abs(q.astype(np.float64) - want)) <= 1e-4
    assert np.array_equal(q.view(np.uint32), q2.view(np.uint32))
    with _env("APTB200_CHUNK_SAMPLES", 65536):          # many small chunks: still the same bits
        with na.Recording(x, rate) as rec:
            q3 = rec.quality()
    assert np.array_equal(q.view(np.uint32), q3.view(np.uint32))
    # the pass in the middle is well above exit, the silence is exactly 0
    assert np.median(q[50:170]) > 0.7
    assert np.all(q[int(2 * 92):int(2 * 103)] == 0.0)


def test_device_quality_through_the_rule(na):
    pcm = recording(11025)
    with na.Recording(pcm, 11025) as rec:
        q = rec.quality()
        found = [p.__dict__ for p in rec.find_passes()]
        for kw in (dict(min_length_s=20), dict(enter=0.9, exit=0.5, max_gap_s=5)):
            assert [p.__dict__ for p in rec.find_passes(**kw)] == po.find_passes(q, pcm.size, 11025, **kw)
    assert found == po.find_passes(q, pcm.size, 11025)


@pytest.mark.parametrize("rate", [11025, 48000])
def test_three_passes_found_near_the_fades(na, rate):
    from noaa_apt_b200 import synth
    pcm = recording(rate)
    with na.Recording(pcm, rate) as rec:
        found = rec.find_passes()
    truth = synth.apt_passes_truth(rate, LAYOUT)
    assert len(found) == 3, found
    for p, (a, b) in zip(found, truth):
        assert abs(p.start - a) <= 10 * rate and abs(p.end - b) <= 10 * rate, (p, a, b)
        assert p.peak_quality > 0.8 and p.mean_quality > 0.5


def test_no_pass_in_noise_silence_or_a_short_recording(na):
    g = np.load(os.path.join(HERE, "golden", "noise_11025hz.npz"))
    with na.Recording(g["pcm"], 11025) as rec:
        q = rec.quality()
        assert rec.find_passes(min_length_s=5) == []
    assert q.size > 50 and np.max(np.abs(q)) < po.EXIT
    with na.Recording(np.zeros(11025 * 120, np.int16), 11025) as rec:
        q = rec.quality()
        assert rec.find_passes() == []
    assert np.all(q == 0.0)
    short = recording(11025, SHORT)[20 * 11025:20 * 11025 + 11025 * 9 // 10]    # 0.9 s: fewer than 2R work samples
    with na.Recording(short, 11025) as rec:
        assert rec.info()["windows"] == 0 and rec.quality().size == 0 and rec.find_passes() == []


def _host(fn):
    try:
        return 0, fn()
    except na_err() as e:
        return e.code, None


def na_err():
    from noaa_apt_b200 import err
    return err.Error


def _ranges(rate, found):
    n = recording(rate).size
    r = [(p.start, p.end) for p in found]
    r.append((found[0].start + 1, found[0].start + 1 + 61 * rate))           # odd start, misaligned for f32 and PCM16
    r.append((7 * rate + 3, 7 * rate + 3 + 3 * rate))                       # 3 s: too short
    r.append((n - 45 * rate - 5, n))                                        # odd start, ends with the recording
    return r


@pytest.mark.parametrize("rate,fmt", [(11025, "pcm16"), (48000, "f32")])
def test_decoded_ranges_equal_the_host_slices(na, rate, fmt):
    from noaa_apt_b200 import image
    pcm = recording(rate)
    x = pcm if fmt == "pcm16" else pcm.astype(np.float32)
    pal = np.random.default_rng(3).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    na._lib.load().apt_cache_clear()
    with na.Recording(x, rate) as rec:
        bytes0 = rec.device_bytes
        found = rec.find_passes()
        assert len(found) == 3
        ranges = _ranges(rate, found)
        rows, sts = rec.decode(ranges, sync=True)
        grey, ginf, gsts = rec.decode_image(ranges, contrast=image.MINMAX)
        pngs, pinf, psts = rec.decode_png(ranges, contrast=image.TELEMETRY, palette=pal, rotate=True)
        assert rec.device_bytes == bytes0
    for i, (a, b) in enumerate(ranges):
        st, want = _host(lambda: na.decode(None, None, x[a:b], rate))
        assert sts[i] == st
        if st == 0:
            assert np.array_equal(rows[i].view(np.uint32), want.view(np.uint32))
        st, want = _host(lambda: image.decode_image(None, None, x[a:b], rate, contrast=image.MINMAX))
        assert gsts[i] == st
        if st == 0:
            assert np.array_equal(grey[i], want[0])
            assert ginf[i]["rows"] == want[1]["rows"] and ginf[i]["low"] == want[1]["low"] and ginf[i]["high"] == want[1]["high"]
        st, want = _host(lambda: image.decode_png(None, None, x[a:b], rate, contrast=image.TELEMETRY, palette=pal,
                                                  rotate=True))
        assert psts[i] == st
        if st == 0:
            assert pngs[i] == want[0]
            for k in ("low", "high", "rows", "telemetry_row"):
                assert pinf[i][k] == want[1][k]
            assert np.array_equal(pinf[i]["wedges_a"], want[1]["wedges_a"])
            assert np.array_equal(pinf[i]["wedges_b"], want[1]["wedges_b"])
    assert sts[:3] == [0, 0, 0] and sts[4] == na._lib.ERR_TOO_SHORT and sts[3] == 0


def test_long_range_against_the_chunked_host_upload(na):
    """A range longer than the host decoder's chunk threshold: apt_decode_png uploads it in chunks, the recording decodes
    it from device memory; the bytes agree.  A range whose PNG does not fit fails alone, with the size it needs."""
    from noaa_apt_b200 import image
    rate = 11025
    pcm = recording(rate)
    with na.Recording(pcm, rate) as rec:
        found = rec.find_passes()
        ranges = [(found[1].start + 1, found[1].end), (found[2].start, found[2].end)]
        pngs, _inf, sts = rec.decode_png(ranges, contrast=image.TELEMETRY)
        lib = na._lib.load()
        arr = (na._lib.CPass * 2)()
        for i, (a, b) in enumerate(ranges):
            arr[i].start, arr[i].end = a, b
        ps, _bpp, _pal = image.process_settings(image.TELEMETRY)
        png = image.png_settings()
        outs = [np.empty(1 << 22, np.uint8), np.empty(100, np.uint8)]
        nouts = (C.c_uint64 * 2)()
        st2 = (C.c_int * 2)()
        rc = lib.apt_recording_decode(rec._h, arr, 2, 1, C.byref(ps), C.byref(png), (C.c_void_p * 2)(*[o.ctypes.data for o in outs]),
                                      (C.c_uint64 * 2)(outs[0].size, outs[1].size), nouts, None, st2)
        assert rc == na._lib.ERR_CAPACITY and list(st2) == [0, na._lib.ERR_CAPACITY]
        assert outs[0][: nouts[0]].tobytes() == pngs[0] and nouts[1] == len(pngs[1])
    assert sts == [0, 0]
    with _env("APTB200_CHUNK_SAMPLES", 1 << 20):
        na._lib.load().apt_cache_clear()
        for (a, b), got in zip(ranges, pngs):
            assert b - a > 2 << 20
            want, _ = image.decode_png(None, None, pcm[a:b], rate, contrast=image.TELEMETRY)
            assert got == want
    na._lib.load().apt_cache_clear()


def test_decode_argument_errors_and_device_bytes(na):
    import torch
    from noaa_apt_b200 import image
    L = na._lib
    lib = L.load()
    pcm = recording(11025, SHORT)
    with na.Recording(pcm, 11025) as warm:       # load every kernel module the cycle uses before measuring
        warm.quality()
        warm.decode([(0, pcm.size)], sync=False)
    lib.apt_cache_clear()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    rec = na.Recording(pcm, 11025)
    used = free0 - torch.cuda.mem_get_info(0)[0]
    db = rec.device_bytes
    assert db >= pcm.size * 2 and abs(used - db) <= 8 << 20, (used, db)
    rec.quality()
    assert rec.device_bytes == db
    k = 2
    arr = (L.CPass * k)()
    arr[0].start, arr[0].end = 0, 30 * 11025
    arr[1].start, arr[1].end = 10, 10
    out = np.empty(1 << 20, np.float32)
    outs = (C.c_void_p * k)(out.ctypes.data, out.ctypes.data)
    caps = (C.c_uint64 * k)(out.size, out.size)
    nouts = (C.c_uint64 * k)()
    sts = (C.c_int * k)()
    assert lib.apt_recording_decode(rec._h, arr, k, 1, None, None, outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    assert list(sts) == [L.ERR_BAD_ARG] * k                       # an empty range
    arr[1].start, arr[1].end = 10, pcm.size + 1
    assert lib.apt_recording_decode(rec._h, arr, k, 1, None, None, outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    arr[1].start, arr[1].end = 10, pcm.size
    png = image.png_settings()
    assert lib.apt_recording_decode(rec._h, arr, k, 1, None, C.byref(png), outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    ps, _bpp, _pal = image.process_settings(image.MINMAX)
    ps.contrast = 17
    assert lib.apt_recording_decode(rec._h, arr, k, 1, C.byref(ps), None, outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    ps.contrast = image.MINMAX
    png.rgb_from_rgba = 1                                         # grey output
    assert lib.apt_recording_decode(rec._h, arr, k, 1, C.byref(ps), C.byref(png), outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    assert list(sts) == [L.ERR_BAD_ARG] * k
    assert lib.apt_recording_decode(rec._h, arr, k, 1, None, None, outs, caps, nouts, None, sts) == L.OK
    assert rec.device_bytes == db
    rec.close()
    lib.apt_cache_clear()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info(0)[0] - free0) <= 8 << 20


def test_decode_passes_png_one_call(na):
    from noaa_apt_b200 import image
    pcm = recording(11025)
    got = na.decode_passes_png(pcm, 11025, contrast=image.MINMAX)
    assert len(got) == 3
    for p, png, info in got:
        want, winfo = image.decode_png(None, None, pcm[p.start:p.end], 11025, contrast=image.MINMAX)
        assert png == want and info["rows"] == winfo["rows"]
