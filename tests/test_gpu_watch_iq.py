"""Watching one SDR's I/Q feed on several channels (DESIGN.md §14).

Kernel: apt_fm_demod_channels equals apt_fm_demod per offset bit for bit, for every format, channel count and chunking.
Contract: for every split of the feed into pushes, channel c's q, LOS passes and each pass's decode equal the recording
path (apt_recording_quality, apt_find_passes_quality, apt_recording_decode) on a_c = fm_demod(feed, offsets[c]), bit for
bit.  Truth: each synthetic pass is found once, on its own channel, where its fades put it.  Then the edges: 1.024 Msps at
the NOAA offsets, max_rows, small segments, reset, device memory, threads and equality with an audio Watch on a_c."""
import os
import threading

import numpy as np
import pytest

import __graft_entry__ as entry

pytestmark = pytest.mark.gpu

RATE = 250_000                                  # audio_rate 50 kHz, D = 5
OFFSETS = [-80_000, 0, 80_000]                  # channel 2 carries a noise band and no carrier
SEARCH = dict(max_gap_s=10.0, min_length_s=30.0)
FADE_S = 10.0
PASSES = [(-80_000, 5, 5.0, 75.0), (0, 6, 35.0, 115.0)]   # (offset, seed, on_s, off_s): they overlap from 35 s to 75 s
BANDS = [(80_000, 30_000, 0.5)]
SECONDS = 125.0
PAL = np.random.default_rng(3).integers(0, 256, (256, 256, 3), dtype=np.uint8)
MODES = {
    "rows": dict(image_out=None),
    "png": dict(image_out="png"),
    "rgba": dict(image_out="image", contrast=2, palette=PAL, rotate=True, rgba=True),   # contrast 2: image.TELEMETRY
}


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.fail("no CUDA device")
    return noaa_apt_b200


_cache = {}


def feed(fmt="cu8"):
    from noaa_apt_b200 import synth
    if fmt not in _cache:
        _cache[fmt] = synth.apt_iq_passes(RATE, SECONDS, PASSES, extra_bands=BANDS, fmt=fmt, fade_s=FADE_S)
    return _cache[fmt]


def iq_settings(na, rate=RATE):
    return na.iq.IqSettings(rate)


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


def _same(a, b):
    return a.size == b.size and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------- the kernel

@pytest.mark.parametrize("fmt", ["cu8", "cs16", "cf32"])
@pytest.mark.parametrize("offsets", [[0], [-400_000, 0, 120_000], [0, -400_000, 120_000, 412_500, -200_000, 120_000,
                                                                  300_000, -37_000]])
@pytest.mark.parametrize("chunk", [None, 100_003, 31_337])
def test_fm_demod_channels_equals_fm_demod_per_offset(na, fmt, offsets, chunk):
    from noaa_apt_b200 import synth
    rate = 1_024_000
    if ("multi", fmt) not in _cache:
        _cache[("multi", fmt)] = synth.apt_iq_multi(rate, 0.3, carriers=((120_000, 3, 0.0, None, 60.0),
                                                                         (-400_000, 4, 0.0, None, 60.0)), fmt=fmt)
    x = _cache[("multi", fmt)]
    s = iq_settings(na, rate)
    env = _env("APTB200_IQ_CHUNK", chunk) if chunk else _env("APTB200_UNUSED", 0)
    with env:
        got = na.iq.fm_demod_channels(x, s, offsets)
        for c, off in enumerate(offsets):
            want = na.iq.fm_demod(x, na.iq.IqSettings(rate, offset_hz=off))
            assert _same(got[c], want), (c, off)
    assert len(got) == len(offsets)


# -------------------------------------------------------------------------------------------------------- the contract

def audio(na, x, offsets=OFFSETS, rate=RATE):
    return [na.iq.fm_demod(x, na.iq.IqSettings(rate, offset_hz=o)) for o in offsets]


def reference(na, a, rate, mode, sync=True, search=SEARCH):
    """q, passes, and (status, data, info) per pass from the recording path on the audio a."""
    kw = dict(MODES[mode])
    image_out = kw.pop("image_out")
    with na.Recording(a, rate) as rec:
        q = rec.quality()
        found = na.find_passes_quality(q, a.size, rate, **search)
        if not found:
            return q, found, []
        if image_out is None:
            data, sts = rec.decode(found, sync)
            infos = [None] * len(found)
        elif image_out == "image":
            data, infos, sts = rec.decode_image(found, sync, **kw)
        else:
            data, infos, sts = rec.decode_png(found, sync, **kw)
    return q, found, list(zip(sts, data, infos))


def run(na, pieces, mode, offsets=OFFSETS, rate=RATE, sync=True, search=SEARCH, w=None, **extra):
    """Pushes the pieces, then finishes: ([q per channel], [(channel, event)])."""
    own = w is None
    if own:
        w = na.IqWatch(iq_settings(na, rate), offsets, sync=sync, search=search, **MODES[mode], **extra)
    qs, evs = [[] for _ in offsets], []
    for piece in pieces:
        q, e = w.push(piece)
        for c in range(len(offsets)):
            qs[c].append(q[c])
        evs += e
    q, e = w.finish()
    for c in range(len(offsets)):
        qs[c].append(q[c])
    evs += e
    if own:
        w.close()
    return [np.concatenate(v) for v in qs], evs


def check(na, a, rate, q, evs, mode, sync=True, search=SEARCH):
    """The check() of test_gpu_watch.py on one channel: q, LOS passes and each pass's bytes."""
    q_ref, found, dec = reference(na, a, rate, mode, sync, search)
    assert _same(q, q_ref)
    los = [e for e in evs if e.kind == "los"]
    aos = [e for e in evs if e.kind == "aos"]
    assert [e.pass_ for e in los] == found
    assert [e.index for e in los] == list(range(len(found)))
    for e in los:
        a0 = [v for v in aos if v.index == e.index]
        pos = [i for i, v in enumerate(evs) if v is a0[0] or v is e]
        assert len(a0) == 1 and evs[pos[0]] is a0[0] and a0[0].pass_.start == e.pass_.start
    for e, (st, data, info) in zip(los, dec):
        assert e.status == st
        if st != 0:
            continue
        if isinstance(data, bytes):
            assert e.data == data
        else:
            assert e.data.shape == data.shape and np.array_equal(e.data.view(np.uint8), data.view(np.uint8))
        if info is not None:
            for k in ("low", "high", "rows", "telemetry_row"):
                assert e.info[k] == info[k]
            assert np.array_equal(e.info["wedges_a"], info["wedges_a"])
    return found


def check_all(na, x_ref, q, evs, mode, offsets=OFFSETS, rate=RATE, sync=True, search=SEARCH):
    """check() on every channel; x_ref: the feed as one array whose fm_demod is each channel's a_c."""
    s = iq_settings(na, rate)
    found = []
    for c, a in enumerate(audio(na, x_ref, offsets, rate)):
        found.append(check(na, a, s.audio_rate, q[c], [e for ch, e in evs if ch == c], mode, sync, search))
    return found


def _split(x, sizes):
    """Interleaved cu8 x cut into pieces of `sizes` complex samples (cycled)."""
    out, at, i = [], 0, 0
    n = x.size // 2
    while at < n:
        k = int(sizes[i % len(sizes)])
        out.append(x[2 * at:2 * min(at + k, n)])
        at += k
        i += 1
    return out


def _mixed(pieces):
    """Pieces in cu8, cs16 and cf32 by turns, and the one cf32 feed whose loaded values are the same: cu8 u loads as
    u - 127.5 and cs16 v as v, so a cs16 piece carries 2u - 255 (the same signal, twice the scale)."""
    out, ref = [], []
    for i, p in enumerate(pieces):
        v = p.astype(np.float32) - np.float32(127.5)
        if i % 3 == 0:
            out.append(p)
            ref.append(v)
        elif i % 3 == 1:
            w = (2 * p.astype(np.int16) - 255).astype(np.int16)
            out.append(w)
            ref.append(w.astype(np.float32))
        else:
            out.append(v.view(np.complex64))
            ref.append(v)
    return out, np.concatenate(ref).view(np.complex64)


@pytest.mark.parametrize("schedule,mode,sync", [("whole", "rows", True), ("half_s", "png", True),
                                                ("random", "rgba", True), ("mixed", "rows", True),
                                                ("random", "rows", False)])
def test_feed_equals_the_recording_path_per_channel(na, schedule, mode, sync):
    x = feed()
    max_push = RATE // 2
    rng = np.random.default_rng(11)
    sizes = {"whole": [x.size // 2], "half_s": [RATE // 2], "random": rng.integers(1, 3 * max_push, 256).tolist(),
             "mixed": rng.integers(1, 3 * max_push, 256).tolist()}[schedule]
    pieces = _split(x, sizes)
    x_ref = x
    if schedule == "mixed":
        pieces, x_ref = _mixed(pieces)
    q, evs = run(na, pieces, mode, sync=sync, max_push=max_push)
    found = check_all(na, x_ref, q, evs, mode, sync=sync)
    assert [len(f) for f in found] == [1, 1, 0]


def test_single_sample_pushes_around_pass_edges(na):
    x = feed()
    s = iq_settings(na)
    D = s.decimation
    a = audio(na, x)
    edges = []
    for c in (0, 1):
        _q, found, _d = reference(na, a[c], s.audio_rate, "rows")
        edges += [e * D for p in found for e in (p.start, p.end)]
    n = x.size // 2
    cuts = sorted(e for e in edges if 2000 < e < n - 2000)
    sizes, at = [], 0
    for e in cuts:
        sizes.append(e - 1000 - at)
        sizes += [1] * 2000
        at = e + 1000
    sizes.append(n - at)
    assert all(k > 0 for k in sizes)
    q, evs = run(na, _split(x, sizes), "rows", max_push=4096)
    check_all(na, x, q, evs, "rows")


# ------------------------------------------------------------------------------------------------------------ the truth

def test_each_pass_found_once_on_its_own_channel(na):
    from noaa_apt_b200 import synth
    x = feed()
    s = iq_settings(na)
    D = s.decimation
    q, evs = run(na, _split(x, [RATE // 2]), "png", max_push=RATE // 2)
    truth = synth.apt_iq_passes_truth(RATE, PASSES, fade_s=FADE_S)
    margin = (0.5 * FADE_S + 12.0) * RATE           # the fade, plus a window, the gap rule and q's threshold
    for c, off in enumerate(OFFSETS):
        los = [e for ch, e in evs if ch == c and e.kind == "los"]
        mine = [t for t in truth if t[0] == off]
        assert len(los) == len(mine), (c, los)
        for e, (_off, t0, t1) in zip(los, mine):
            assert e.status == 0 and e.data[:8] == b"\x89PNG\r\n\x1a\n"
            assert abs(e.pass_.start * D - t0) < margin and abs(e.pass_.end * D - t1) < margin, (c, e.pass_, t0, t1)
    assert [e for ch, e in evs if ch == 2] == []     # the noise band's channel
    # both passes open when the feed ends: one push and the finish fire LOS on channels 0 and 1 in channel order
    cut = 2 * int(74 * RATE)
    w = na.IqWatch(s, OFFSETS, search=SEARCH)
    _q, e1 = w.push(x[:cut])
    _q, e2 = w.finish()
    w.close()
    assert all(e.kind == "aos" for _c, e in e1)
    assert [(c, e.kind) for c, e in e2] == [(0, "los"), (1, "los")]


# ---------------------------------------------------------------------------------------------------------- once each

def test_noaa_offsets_at_1024_ksps(na):
    from noaa_apt_b200 import synth
    rate = 1_024_000
    offs = [-400_000, 120_000, 412_500]
    search = dict(max_gap_s=5.0, min_length_s=20.0)
    x = synth.apt_iq_passes(rate, 50.0, [(-400_000, 3, 2.0, 38.0), (412_500, 4, 10.0, 50.0)], fmt="cu8", fade_s=4.0)
    q, evs = run(na, _split(x, [rate // 2]), "png", offsets=offs, rate=rate, search=search, max_push=rate // 2)
    found = check_all(na, x, q, evs, "png", offsets=offs, rate=rate, search=search)
    assert [len(f) for f in found] == [1, 0, 1]


def test_pass_longer_than_max_rows_beside_a_good_one(na):
    x = feed()
    s = iq_settings(na)
    a = audio(na, x)
    _q0, f0, _ = reference(na, a[0], s.audio_rate, "png")
    _q1, f1, dec1 = reference(na, a[1], s.audio_rate, "png")
    r0, r1 = (2 * (f[0].end - f[0].start) // s.audio_rate for f in (f0, f1))
    max_rows = (r0 + r1) // 2
    assert r0 + 4 < max_rows < r1 - 4
    q, evs = run(na, _split(x, [RATE]), "png", max_rows=max_rows)
    los = [(c, e) for c, e in evs if e.kind == "los"]
    assert [c for c, _e in los] == [0, 1]
    assert los[0][1].status == 0
    assert los[1][1].status == na._lib.ERR_CAPACITY and los[1][1].rows > max_rows and los[1][1].data is None
    _qr, _f, dec0 = reference(na, a[0], s.audio_rate, "png")
    assert los[0][1].data == dec0[0][1]


def test_small_segments_roll_per_channel(na):
    x = feed()
    s = iq_settings(na)
    a = audio(na, x)
    T = 40 * 12480                                  # 40 s of work samples
    with _env("APTB200_WATCH_SEGMENT", T):
        q, evs = run(na, _split(x, [RATE // 2]), "rows", max_push=RATE // 2)
    rolls = {}
    for c in range(3):
        segs = [e for ch, e in evs if ch == c and e.kind == "segment"]
        starts = [0] + [e.pass_.start for e in segs] + [a[c].size]
        rolls[c] = starts
        assert len(starts) >= 3
        qat = 0
        for lo, hi in zip(starts, starts[1:]):
            with na.Recording(a[c][lo:hi], s.audio_rate) as rec:
                q_ref = rec.quality()
            assert _same(q[c][qat:qat + q_ref.size], q_ref)
            qat += q_ref.size
            found = na.find_passes_quality(q_ref, hi - lo, s.audio_rate, **SEARCH)
            los = [e.pass_ for ch, e in evs if ch == c and e.kind == "los" and lo <= e.pass_.start < hi]
            assert [(p.start - lo, p.end - lo, p.first_window, p.windows, p.mean_quality) for p in los] == \
                [(p.start, p.end, p.first_window, p.windows, p.mean_quality) for p in found]
        assert qat == q[c].size
    assert rolls[0] != rolls[2]                     # the empty channel rolls at other steps than the busy ones


def test_reset_device_bytes_threads_and_the_audio_watcher(na):
    x = feed()
    s = iq_settings(na)
    from noaa_apt_b200.passes import watch_iq_geometry
    geo = watch_iq_geometry(s, OFFSETS, search=SEARCH, max_push=RATE // 2, **MODES["png"])
    w = na.IqWatch(s, OFFSETS, search=SEARCH, max_push=RATE // 2, **MODES["png"])
    assert w.device_bytes == geo["device_bytes"]
    run(na, _split(x[: 2 * 80 * RATE], [RATE // 2]), "png", w=w)
    assert w.device_bytes == geo["device_bytes"]
    info = w.info(1)
    assert info["samples_in"] == 80 * RATE and info["max_push"] == RATE // 2 and info["passes"] == 1
    w.reset()
    q2, e2 = run(na, _split(x, [RATE // 2]), "png", w=w)
    assert w.device_bytes == geo["device_bytes"]
    w.close()
    q3, e3 = run(na, _split(x, [RATE // 2]), "png", max_push=RATE // 2)
    key = [(c, e.kind, e.pass_, e.status, e.data) for c, e in e3]
    assert all(_same(u, v) for u, v in zip(q2, q3)) and [(c, e.kind, e.pass_, e.status, e.data) for c, e in e2] == key

    results, errors = [None] * 2, []

    def work(i):
        try:
            results[i] = run(na, _split(x, [RATE // (2 * (i + 1))]), "png", max_push=RATE // 2)
        except Exception as ex:   # reported below
            errors.append(ex)
    ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors
    for q, evs in results:
        assert all(_same(u, v) for u, v in zip(q, q3))
        assert [(c, e.kind, e.pass_, e.status, e.data) for c, e in evs] == key
    # under the default segment length, channel c is an audio Watch fed a_c
    a = audio(na, x)
    for c in range(3):
        wa = na.Watch(s.audio_rate, search=SEARCH, **MODES["png"])
        qa, ea = wa.push(a[c])
        qf, ef = wa.finish()
        wa.close()
        assert _same(q3[c], np.concatenate([qa, qf]))
        assert [(e.kind, e.window, e.pass_, e.index, e.status, e.data) for e in ea + ef] == \
            [(e.kind, e.window, e.pass_, e.index, e.status, e.data) for ch, e in e3 if ch == c]


def test_audio_formats_and_callbacks_into_the_watcher_are_refused(na):
    import ctypes as C
    L = na._lib
    lib = L.load()
    s = iq_settings(na)
    w = na.IqWatch(s, OFFSETS, search=SEARCH)
    q = np.empty(4096, np.float32)
    nq = (C.c_uint64 * 3)()
    x = np.zeros(8, np.float32)
    for fmt in (L.F32, L.PCM16):
        assert lib.apt_watch_iq_push(w._h, x.ctypes.data, fmt, 4, q.ctypes.data, q.size, nq) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_get_info(w._h, 3, C.byref(L.CWatchInfo())) == L.ERR_BAD_ARG
    w.close()

    seen = []
    h = C.c_void_p(None)

    def cb(channel, pev, _user):
        info = L.CWatchInfo()
        seen.append((channel, pev.contents.ev.kind, lib.apt_watch_iq_get_info(h, channel, C.byref(info)),
                     lib.apt_watch_iq_reset(h)))
    ccb = L.WATCH_IQ_CB(cb)
    from noaa_apt_b200.passes import watch_settings
    ws = watch_settings(search=SEARCH)
    cs = na.Settings().to_c()
    qs = s.to_c()
    offs = (C.c_int32 * 3)(*OFFSETS)
    assert lib.apt_watch_iq_create(0, C.byref(qs), offs, 3, C.byref(cs), C.byref(ws), ccb, None, C.byref(h)) == L.OK
    xf = feed()[: 2 * 60 * RATE]
    cap = C.c_uint64(0)
    assert lib.apt_watch_iq_push_bound(h, xf.size // 2, C.byref(cap)) == L.OK
    qb = np.empty(3 * cap.value, np.float32)
    assert lib.apt_watch_iq_push(h, xf.ctypes.data, L.CU8, xf.size // 2, qb.ctypes.data, cap.value, nq) == L.OK
    lib.apt_watch_iq_destroy(h)
    assert seen and seen[0][:2] == (0, L.PASS_AOS)
    assert all(r[2:] == (L.ERR_BAD_ARG, L.ERR_BAD_ARG) for r in seen)
