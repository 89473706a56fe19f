"""Watching a feed on the device (DESIGN.md §13): for every split of a feed into pushes, the watcher's q, its passes and
each pass's decode equal what the recording path (apt_recording_quality, apt_find_passes_quality, apt_recording_decode)
returns for the same samples, bit for bit; no events in real noise or silence; dropped bursts, passes open at finish,
passes longer than max_rows, segments, reset, constant device memory and watchers in threads."""
import os
import threading

import numpy as np
import pytest

import __graft_entry__ as entry

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

SEARCH = dict(max_gap_s=10.0, min_length_s=30.0)
# noise, a pass, silence, a pass, noise: 175 s
LAYOUT = [("noise", 20), ("pass", 65, 5), ("silence", 25), ("pass", 55, 6), ("noise", 10)]
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


def recording(rate, layout=LAYOUT, seed=0):
    from noaa_apt_b200 import synth
    key = (rate, id(layout), seed)
    if key not in _cache:
        _cache[key] = synth.apt_passes(rate, layout, seed=seed)
    return _cache[key]


def reference(na, x, rate, mode, sync=True, search=SEARCH, max_rows=None):
    """q, passes, and (status, rows, data, info) per pass from the recording path."""
    kw = dict(MODES[mode])
    image_out = kw.pop("image_out")
    with na.Recording(x, rate) as rec:
        q = rec.quality()
        found = na.find_passes_quality(q, x.size, rate, **search)
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


def run(na, x, rate, sizes, mode, sync=True, search=SEARCH, mixed=False, w=None, **extra):
    """Pushes x in pieces of `sizes` (cycled), then finishes: (q, events)."""
    own = w is None
    if own:
        w = na.Watch(rate, sync=sync, search=search, **MODES[mode], **extra)
    qs, evs = [], []
    at, i = 0, 0
    while at < x.size:
        k = int(sizes[i % len(sizes)])
        piece = x[at:at + k]
        if mixed and i % 2:
            piece = piece.astype(np.float32)
        q, e = w.push(piece)
        qs.append(q)
        evs += e
        at += k
        i += 1
    q, e = w.finish()
    qs.append(q)
    evs += e
    if own:
        w.close()
    return np.concatenate(qs), evs


def check(na, x, rate, q, evs, mode, sync=True, search=SEARCH):
    q_ref, found, dec = reference(na, x, rate, mode, sync, search)
    assert q.size == q_ref.size and np.array_equal(q.view(np.uint32), q_ref.view(np.uint32))
    los = [e for e in evs if e.kind == "los"]
    aos = [e for e in evs if e.kind == "aos"]
    assert [e.pass_ for e in los] == found
    assert [e.index for e in los] == list(range(len(found)))
    for e in los:   # each AOS precedes its LOS, with the same start
        a = [v for v in aos if v.index == e.index]
        pos = [i for i, v in enumerate(evs) if v is a[0] or v is e]
        assert len(a) == 1 and evs[pos[0]] is a[0] and a[0].pass_.start == e.pass_.start
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


def _schedules(rate, max_push):
    rng = np.random.default_rng(rate)
    return {
        "1s": [rate],
        "random": rng.integers(1, 3 * max_push, 64).tolist(),
    }


@pytest.mark.parametrize("rate", [11025, 48000])
@pytest.mark.parametrize("schedule,mode,mixed,sync", [("1s", "rows", False, True), ("random", "png", False, True),
                                                      ("1s", "rgba", True, True), ("random", "rows", True, False)])
def test_feed_equals_the_recording_path(na, rate, schedule, mode, mixed, sync):
    x = recording(rate)
    max_push = rate // 2
    sizes = _schedules(rate, max_push)[schedule]
    q, evs = run(na, x, rate, sizes, mode, sync=sync, mixed=mixed, max_push=max_push)
    found = check(na, x, rate, q, evs, mode, sync)
    assert len(found) == 2


def test_single_sample_pushes_around_a_start_and_an_end(na):
    rate = 11025
    x = recording(rate)
    q_ref, found, _ = reference(na, x, rate, "rows")
    assert len(found) == 2
    cuts = []
    for p in found:
        for c in (p.start, p.end):
            cuts += [c - rate, c + rate]
    sizes, at = [], 0
    for a, b in zip(cuts[::2], cuts[1::2]):
        sizes.append(a - at)
        sizes += [1] * (b - a)
        at = b
    sizes.append(x.size - at)
    w = na.Watch(rate, search=SEARCH, max_push=4096)
    qs, evs, at = [], [], 0
    for k in sizes:
        q, e = w.push(x[at:at + k])
        qs.append(q)
        evs += e
        at += k
    q, e = w.finish()
    w.close()
    check(na, x, rate, np.concatenate(qs + [q]), evs + e, "rows")


def test_no_events_in_real_noise_or_silence(na):
    g = np.load(os.path.join(HERE, "golden", "noise_11025hz.npz"))
    for x in (g["pcm"], np.zeros(11025 * 40, np.int16)):
        q, evs = run(na, x, 11025, [11025], "rows", search={})
        assert evs == []
        with na.Recording(x, 11025) as rec:
            q_ref = rec.quality()
        assert np.array_equal(q.view(np.uint32), q_ref.view(np.uint32))


def test_burst_then_pass_and_a_pass_open_at_finish(na):
    rate = 11025
    # a 20 s burst (shorter than min_length) and a pass the feed ends inside
    layout = [("noise", 10), ("pass", 20, 7), ("noise", 15), ("pass", 60, 8), ("noise", 12), ("pass", 80, 9)]
    x = recording(rate, layout)[: -20 * rate]
    q, evs = run(na, x, rate, [rate], "png")
    found = check(na, x, rate, q, evs, "png")
    assert len(found) == 2 and found[0].start > 35 * rate
    assert found[-1].end > x.size - rate                   # its LOS came at finish
    assert [e.kind for e in evs if e.pass_.start < 35 * rate] == []


def test_pass_longer_than_max_rows_then_a_good_one(na):
    rate = 11025
    x = recording(rate)
    q_ref, found, dec = reference(na, x, rate, "png")
    rows0, rows1 = (2 * (p.end - p.start) // rate for p in found)
    # max_rows between the two passes' row counts: the first is refused, the second decodes
    max_rows = (rows0 + rows1) // 2
    assert rows1 + 4 < max_rows < rows0 - 4
    for mode in ("png", "rows"):
        q, evs = run(na, x, rate, [rate], mode, max_rows=max_rows)
        los = [e for e in evs if e.kind == "los"]
        assert [e.pass_ for e in los] == found
        assert los[0].status == na._lib.ERR_CAPACITY and los[0].rows > max_rows and los[0].data is None
        _q, _f, dec = reference(na, x, rate, mode)
        assert los[1].status == 0
        want = dec[1][1]
        if isinstance(want, bytes):
            assert los[1].data == want
        else:
            assert np.array_equal(los[1].data.view(np.uint32), want.view(np.uint32))


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


def test_segments_each_equal_the_recording_path(na):
    rate = 11025
    x = recording(rate)
    T = 60 * 12480                      # 60 s of work samples
    with _env("APTB200_WATCH_SEGMENT", T):
        w = na.Watch(rate, search=SEARCH)
    qs, evs, at = [], [], 0
    while at < x.size:
        q, e = w.push(x[at:at + rate])
        qs.append(q)
        evs += e
        at += rate
    q, e = w.finish()
    qs.append(q)
    evs += e
    w.close()
    q = np.concatenate(qs)
    starts = [0] + [e.pass_.start for e in evs if e.kind == "segment"] + [x.size]
    assert len(starts) >= 3                 # the first segment ends after the first pass (open at T)
    qat = 0
    for a, b in zip(starts, starts[1:]):
        seg = x[a:b]
        with na.Recording(seg, rate) as rec:
            q_ref = rec.quality()
        assert np.array_equal(q[qat:qat + q_ref.size].view(np.uint32), q_ref.view(np.uint32))
        qat += q_ref.size
        found = na.find_passes_quality(q_ref, seg.size, rate, **SEARCH)
        los = [e.pass_ for e in evs if e.kind == "los" and a <= e.pass_.start < b]
        assert [(p.start - a, p.end - a, p.first_window, p.windows, p.mean_quality, p.peak_quality) for p in los] == \
            [(p.start, p.end, p.first_window, p.windows, p.mean_quality, p.peak_quality) for p in found]
    assert qat == q.size
    # with T = 30 s a pass is still open when its segment reaches 2T: its LOS fires at that segment's finish (window W of
    # the segment), right before the SEGMENT event
    with _env("APTB200_WATCH_SEGMENT", 30 * 12480):
        q2, evs2 = run(na, x, rate, [rate], "rows")
    kinds = [(e.kind, e.window) for e in evs2]
    assert any(a == ("los", b[1]) and b[0] == "segment" for a, b in zip(kinds, kinds[1:]))


def test_reset_device_bytes_and_threads(na):
    rate = 11025
    x = recording(rate)
    from noaa_apt_b200.passes import watch_geometry
    geo = watch_geometry(rate, search=SEARCH, **MODES["png"])
    w = na.Watch(rate, search=SEARCH, **MODES["png"])
    assert w.device_bytes == geo["device_bytes"]
    q1, e1 = run(na, x[: 120 * rate], rate, [rate], "png", w=w)
    assert w.device_bytes == geo["device_bytes"]
    w.reset()
    q2, e2 = run(na, x, rate, [rate], "png", w=w)
    assert w.device_bytes == geo["device_bytes"]
    w.close()
    q3, e3 = run(na, x, rate, [rate], "png")
    assert np.array_equal(q2.view(np.uint32), q3.view(np.uint32))
    assert [(e.kind, e.pass_, e.status, e.data) for e in e2] == [(e.kind, e.pass_, e.status, e.data) for e in e3]

    results, errors = [None] * 4, []

    def work(i):
        try:
            results[i] = run(na, x, rate, [rate // (i + 1)], "png")
        except Exception as ex:   # reported below
            errors.append(ex)
    ts = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors
    for q, evs in results:
        assert np.array_equal(q.view(np.uint32), q3.view(np.uint32))
        assert [(e.kind, e.pass_, e.status, e.data) for e in evs] == [(e.kind, e.pass_, e.status, e.data) for e in e3]


def test_callback_may_not_call_its_own_watcher(na):
    import ctypes as C
    L = na._lib
    lib = L.load()
    seen = []
    h = C.c_void_p(None)

    def cb(pev, _user):
        info = L.CWatchInfo()
        seen.append((pev.contents.ev.kind, lib.apt_watch_get_info(h, C.byref(info)), lib.apt_watch_reset(h)))
    ccb = L.WATCH_CB(cb)
    from noaa_apt_b200.passes import watch_settings
    ws = watch_settings(search=SEARCH)
    s = na.Settings().to_c()
    assert lib.apt_watch_create(0, 11025, C.byref(s), C.byref(ws), ccb, None, C.byref(h)) == L.OK
    x = recording(11025)[: 100 * 11025]
    q = np.empty(1024, np.float32)
    nq = C.c_uint64(0)
    assert lib.apt_watch_push(h, x.ctypes.data, L.PCM16, x.size, q.ctypes.data, q.size, C.byref(nq)) == L.OK
    lib.apt_watch_destroy(h)
    assert seen and seen[0][0] == L.PASS_AOS and all(r[1:] == (L.ERR_BAD_ARG, L.ERR_BAD_ARG) for r in seen)
