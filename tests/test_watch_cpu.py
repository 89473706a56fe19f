"""Watching a feed without a GPU (DESIGN.md §13): the incremental pass rule (apt_pass_tracker) against
apt_find_passes_quality for every split of q, the earliest windows its AOS / LOS events may fire at, its capacity rule,
apt_watch_geometry on the host, and every argument error of apt_watch_create before the device is touched."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as entry
import _passes_oracle as po

NEW = ("apt_pass_tracker_create", "apt_pass_tracker_feed", "apt_pass_tracker_finish", "apt_pass_tracker_destroy",
       "apt_watch_create", "apt_watch_geometry", "apt_watch_push_bound", "apt_watch_push", "apt_watch_finish",
       "apt_watch_reset", "apt_watch_get_info", "apt_watch_destroy")


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def test_abi_exports_the_watcher(na):
    lib = C.CDLL(na.library_path())
    for name in NEW:
        assert hasattr(lib, name) and name in na._lib.SIGNATURES
    assert lib.apt_abi_version() == 1
    L = na._lib
    assert C.sizeof(L.CPassEvent) == 56 and C.sizeof(L.CWatchInfo) == 64
    assert C.sizeof(L.CWatchSettings) == 4 + 16 + 4 + 8 + 8 + 8 + 8


def _crafted():
    """(q, rule keywords) covering passes at both ends, gaps of max_gap - 1 and max_gap, lengths of min_length - 1 and
    min_length, q equal to enter and exit, max_gap 0, W = 0 and a one-window pass."""
    W = 1000
    cases = []
    q = np.zeros(W, np.float32)
    q[:200] = 0.9
    q[850:] = 0.8
    cases.append((q, {}))
    q = np.zeros(W, np.float32)
    q[100:200] = 0.5
    q[259:400] = 0.5
    q[460:600] = 0.5
    q[230] = 0.1                               # a gap window that is summed into the mean
    cases.append((q, {}))
    q = np.zeros(W, np.float32)
    q[10:130] = 0.6
    q[300:419] = 0.6
    cases.append((q, {}))
    q = np.zeros(W, np.float32)
    q[50:250] = np.float32(0.15)
    q[120] = np.float32(0.30)
    cases.append((q, {}))
    q = np.zeros(W, np.float32)
    q[50:250] = np.float32(0.15)
    q[247] = np.float32(0.30)                  # enter reached after first + min_length - 1
    cases.append((q, {}))
    q = np.zeros(300, np.float32)
    q[[3, 4, 7, 100, 101, 102, 299]] = [0.9, 0.2, 0.5, 0.16, 0.31, 0.4, 0.9]
    cases.append((q, dict(max_gap_s=0.0001, min_length_s=0.0001)))          # max_gap 0 windows, 1-window passes
    cases.append((q, dict(max_gap_s=0.5, min_length_s=0.5)))                # max_gap 1, min_length 1
    cases.append((np.zeros(0, np.float32), {}))                             # W = 0
    rng = np.random.default_rng(11)
    for _ in range(12):
        q = (rng.random(1500) ** 3).astype(np.float32)
        q[rng.integers(0, 1500, 40)] = -0.5
        kw = dict(enter=float(rng.uniform(0.3, 0.9)), exit=float(rng.uniform(0.05, 0.3)),
                  max_gap_s=float(rng.choice([0.0001, 0.5, 1.0, 3.0, 20.0])), min_length_s=float(rng.uniform(0.1, 30)))
        kw["enter"] = max(kw["enter"], kw["exit"])
        cases.append((q, kw))
    return cases


def _splits(n, rng):
    yield [n]
    yield [1] * n
    cuts = sorted(set(rng.integers(0, n + 1, size=min(n, 12)).tolist()) | {0, n}) if n else [0]
    yield [b - a for a, b in zip(cuts, cuts[1:])]


def _expected_events(q, kw):
    """The earliest windows the rule allows, from the offline passes: AOS at the first window with q >= exit at or after
    max(the first window reaching enter, first + min_length - 1); LOS at last + max_gap, or at finish."""
    enter, exit_ = np.float32(kw.get("enter", po.ENTER)), np.float32(kw.get("exit", po.EXIT))
    max_gap = po.windows_of(kw.get("max_gap_s", po.MAX_GAP_S))
    min_length = po.windows_of(kw.get("min_length_s", po.MIN_LENGTH_S))
    out = []
    for p in po.find_passes(q, 10 ** 15, 11025, **kw):
        a, b = p["first_window"], p["first_window"] + p["windows"] - 1
        seg = q[a:b + 1]
        e = a + int(np.nonzero(seg >= enter)[0][0])
        t = max(e, a + max(min_length, 1) - 1)
        aos = t + int(np.nonzero(q[t:b + 1] >= exit_)[0][0])
        los = b + max_gap if b + max_gap < q.size else None
        out.append((a, aos, los))
    return out


def test_tracker_equals_the_offline_rule_for_every_split(na):
    rng = np.random.default_rng(3)
    for q, kw in _crafted():
        n = (q.size + 2) * 11025 // 2 + 17
        want = po.find_passes(q, n, 11025, **kw)
        assert [p.__dict__ for p in na.find_passes_quality(q, n, 11025, **kw)] == want
        expect = _expected_events(q, kw)
        for split in _splits(q.size, rng):
            t = na.PassTracker(11025, **kw)
            evs, at = [], 0
            for k in split:
                evs += t.feed(q[at:at + k])
                at += k
            fin = t.finish(n)
            evs += fin
            los = [e for e in evs if e.kind == "los"]
            aos = [e for e in evs if e.kind == "aos"]
            assert [e.pass_.__dict__ for e in los] == want, (kw, split[:5])
            assert len(aos) == len(los)
            for (a, aos_w, los_w), ea, el in zip(expect, aos, los):
                assert ea.pass_.start == el.pass_.start == a * 11025 // 2 and ea.pass_.end == 0
                assert ea.window == aos_w and ea.pass_.first_window == a and ea.pass_.windows == aos_w - a + 1
                assert el.window == (los_w if los_w is not None else q.size)
                assert (los_w is None) == (el in fin)
            # every AOS comes before its own LOS
            kinds = [e.kind for e in evs]
            assert kinds == ["aos", "los"] * len(los)
            # after finish the tracker starts over
            assert [e.pass_.__dict__ for e in t.feed(q) + t.finish(n) if e.kind == "los"] == want


def test_tracker_capacity_leaves_the_state_unchanged(na):
    lib = na._lib.load()
    L = na._lib
    q = np.zeros(400, np.float32)
    q[10:380] = 0.9                         # still open at window 399: its LOS comes at finish
    h = C.c_void_p(None)
    ps = L.CPassSearch(0, 0, 0, 0)
    assert lib.apt_pass_tracker_create(11025, C.byref(ps), C.byref(h)) == L.OK
    evs = (L.CPassEvent * 800)()
    nev = C.c_uint64(7)
    assert lib.apt_pass_tracker_feed(h, q.ctypes.data, q.size, evs, 2 * q.size - 1, C.byref(nev)) == L.ERR_CAPACITY
    assert nev.value == 0
    assert lib.apt_pass_tracker_feed(h, q.ctypes.data, q.size, evs, 2 * q.size, C.byref(nev)) == L.OK
    assert [evs[i].kind for i in range(nev.value)] == [L.PASS_AOS]
    assert lib.apt_pass_tracker_finish(h, 10 ** 9, evs, 0, C.byref(nev)) == L.ERR_CAPACITY
    assert lib.apt_pass_tracker_finish(h, 10 ** 9, evs, 1, C.byref(nev)) == L.OK
    assert nev.value == 1 and evs[0].kind == L.PASS_LOS and evs[0].pass_.first_window == 10 and evs[0].pass_.windows == 370
    assert evs[0].window == 400
    lib.apt_pass_tracker_destroy(h)
    lib.apt_pass_tracker_destroy(None)
    for bad in (L.CPassSearch(0.2, 0.3, 0, 0), L.CPassSearch(0, 0, -1, 0), L.CPassSearch(float("nan"), 0, 0, 0)):
        assert lib.apt_pass_tracker_create(11025, C.byref(bad), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_pass_tracker_create(0, C.byref(ps), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_pass_tracker_create(11025, C.byref(ps), None) == L.ERR_BAD_ARG
    assert lib.apt_pass_tracker_feed(None, q.ctypes.data, 1, evs, 2, C.byref(nev)) == L.ERR_BAD_ARG


def test_geometry_needs_no_device_and_grows_with_the_settings(na):
    from noaa_apt_b200 import image
    from noaa_apt_b200.passes import watch_geometry
    base = watch_geometry(48000)
    assert base["device_bytes"] > 0 and base["max_push"] == 48000 and base["latency_windows"] >= 2
    assert watch_geometry(48000, search=dict(max_gap_s=60))["device_bytes"] > base["device_bytes"]
    img = watch_geometry(48000, image_out="image", contrast=image.MINMAX)
    assert img["device_bytes"] > base["device_bytes"]
    assert watch_geometry(48000, image_out="image", max_rows=4000)["device_bytes"] > img["device_bytes"]
    png = watch_geometry(48000, image_out="png")
    assert png["device_bytes"] > img["device_bytes"]
    assert watch_geometry(48000, image_out="png", max_rows=4000)["device_bytes"] > png["device_bytes"]
    assert watch_geometry(11025, max_push=4096)["max_push"] == 4096


def test_create_argument_errors_before_the_device(na):
    """Every one of these would be APT_ERR_CUDA without a device if it reached one."""
    from noaa_apt_b200 import image
    from noaa_apt_b200.passes import watch_settings
    lib = na._lib.load()
    L = na._lib
    s = na.Settings().to_c()
    h = C.c_void_p(None)
    cb = L.WATCH_CB(lambda e, u: None)

    def create(ws, rate=48000, settings=s, out=True):
        return lib.apt_watch_create(0, rate, C.byref(settings) if settings is not None else None,
                                    C.byref(ws) if ws is not None else None, cb, None, C.byref(h) if out else None)

    ok = watch_settings()
    assert create(ok, out=False) == L.ERR_BAD_ARG
    assert create(None) == L.ERR_BAD_ARG
    assert create(ok, settings=None) == L.ERR_BAD_ARG
    for search in (dict(enter=0.2, exit=0.3), dict(max_gap_s=-1), dict(min_length_s=float("inf"))):
        assert create(watch_settings(search=search)) == L.ERR_BAD_ARG
    ps, _bpp, _pal = image.process_settings(image.MINMAX)
    bad_ps, _b, _p = image.process_settings(image.MINMAX)
    bad_ps.contrast = 9
    assert create(watch_settings(ps=bad_ps)) == L.ERR_BAD_ARG
    png = image.png_settings()
    assert create(watch_settings(png=png)) == L.ERR_BAD_ARG                 # PNG without process settings
    bad_png = image.png_settings(block_bytes=1000)
    assert create(watch_settings(ps=ps, png=bad_png)) == L.ERR_BAD_ARG
    assert create(watch_settings(ps=ps, png=image.png_settings(rgb_from_rgba=True))) == L.ERR_BAD_ARG   # grey output
    assert create(watch_settings(max_rows=1 << 31)) == L.ERR_BAD_ARG
    assert create(watch_settings(max_push=(1 << 28) + 1)) == L.ERR_BAD_ARG
    bad = na.Settings().to_c()
    bad.work_rate = 12000                                                   # not a multiple of 4160
    assert create(ok, settings=bad) != L.OK
    assert create(ok, rate=0) != L.OK
    assert h.value is None
    for rc in (create(ok), create(watch_settings(ps=ps, png=png, sync=False))):
        assert rc in (L.OK, L.ERR_CUDA)
        if rc == L.OK:   # a machine with a device
            lib.apt_watch_destroy(h)
            h.value = None
    if na.device_count() == 0:
        assert create(ok) == L.ERR_CUDA
    nq = C.c_uint64(0)
    info = L.CWatchInfo()
    assert lib.apt_watch_push(None, None, L.F32, 0, None, 0, C.byref(nq)) == L.ERR_BAD_ARG
    assert lib.apt_watch_finish(None, None, 0, C.byref(nq)) == L.ERR_BAD_ARG
    assert lib.apt_watch_reset(None) == L.ERR_BAD_ARG
    assert lib.apt_watch_get_info(None, C.byref(info)) == L.ERR_BAD_ARG
    assert lib.apt_watch_push_bound(None, 0, C.byref(nq)) == L.ERR_BAD_ARG
    assert lib.apt_watch_geometry(48000, C.byref(s), None, C.byref(info)) == L.ERR_BAD_ARG
    lib.apt_watch_destroy(None)


def test_a_huge_max_gap_allocates_nothing_up_front(na):
    """The rule holds only the q of the current gap, so any max_gap_s the search accepts works without reserving memory;
    a watcher, whose input window holds max_gap windows of samples, refuses one that cannot fit before the device."""
    q = np.zeros(3000, np.float32)
    q[100:400] = 0.9
    q[2500:2900] = 0.8
    for gap in (1e9, 1e17):
        want = po.find_passes(q, 10 ** 7, 11025, max_gap_s=gap)
        assert [p.__dict__ for p in na.find_passes_quality(q, 10 ** 7, 11025, max_gap_s=gap)] == want
        assert len(want) == 1 and want[0]["windows"] == 2800
        t = na.PassTracker(11025, max_gap_s=gap)
        evs = t.feed(q) + t.finish(10 ** 7)
        assert [e.pass_.__dict__ for e in evs if e.kind == "los"] == want
    from noaa_apt_b200.passes import watch_geometry
    L = na._lib
    with pytest.raises(na.err.Error) as e:
        watch_geometry(48000, search=dict(max_gap_s=1e9))
    assert e.value.code == L.ERR_BAD_ARG
    assert watch_geometry(48000, search=dict(max_gap_s=3600))["device_bytes"] < 2 ** 31
