"""Finding passes without a GPU (DESIGN.md §12): the new entry points are exported, apt_find_passes_quality equals the
numpy rule on crafted quality arrays, the float64 restatement of q rises through `exit` where the real pass begins,
every argument error comes back before any device is touched, and the receiver-noise fixture is intact."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import __graft_entry__ as entry
import _passes_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
NEW = ("apt_recording_create", "apt_recording_destroy", "apt_recording_get_info", "apt_recording_quality",
       "apt_find_passes_quality", "apt_recording_decode")


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def test_abi_exports_the_pass_search(na):
    lib = C.CDLL(na.library_path())
    for name in NEW:
        assert hasattr(lib, name) and name in na._lib.SIGNATURES
    assert lib.apt_abi_version() == 1
    L = na._lib
    assert C.sizeof(L.CPassSearch) == 16 and C.sizeof(L.CPass) == 40 and C.sizeof(L.CRecordingInfo) == 40


def _lib_passes(na, q, n, rate, **kw):
    return [p.__dict__ for p in na.find_passes_quality(q, n, rate, **kw)]


def _check(na, q, n=None, rate=11025, **kw):
    q = np.asarray(q, dtype=np.float32)
    n = (q.size + 2) * rate // 2 + 17 if n is None else n
    want = po.find_passes(q, n, rate, **kw)
    got = _lib_passes(na, q, n, rate, **kw)
    assert got == want
    return got


def test_rule_on_crafted_quality(na):
    W = 1000
    # a pass touching window 0 and one touching window W - 1
    q = np.zeros(W, np.float32)
    q[:200] = 0.9
    q[850:] = 0.8
    got = _check(na, q)
    assert [(p["first_window"], p["windows"]) for p in got] == [(0, 200), (850, 150)]
    assert got[-1]["end"] == min((W + 1) * 11025 // 2 + 17, -(-(W - 1 + 2) * 11025 // 2))

    # gaps of exactly max_gap - 1 windows (joined) and exactly max_gap windows (split): default max_gap 60
    q = np.zeros(W, np.float32)
    q[100:200] = 0.5
    q[259:400] = 0.5          # 59 windows between 199 and 259
    q[460:600] = 0.5          # 60 windows between 399 and 460
    got = _check(na, q)
    assert [(p["first_window"], p["windows"]) for p in got] == [(100, 300), (460, 140)]

    # groups exactly min_length (kept) and min_length - 1 (dropped) long: default min_length 120
    q = np.zeros(W, np.float32)
    q[10:130] = 0.6
    q[300:419] = 0.6
    got = _check(na, q)
    assert [(p["first_window"], p["windows"]) for p in got] == [(10, 120)]

    # q equal to enter and to exit: both comparisons are >=
    q = np.zeros(W, np.float32)
    q[50:250] = np.float32(0.15)
    q[120] = np.float32(0.30)
    got = _check(na, q)
    assert [(p["first_window"], p["windows"]) for p in got] == [(50, 200)]
    q[120] = np.nextafter(np.float32(0.30), np.float32(0))
    assert _check(na, q) == []                                # a group with no window reaching enter
    q[50:250] = np.nextafter(np.float32(0.15), np.float32(0))
    q[120] = 0.9
    assert _check(na, q) == []                                # only one window reaches exit

    # W = 0, and a recording whose last pass is cut at n
    assert _check(na, np.zeros(0, np.float32), n=1000) == []
    q = np.full(300, 0.7, np.float32)
    got = _check(na, q, n=300 * 11025 // 2 + 3)
    assert got[0]["end"] == 300 * 11025 // 2 + 3


def test_rule_with_settings_and_noise(na):
    rng = np.random.default_rng(5)
    for trial in range(30):
        q = (rng.random(3000) ** 3).astype(np.float32)
        q[rng.integers(0, 3000, 40)] = -0.5
        kw = dict(enter=float(rng.uniform(0.3, 0.9)), exit=float(rng.uniform(0.05, 0.3)),
                  max_gap_s=float(rng.uniform(0.5, 40)), min_length_s=float(rng.uniform(0.5, 30)))
        kw["enter"] = max(kw["enter"], kw["exit"])
        rate = int(rng.choice([11025, 48000, 96000]))
        _check(na, q, rate=rate, **kw)


def test_capacity_and_counting(na):
    lib = na._lib.load()
    L = na._lib
    q = np.zeros(2000, np.float32)
    for k in range(5):
        q[k * 400:k * 400 + 200] = 0.9
    cnt = C.c_uint32(0)
    ps = L.CPassSearch(0, 0, 0, 0)
    assert lib.apt_find_passes_quality(q.ctypes.data, q.size, 10 ** 9, 48000, C.byref(ps), None, 0, C.byref(cnt)) == L.ERR_CAPACITY
    assert cnt.value == 5
    out = (L.CPass * 3)()
    assert lib.apt_find_passes_quality(q.ctypes.data, q.size, 10 ** 9, 48000, C.byref(ps), out, 3, C.byref(cnt)) == L.ERR_CAPACITY
    assert cnt.value == 5 and [out[i].first_window for i in range(3)] == [0, 400, 800]
    out = (L.CPass * 5)()
    assert lib.apt_find_passes_quality(q.ctypes.data, q.size, 10 ** 9, 48000, None, out, 5, C.byref(cnt)) == L.OK
    assert cnt.value == 5 and out[4].start == 1600 * 48000 // 2 and out[4].end == (1799 + 2) * 48000 // 2


def test_restated_quality_rises_through_exit_at_the_real_aos(na):
    """The first 40 s of the reference's real pass (AOS included): q stays below exit over the first 8 windows and reaches
    it at window 8, where the whole-file estimate puts the pass's start, and the rule sees one group from there to the
    end of the excerpt that reaches enter."""
    import oracle
    g = np.load(os.path.join(HERE, "golden", "test_11025hz_excerpts.npz"))
    x = oracle.pcm16_to_f32(g["pcm_start"])
    _, st = oracle.decode_steps(x, 11025)
    q = po.quality(st["demodulated"], 6240)
    assert q.size == len(st["demodulated"]) // 6240 - 1 == 78
    assert np.all(q[:8] < po.EXIT) and q[8] >= po.EXIT
    assert q.max() >= po.ENTER
    got = _check(na, q.astype(np.float32), n=x.size, min_length_s=30)
    assert [(p["first_window"], p["windows"]) for p in got] == [(8, 70)]
    assert got[0]["start"] == 8 * 11025 // 2
    assert _check(na, q.astype(np.float32), n=x.size) == []    # 35 s: shorter than the default 60 s


def test_argument_errors_before_the_device(na):
    """Every one of these would be APT_ERR_CUDA without a device if it reached one."""
    lib = na._lib.load()
    L = na._lib
    s = na.Settings().to_c()
    x = np.zeros(48000 * 20, np.float32)
    h = C.c_void_p(None)
    assert lib.apt_recording_create(0, None, L.F32, x.size, 48000, C.byref(s), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_recording_create(0, x.ctypes.data, L.F32, 0, 48000, C.byref(s), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_recording_create(0, x.ctypes.data, L.CU8, x.size, 48000, C.byref(s), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_recording_create(0, x.ctypes.data, 9, x.size, 48000, C.byref(s), C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_recording_create(0, x.ctypes.data, L.F32, x.size, 48000, None, C.byref(h)) == L.ERR_BAD_ARG
    assert lib.apt_recording_create(0, x.ctypes.data, L.F32, x.size, 48000, C.byref(s), None) == L.ERR_BAD_ARG
    bad = na.Settings().to_c()
    bad.work_rate = 12000                                                  # not a multiple of 4160
    assert lib.apt_recording_create(0, x.ctypes.data, L.F32, x.size, 48000, C.byref(bad), C.byref(h)) == L.ERR_WORK_RATE
    assert lib.apt_recording_create(0, x.ctypes.data, L.F32, x.size, 0, C.byref(s), C.byref(h)) != L.OK
    assert h.value is None
    nq = C.c_uint64(0)
    assert lib.apt_recording_quality(None, None, 0, C.byref(nq)) == L.ERR_BAD_ARG
    info = L.CRecordingInfo()
    assert lib.apt_recording_get_info(None, C.byref(info)) == L.ERR_BAD_ARG
    lib.apt_recording_destroy(None)

    q = np.zeros(10, np.float32)
    cnt = C.c_uint32(0)
    out = (L.CPass * 4)()
    for enter, exit_, gap, length in ((0.2, 0.3, 0, 0), (0, -0.1, 0, 0), (1.5, 0, 0, 0), (0, 0, -1, 0), (0, 0, 0, -1),
                                      (float("nan"), 0, 0, 0), (0, 0, float("inf"), 0), (0.1, 0, 0, 0)):
        ps = L.CPassSearch(enter, exit_, gap, length)
        assert lib.apt_find_passes_quality(q.ctypes.data, q.size, 1000, 11025, C.byref(ps), out, 4, C.byref(cnt)) == L.ERR_BAD_ARG
    ps = L.CPassSearch(0, 0, 0, 0)
    assert lib.apt_find_passes_quality(None, 10, 1000, 11025, C.byref(ps), out, 4, C.byref(cnt)) == L.ERR_BAD_ARG
    assert lib.apt_find_passes_quality(q.ctypes.data, 10, 1000, 11025, C.byref(ps), None, 4, C.byref(cnt)) == L.ERR_BAD_ARG
    assert lib.apt_find_passes_quality(q.ctypes.data, 10, 1000, 11025, C.byref(ps), out, 4, None) == L.ERR_BAD_ARG
    assert lib.apt_find_passes_quality(q.ctypes.data, 10, 1000, 0, C.byref(ps), out, 4, C.byref(cnt)) == L.ERR_BAD_ARG

    # decode: a NULL recording or NULL arrays, before anything else
    rng = (L.CPass * 1)()
    outs = (C.c_void_p * 1)(q.ctypes.data)
    caps = (C.c_uint64 * 1)(10)
    nouts = (C.c_uint64 * 1)()
    sts = (C.c_int * 1)()
    assert lib.apt_recording_decode(None, rng, 1, 1, None, None, outs, caps, nouts, None, sts) == L.ERR_BAD_ARG
    with pytest.raises(na.err.Error):
        na.Recording(np.zeros(0, np.float32), 48000)
    with pytest.raises(TypeError):
        na.Recording(np.zeros(10, np.float64), 48000)


def test_noise_fixture_is_intact():
    g = np.load(os.path.join(HERE, "golden", "noise_11025hz.npz"))
    pcm = g["pcm"]
    assert pcm.dtype == np.int16 and pcm.size == 330745 and int(g["rate"]) == 11025
    assert str(g["sha256"]) == "b817339df8bc9ef53c8839b85ebe3b45aab48f0e9c1aa2528d7f3e3b47bf68ec"
    assert hashlib.sha256(pcm.tobytes()).hexdigest() == str(g["pcm_sha256"])


def test_synthetic_passes_are_chunk_invariant(na):
    from noaa_apt_b200 import synth
    layout = [("noise", 7), ("pass", 30, 3), ("silence", 4), ("pass", 25, 4), ("noise", 3)]
    x = synth.apt_passes(11025, layout, seed=2)
    assert x.size == synth.apt_passes_len(11025, layout) == 69 * 11025
    parts = [synth.apt_passes(11025, layout, seed=2, start=a, n_samples=min(65_537, x.size - a))
             for a in range(0, x.size, 65_537)]
    assert np.array_equal(np.concatenate(parts), x)
    a, b = 37 * 11025, 41 * 11025
    assert not x[a:b].any()                                            # silence is exact zeros
    assert synth.apt_passes_truth(11025, layout) == [(7 * 11025 + 5 * 11025, 37 * 11025 - 5 * 11025),
                                                     (41 * 11025 + 5 * 11025, 66 * 11025 - 5 * 11025)]
