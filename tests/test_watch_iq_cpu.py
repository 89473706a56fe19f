"""The I/Q watcher and the multi-channel FM stage without a GPU (DESIGN.md §14): the exports and their ctypes structs,
apt_watch_iq_geometry against the DESIGN.md formula, every argument error of apt_watch_iq_create / geometry and of
apt_fm_demod_channels before the device is touched, from the ABI and from the Python classes, and the synthetic pass feed's
independence of its generation chunk."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as entry

NEW = ("apt_fm_demod_channels", "apt_watch_iq_geometry", "apt_watch_iq_create", "apt_watch_iq_push_bound",
       "apt_watch_iq_push", "apt_watch_iq_finish", "apt_watch_iq_reset", "apt_watch_iq_get_info", "apt_watch_iq_destroy")
NOAA = [-400_000, 120_000, 412_500]   # NOAA 19, 15 and 18 seen from a 137.5 MHz centre


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def test_abi_exports_the_iq_watcher(na):
    lib = C.CDLL(na.library_path())
    for name in NEW:
        assert hasattr(lib, name) and name in na._lib.SIGNATURES
    assert lib.apt_abi_version() == 1
    L = na._lib
    assert C.sizeof(L.CIqSettings) == 24 and C.sizeof(L.CWatchInfo) == 64
    assert L.WATCH_IQ_MAX_CHANNELS == 8
    assert na.IqWatch is na.passes.IqWatch


def _taps(na, s):
    import oracle
    return oracle.design(oracle.FILTER_LOWPASS, oracle.freq_hz(s.cutout, s.iq_rate), s.atten,
                         oracle.freq_hz(s.delta_freq, s.iq_rate)).size


@pytest.mark.parametrize("iq_rate,max_push,image_out", [(2_400_000, 0, None), (2_400_000, 1_200_000, "png"),
                                                        (250_000, 125_000, "image"), (1_024_000, 4096, None)])
def test_geometry_is_the_design_formula(na, iq_rate, max_push, image_out):
    from noaa_apt_b200.passes import watch_geometry, watch_iq_geometry
    s = na.iq.IqSettings(iq_rate)
    D, N = s.decimation, _taps(na, s)
    mp = max_push or iq_rate
    qpad = -(-(-(-N // D)) // 16) * 16
    proc = dict(contrast=na.image.MINMAX) if image_out else {}
    offsets = [o for o in NOAA if abs(o) + 22000 < iq_rate / 2] or [0]
    offsets = (offsets + [0, -37_000, 51_000, 10_000, -60_000, 20_000, -80_000, 80_000])[:8]
    per = watch_geometry(s.audio_rate, search=dict(max_gap_s=10), image_out=image_out, max_push=mp // D + 1,
                         **proc)["device_bytes"]
    for count in range(1, 9):
        g = watch_iq_geometry(s, offsets[:count], search=dict(max_gap_s=10), image_out=image_out, max_push=max_push, **proc)
        shared = (2 * (N + 2 * D) + mp + 64) * 8 + mp * 8 + D * qpad * 4 + count * 4096 * 2 * 4
        assert g["device_bytes"] == shared + count * per
        assert g["max_push"] == mp
    # linear in the channel count beyond the shared part
    g1, g2, g3 = (watch_iq_geometry(s, offsets[:k], max_push=max_push)["device_bytes"] for k in (1, 2, 3))
    assert g3 - g2 == g2 - g1 > 0


def test_create_and_geometry_argument_errors_before_the_device(na):
    """Every one of these would be APT_ERR_CUDA without a device if it reached one."""
    from noaa_apt_b200 import image
    from noaa_apt_b200.passes import watch_settings
    lib = na._lib.load()
    L = na._lib
    s = na.Settings().to_c()
    qs = na.iq.IqSettings(2_400_000).to_c()
    h = C.c_void_p(None)
    cb = L.WATCH_IQ_CB(lambda c, e, u: None)
    info = L.CWatchInfo()

    def offs(v):
        return (C.c_int32 * max(len(v), 1))(*v)

    def both(ws, offsets=NOAA, count=None, iq=qs, settings=s, out=True):
        count = len(offsets) if count is None else count
        o = offs(offsets) if offsets is not None else None
        args = (C.byref(iq) if iq is not None else None, o, count, C.byref(settings) if settings is not None else None,
                C.byref(ws) if ws is not None else None)
        rc_c = lib.apt_watch_iq_create(0, *args, cb, None, C.byref(h) if out else None)
        rc_g = lib.apt_watch_iq_geometry(*args, C.byref(info))
        return rc_c, rc_g

    ok = watch_settings()
    bad = (L.ERR_BAD_ARG, L.ERR_BAD_ARG)
    assert lib.apt_watch_iq_create(0, C.byref(qs), offs(NOAA), 3, C.byref(s), C.byref(ok), cb, None, None) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_geometry(C.byref(qs), offs(NOAA), 3, C.byref(s), C.byref(ok), None) == L.ERR_BAD_ARG
    assert both(None) == bad
    assert both(ok, settings=None) == bad
    assert both(ok, iq=None) == bad
    assert both(ok, offsets=None, count=3) == bad
    assert both(ok, offsets=[], count=0) == bad
    assert both(ok, offsets=NOAA * 3) == bad                                 # 9 channels
    assert both(ok, offsets=[0] * 9) == bad
    assert both(ok, offsets=NOAA, count=-1) == bad
    assert both(ok, offsets=[0, 1_200_000 - 22_000]) == bad                  # at the band edge
    assert both(ok, offsets=[-(1_200_000 - 22_000)]) == bad
    # the checks of apt_iq_settings
    for field, value in (("audio_rate", 47_000), ("cutout", 0.0), ("cutout", 30_000.0), ("atten", 8.0),
                         ("delta_freq", 300.0)):
        b = na.iq.IqSettings(2_400_000).to_c()
        setattr(b, field, value)
        assert both(ok, iq=b) == bad, field
    # what apt_watch_geometry refuses at audio_rate
    for search in (dict(enter=0.2, exit=0.3), dict(max_gap_s=-1), dict(min_length_s=float("inf"))):
        assert both(watch_settings(search=search)) == bad
    ps, _bpp, _pal = image.process_settings(image.MINMAX)
    bad_ps, _b, _p = image.process_settings(image.MINMAX)
    bad_ps.contrast = 9
    assert both(watch_settings(ps=bad_ps)) == bad
    assert both(watch_settings(png=image.png_settings())) == bad              # PNG without process settings
    assert both(watch_settings(ps=ps, png=image.png_settings(block_bytes=1000))) == bad
    assert both(watch_settings(max_rows=1 << 31)) == bad
    assert both(watch_settings(max_push=(1 << 28) + 1)) == bad
    ws_bad = na.Settings().to_c()
    ws_bad.work_rate = 12000                                                  # not a multiple of 4160
    rc = both(ok, settings=ws_bad)
    assert rc[0] != L.OK and rc[0] != L.ERR_CUDA and rc[1] == rc[0]
    assert h.value is None
    # iq.offset_hz is ignored
    far = na.iq.IqSettings(2_400_000).to_c()
    far.offset_hz = 5_000_000
    assert lib.apt_watch_iq_geometry(C.byref(far), offs(NOAA), 3, C.byref(s), C.byref(ok), C.byref(info)) == L.OK
    if na.device_count() == 0:
        assert both(ok)[0] == L.ERR_CUDA and h.value is None
    nq = (C.c_uint64 * 8)()
    assert lib.apt_watch_iq_push(None, None, L.CU8, 0, None, 0, nq) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_finish(None, None, 0, nq) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_reset(None) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_get_info(None, 0, C.byref(info)) == L.ERR_BAD_ARG
    assert lib.apt_watch_iq_push_bound(None, 0, nq) == L.ERR_BAD_ARG
    lib.apt_watch_iq_destroy(None)


def test_python_classes_refuse_before_the_device(na):
    s = na.iq.IqSettings(2_400_000)
    refused = na.err.InvalidInput   # APT_ERR_BAD_ARG; without a device, reaching it would raise CudaError
    for offsets in ([], NOAA * 3, [1_190_000]):
        with pytest.raises(refused):
            na.IqWatch(s, offsets)
        with pytest.raises(refused):
            na.passes.watch_iq_geometry(s, offsets)
    with pytest.raises(refused):
        na.IqWatch(s, NOAA, search=dict(enter=0.2, exit=0.3))
    with pytest.raises(refused):
        na.IqWatch(s, NOAA, max_push=(1 << 28) + 1)
    x = np.zeros(2 * 1000, np.uint8)
    for offsets in ([], NOAA * 3, [1_190_000]):
        with pytest.raises(refused):
            na.iq.fm_demod_channels(x, s, offsets)


def test_fm_demod_channels_argument_errors_before_the_device(na):
    lib = na._lib.load()
    L = na._lib
    qs = na.iq.IqSettings(2_400_000).to_c()
    x = np.zeros(2 * 5000, np.uint8)
    outs = [np.empty(100, np.float32) for _ in range(9)]
    ptrs = (C.c_void_p * 9)(*[o.ctypes.data for o in outs])
    got = C.c_uint64(0)

    def call(offsets, fmt=L.CU8, cap=100, count=None, iq=qs, p=ptrs, data=x.ctypes.data, n=5000):
        o = (C.c_int32 * max(len(offsets), 1))(*offsets)
        return lib.apt_fm_demod_channels(data, fmt, n, C.byref(iq) if iq is not None else None, o,
                                         len(offsets) if count is None else count, p, cap, C.byref(got))

    assert call(NOAA, iq=None) == L.ERR_BAD_ARG
    assert call(NOAA, p=None) == L.ERR_BAD_ARG
    assert call(NOAA, data=None) == L.ERR_BAD_ARG
    assert call([], count=0) == L.ERR_BAD_ARG
    assert call([0] * 9) == L.ERR_BAD_ARG
    assert call([0, 1_178_000]) == L.ERR_BAD_ARG                             # |offset| + cutout = iq_rate / 2
    assert call(NOAA, fmt=L.F32) == L.ERR_BAD_ARG
    assert call(NOAA, fmt=L.PCM16) == L.ERR_BAD_ARG
    assert call(NOAA, fmt=99) == L.ERR_BAD_ARG
    assert call(NOAA, cap=99) == L.ERR_CAPACITY and got.value == 100           # ceil(5000 / 50)
    assert call(NOAA, n=0, data=None) == L.OK and got.value == 0
    if na.device_count() == 0:
        assert call(NOAA) == L.ERR_CUDA


def test_iq_passes_do_not_depend_on_the_chunk(na):
    from noaa_apt_b200 import synth
    passes = [(-80_000, 5, 0.5, 3.0), (0, 6, 1.5, 4.0), (0, 7, 3.5, 4.5)]
    for fmt in ("cu8", "cs16", "cf32"):
        a = synth.apt_iq_passes(250_000, 5.0, passes, extra_bands=[(80_000, 30_000, 0.5)], fmt=fmt, fade_s=0.5,
                                chunk=1 << 20)
        b = synth.apt_iq_passes(250_000, 5.0, passes, extra_bands=[(80_000, 30_000, 0.5)], fmt=fmt, fade_s=0.5,
                                chunk=99_991)
        assert a.dtype == b.dtype and np.array_equal(a, b)
    truth = synth.apt_iq_passes_truth(250_000, passes, fade_s=0.5)
    assert truth == [(-80_000, 187_500, 687_500), (0, 437_500, 937_500), (0, 937_500, 1_062_500)]
    # a carrier is off outside its passes: before 0.5 s only noise and the band
    x = synth.apt_iq_passes(250_000, 1.0, passes[:1], fmt="cf32", noise_rel=0.0)
    assert np.all(x[:125_000] == 0) and np.any(x[130_000:] != 0)
