"""The I/Q stage on the device (DESIGN.md §10): parity with its CPU restatement, chunk invariance, decode composition and
parity, and an end-to-end check that it demodulates FM."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from _parity import rows_without, sync_ties
from test_iq_cpu import oracle_for

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


def _noise(n, fmt, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(2 * n)
    if fmt == "cu8":
        return np.clip(np.rint(127.5 + 3.0 * v), 0, 255).astype(np.uint8)
    if fmt == "cs16":
        return np.rint(600.0 * v).astype(np.int16)
    return (0.03 * v).astype(np.float32).view(np.complex64)


def _pass(iq_rate, seconds, seed, offset, fmt, noise_s=0.0):
    """noise_s seconds of noise alone, then a synthetic APT pass; both in `fmt`."""
    from noaa_apt_b200 import synth
    x = synth.apt_iq(iq_rate, seconds, seed=seed, offset_hz=offset, fmt=fmt)
    if noise_s:
        x = np.concatenate([_noise(int(iq_rate * noise_s), fmt, seed), x])
    return x


def _with_chunk(chunk, fn):
    old = os.environ.get("APTB200_IQ_CHUNK")
    os.environ["APTB200_IQ_CHUNK"] = str(chunk)
    try:
        return fn()
    finally:
        if old is None:
            del os.environ["APTB200_IQ_CHUNK"]
        else:
            os.environ["APTB200_IQ_CHUNK"] = old


@pytest.mark.parametrize("iq_rate", [2_400_000, 1_200_000, 1_024_000, 250_000])
@pytest.mark.parametrize("fmt", ["cu8", "cs16", "cf32"])
@pytest.mark.parametrize("offset", [0, 37_000, -120_000])
def test_oracle_parity(na, iq_rate, fmt, offset):
    if 2 * (abs(offset) + 22_000) >= iq_rate:
        offset = 0 if offset == 0 else int(np.sign(offset)) * (iq_rate // 2 - 22_000 - 1000)
    s = na.iq.IqSettings(iq_rate, offset_hz=offset)
    noise_s = 0.25
    x = _pass(iq_rate, 2.0, 11, offset, fmt, noise_s)
    got = na.iq.fm_demod(x, s)
    ref = oracle_for(x, fmt, s)
    assert got.shape == ref.shape
    assert np.all(np.isfinite(got))
    assert np.array_equal(got, na.iq.fm_demod(x, s))          # the same bits on every run, noise included
    # the discriminator is ill-conditioned on noise alone: parity starts once the filter has seen only the pass
    first = int(iq_rate * noise_s) // s.decimation + 20
    err = np.max(np.abs(got[first:] - ref[first:])) / np.max(np.abs(ref[first:]))
    assert err <= 1e-5, err


@pytest.mark.parametrize("fmt", ["cu8", "cf32"])
def test_chunk_invariance(na, fmt):
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    D = s.decimation
    x = _pass(1_200_000, 0.25, 5, 37_000, fmt)
    whole = na.iq.fm_demod(x, s)
    for chunk in (7919, D - 1, D + 1, 1):
        if chunk == 1:
            x1 = x[: 2 * 3000] if fmt == "cu8" else x[:3000]
            got = _with_chunk(chunk, lambda: na.iq.fm_demod(x1, s))
            assert np.array_equal(got, whole[: got.size]), chunk
            continue
        got = _with_chunk(chunk, lambda: na.iq.fm_demod(x, s))
        assert np.array_equal(got, whole), chunk


def test_new_formats_rejected_by_audio_entry_points(na):
    lib = na._lib.load()
    x = np.zeros(2 * 200_000, np.uint8)
    s = na.Settings().to_c()
    out = np.empty(na.decode_len_bound(200_000, 48_000), np.float32)
    for fmt in (na._lib.CU8, na._lib.CF32, na._lib.CS16):
        with na.Decoder(48_000, max_samples=200_000) as dec:
            with pytest.raises(na.err.InvalidInput):
                dec.submit_host_ptr(x.ctypes.data, fmt, 200_000, True, out.ctypes.data, out.size)
        with na.Stream(48_000) as st:
            rows = np.empty(1 << 20, np.float32)
            got = C.c_uint64(0)
            assert lib.apt_stream_push(st._h, x.ctypes.data, fmt, 1000, rows.ctypes.data, rows.size, C.byref(got)) == na._lib.ERR_BAD_ARG
        sigs = (C.c_void_p * 1)(x.ctypes.data)
        lens = (C.c_uint64 * 1)(200_000)
        outs = (C.c_void_p * 1)(out.ctypes.data)
        caps = (C.c_uint64 * 1)(out.size)
        nouts = (C.c_uint64 * 1)(0)
        sts = (C.c_int * 1)(0)
        rc = lib.apt_decode_batch(sigs, fmt, lens, 1, 48_000, C.byref(s), 1, outs, caps, nouts, sts, None, 0, 1)
        assert rc == na._lib.ERR_BAD_ARG and sts[0] == na._lib.ERR_BAD_ARG


@pytest.fixture(scope="module")
def pass12(na):
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    x = _pass(1_200_000, 12.0, 21, -120_000, "cu8")
    return s, x


@pytest.mark.parametrize("sync", [True, False])
def test_decode_composition(na, pass12, sync):
    s, x = pass12
    audio = na.iq.fm_demod(x, s)
    want = na.decode(None, None, audio, s.audio_rate, sync=sync)
    got = na.iq.decode_iq(x, s, sync=sync)
    assert got.size > 0 and np.array_equal(got, want)
    # and in chunks, whose boundaries fall inside the pass
    got = _with_chunk(1_000_003, lambda: na.iq.decode_iq(x, s, sync=sync))
    assert np.array_equal(got, want)
    # from pinned memory, without the staging ring
    ptr = C.c_void_p(None)
    lib = na._lib.load()
    assert lib.apt_host_alloc(C.byref(ptr), x.nbytes) == 0
    try:
        pinned = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(x.size,))
        pinned[:] = x
        assert np.array_equal(na.iq.decode_iq(pinned, s, sync=sync), want)
    finally:
        lib.apt_host_free(ptr)


def test_decode_composition_errors(na, pass12):
    s, x = pass12
    short = x[: 2 * 1_200_000 * 4]          # 4 s: fewer than 10 rows
    for fn in (lambda: na.iq.decode_iq(short, s), lambda: na.decode(None, None, na.iq.fm_demod(short, s), s.audio_rate)):
        with pytest.raises(na.err.Internal) as e:
            fn()
        assert e.value.code == na._lib.ERR_TOO_SHORT
    # noise alone: both fail to find five sync frames
    noise = _noise(1_200_000 * 11, "cu8", 3)
    codes = []
    for fn in (lambda: na.iq.decode_iq(noise, s), lambda: na.decode(None, None, na.iq.fm_demod(noise, s), s.audio_rate)):
        try:
            codes.append(fn().size)
        except na.err.Error as e:
            codes.append(("err", e.code))
    assert codes[0] == codes[1]


def test_decode_parity(na, pass12):
    s, x = pass12
    got = na.iq.decode_iq(x, s)
    audio_ref = oracle_for(x, "cu8", s)
    ref, steps = oracle.decode_steps(audio_ref, s.audio_rate)
    audio = na.iq.fm_demod(x, s)
    with na.Decoder(s.audio_rate, max_samples=audio.size) as dec:
        assert np.array_equal(dec.decode(audio, sync=True), got)
        pos = dec.last_sync()
    ties = sync_ties(pos, steps["sync_pos"], steps["filtered"], 12480)
    g, r = rows_without(got, ties), rows_without(ref, ties)
    assert g.shape == r.shape
    err = float(np.max(np.abs(g - r)) / np.max(np.abs(r)))
    assert err <= 1e-5, err


def test_demodulates_fm(na):
    from noaa_apt_b200 import synth
    fs, off = 1_200_000, 37_000
    s = na.iq.IqSettings(fs, offset_hz=off)
    x = synth.apt_iq(fs, 30.0, seed=9, offset_hz=off, fmt="cu8")
    clean = synth.apt_signal(s.audio_rate, 30.0, seed=9)
    got = na.iq.decode_iq(x, s)
    want = na.decode(None, None, clean, s.audio_rate)
    assert got.size == want.size and got.size > 0
    with na.Decoder(s.audio_rate, max_samples=clean.size) as dec:
        dec.decode(na.iq.fm_demod(x, s), sync=True)
        n_iq = dec.last_sync().size
        dec.decode(clean, sync=True)
        n_clean = dec.last_sync().size
    assert n_iq == n_clean
    g, w = got.reshape(-1, 2080), want.reshape(-1, 2080)
    cols = np.r_[86:995, 1126:2035]            # the two image channels
    c = np.corrcoef(g[:, cols].ravel(), w[:, cols].ravel())[0, 1]
    assert c >= 0.98, c


def _schedules(n, D, max_push, seed):
    """Push sizes covering n I/Q samples; the tiny pushes cover a stretch only, so a schedule stays a few thousand calls."""
    rng = np.random.default_rng(seed)
    stretch = 40_000

    def fill(head):
        out, done = list(head), sum(head)
        while done < n:
            k = min(n - done, int(rng.integers(1, 3 * max_push + 1)))
            out.append(k)
            done += k
        return out

    tiny = []
    while sum(tiny) < stretch:
        tiny.append(int(rng.integers(1, 8)))
    around = []
    while sum(around) < stretch:
        around.append([D - 1, D, D + 1][len(around) % 3])
    return {"one": [n], "1_to_7": fill(tiny), "D-1_D_D+1": fill(around), "random": fill([])}


def _stream_rows(na, s, x, sizes, sync, max_push, mix=False):
    rows, info0 = [], None
    with na.Stream.for_iq(s, sync=sync, max_push=max_push) as st:
        info0 = st.info()
        done = 0
        for j, k in enumerate(sizes):
            part = x[2 * done: 2 * (done + k)]
            if mix and j % 2:
                part = (part.astype(np.float32) - np.float32(127.5)).view(np.complex64)   # the same values as cf32
            rows.append(st.push(part))
            assert st.info()["device_bytes"] == info0["device_bytes"]
            done += k
        status = None
        try:
            rows.append(st.finish())
        except na.err.Error as e:
            status = e.code
        info = st.info()
        pos = st.positions()
    assert info["samples_in"] == done == x.size // 2
    return np.concatenate([r.ravel() for r in rows]), pos, status, info0


@pytest.mark.parametrize("sync", [True, False])
def test_stream_bit_identical(na, pass12, sync):
    s, x = pass12
    max_push = 240_000
    want = na.iq.decode_iq(x, s, sync=sync)
    audio = na.iq.fm_demod(x, s)
    with na.Decoder(s.audio_rate, max_samples=audio.size) as dec:
        assert np.array_equal(dec.decode(audio, sync=sync), want)
        want_pos = dec.last_sync() if sync else None
    geo = na.stream_geometry_iq(s, sync=sync, max_push=max_push)
    scheds = _schedules(x.size // 2, s.decimation, max_push, 7)
    for name, sizes in list(scheds.items()) + [("cu8_cf32", scheds["random"])]:
        got, pos, status, info0 = _stream_rows(na, s, x, sizes, sync, max_push, mix=name == "cu8_cf32")
        assert status is None, name
        assert info0["device_bytes"] == geo["device_bytes"] and info0["max_push"] == max_push
        assert np.array_equal(got, want), name
        if sync:
            assert np.array_equal(pos.astype(np.int64), want_pos.astype(np.int64)), name


def test_stream_status_and_formats(na, pass12):
    s, x = pass12
    short = x[: 2 * 1_200_000 * 4]
    _, _, status, _ = _stream_rows(na, s, short, [short.size // 2], True, 240_000)
    assert status == na._lib.ERR_TOO_SHORT
    lib = na._lib.load()
    rows = np.empty(1 << 20, np.float32)
    got = C.c_uint64(0)
    with na.Stream.for_iq(s, max_push=240_000) as st:
        a = np.zeros(1000, np.float32)
        assert lib.apt_stream_push(st._h, a.ctypes.data, na._lib.F32, 1000, rows.ctypes.data, rows.size, C.byref(got)) == na._lib.ERR_BAD_ARG
        assert lib.apt_stream_push(st._h, a.ctypes.data, na._lib.PCM16, 1000, rows.ctypes.data, rows.size, C.byref(got)) == na._lib.ERR_BAD_ARG
