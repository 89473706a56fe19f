"""The I/Q stage without a device: default settings, validation, the WAV reader, and the stage's CPU restatement.

`oracle_fm_demod` restates DESIGN.md §10 in scalar f32 (every numpy operation on float32 arrays rounds once, sums in
ascending k).  The reference has no I/Q path: this stage is the project's own specification, and this function is its
executable form, not a restatement of the reference.  tests/test_gpu_iq.py compares the kernel against it.
"""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B = 4096


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def _load(iq, fmt):
    """(I, Q) as float32 of an interleaved uint8 / int16 / float32 array or a complex64 array."""
    if fmt == "cf32":
        x = np.asarray(iq)
        if x.dtype == np.complex64:
            return x.real.astype(np.float32), x.imag.astype(np.float32)
        return x[0::2].astype(np.float32), x[1::2].astype(np.float32)
    x = np.asarray(iq)
    v = x.astype(np.float32)
    if fmt == "cu8":
        v = v - np.float32(127.5)
    return v[0::2], v[1::2]


def _phasor(v, fs):
    ang = -2.0 * np.pi * v.astype(np.float64) / fs
    return np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)


def oracle_fm_demod(iq, fmt, iq_rate, audio_rate, offset_hz, cutout, delta_freq, atten):
    import oracle
    xr, xi = _load(iq, fmt)
    n = xr.size
    D = iq_rate // audio_rate
    h = oracle.design(oracle.FILTER_LOWPASS, oracle.freq_hz(cutout, iq_rate), atten, oracle.freq_hz(delta_freq, iq_rate))
    f = offset_hz % iq_rate
    if f:
        i = np.arange(n, dtype=np.uint64)
        q, t = i // np.uint64(B), i % np.uint64(B)
        fs = np.uint64(iq_rate)
        Pr, Pi = _phasor(((q * np.uint64(B)) % fs) * np.uint64(f) % fs, iq_rate)
        Wr, Wi = _phasor((t * np.uint64(f)) % fs, iq_rate)
        pr, pi = Pr * Wr - Pi * Wi, Pr * Wi + Pi * Wr
        xr, xi = xr * pr - xi * pi, xr * pi + xi * pr
    M = (n + D - 1) // D
    N = h.size
    sr = np.concatenate([np.zeros(N - 1, np.float32), xr])
    si = np.concatenate([np.zeros(N - 1, np.float32), xi])
    zr = np.zeros(M, np.float32)
    zi = np.zeros(M, np.float32)
    for k in range(N):               # z[m] += h[k] * s[mD - k], ascending k; s[<0] = 0
        a = N - 1 - k
        zr = zr + h[k] * sr[a: a + (M - 1) * D + 1: D]
        zi = zi + h[k] * si[a: a + (M - 1) * D + 1: D]
    out = np.zeros(M, np.float32)
    if M > 1:
        re = zr[1:] * zr[:-1] + zi[1:] * zi[:-1]
        im = zi[1:] * zr[:-1] - zr[1:] * zi[:-1]
        out[1:] = np.arctan2(im, re) * np.float32(audio_rate / (2.0 * np.pi))
    return out


def oracle_for(iq, fmt, s):
    return oracle_fm_demod(iq, fmt, s.iq_rate, s.audio_rate, s.offset_hz, s.cutout, s.delta_freq, s.atten)


# iq_rate -> (audio_rate, D, taps): the table of DESIGN.md §10
TABLE = {2_400_000: (48_000, 50, 671), 1_200_000: (48_000, 25, 337), 1_024_000: (51_200, 20, 287),
         2_048_000: (51_200, 40, 573), 250_000: (50_000, 5, 71)}


@pytest.mark.parametrize("iq_rate", sorted(TABLE))
def test_default_settings(na, iq_rate):
    import oracle
    s = na.iq.IqSettings(iq_rate)
    audio, D, taps = TABLE[iq_rate]
    assert (s.audio_rate, s.decimation) == (audio, D)
    assert (s.cutout, s.delta_freq, s.atten) == (22000.0, 8000.0, 40.0)
    h = oracle.design(oracle.FILTER_LOWPASS, oracle.freq_hz(s.cutout, iq_rate), s.atten, oracle.freq_hz(s.delta_freq, iq_rate))
    assert h.size == taps
    # the library designs the same taps
    f = na._lib.CFilter(na._lib.FILTER_LOWPASS, na._lib.load().apt_freq_hz(s.cutout, iq_rate), s.atten,
                        na._lib.load().apt_freq_hz(s.delta_freq, iq_rate))
    got = np.empty(taps, np.float32)
    n = C.c_size_t(0)
    assert na._lib.load().apt_filter_design(C.byref(f), got.ctypes.data, got.size, C.byref(n)) == 0
    assert n.value == taps and np.array_equal(got, h)
    assert na.iq.fm_demod_len(1000 * D + 1, s) == 1001
    assert na.iq.fm_demod_len(0, s) == 0


def test_default_settings_without_an_audio_rate(na):
    c = na._lib.CIqSettings()
    assert na._lib.load().apt_iq_default_settings(40_000, 0, C.byref(c)) == na._lib.ERR_BAD_ARG
    # a prime rate: D = 1, the audio rate is the I/Q rate
    assert na._lib.load().apt_iq_default_settings(96_001, 0, C.byref(c)) == 0 and c.audio_rate == 96_001


@pytest.mark.parametrize("change", [
    {"audio_rate": 47_000},                      # does not divide iq_rate
    {"cutout": 0.0}, {"delta_freq": -1.0}, {"atten": 8.0},
    {"cutout": 24_000.0},                        # not below audio_rate / 2
    {"offset_hz": 578_000}, {"offset_hz": -578_000},   # |offset| + cutout >= iq_rate / 2
    {"delta_freq": 300.0},                       # more than 8191 taps
])
def test_validation(na, change):
    s = na.iq.IqSettings(1_200_000)
    for k, v in change.items():
        setattr(s, k, v)
    with pytest.raises(na.err.InvalidInput):
        na.iq.fm_demod_len(100, s)
    c = s.to_c()
    out = C.c_uint64(0)
    assert na._lib.load().apt_fm_demod(None, na._lib.CU8, 0, C.byref(c), None, 0, C.byref(out)) == na._lib.ERR_BAD_ARG


def test_validation_edges_that_pass(na):
    s = na.iq.IqSettings(1_200_000, offset_hz=577_999)
    assert na.iq.fm_demod_len(100, s) == 4
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    assert na.iq.fm_demod_len(100, s) == 4


def test_formats_from_dtype(na):
    f = na.iq.iq_format
    assert f(np.zeros(8, np.uint8))[1:] == (na._lib.CU8, 4)
    assert f(np.zeros(8, np.int16))[1:] == (na._lib.CS16, 4)
    assert f(np.zeros(8, np.float32))[1:] == (na._lib.CF32, 4)
    assert f(np.zeros(8, np.complex64))[1:] == (na._lib.CF32, 8)
    with pytest.raises(ValueError):
        f(np.zeros(7, np.uint8))
    with pytest.raises(TypeError):
        f(np.zeros(8, np.float64))
    # an unknown format is refused before any device is touched
    s = na.iq.IqSettings(1_200_000).to_c()
    out = C.c_uint64(0)
    buf = np.zeros(8, np.uint8)
    assert na._lib.load().apt_fm_demod(buf.ctypes.data, na._lib.PCM16, 4, C.byref(s), None, 0, C.byref(out)) == na._lib.ERR_BAD_ARG


def test_decode_iq_errors_before_the_device(na):
    s = na.iq.IqSettings(250_000)
    with pytest.raises(na.err.Internal) as e:
        na.iq.decode_iq(np.full(2 * 250_000, 128, np.uint8), s)       # 1 s of audio: fewer than 10 rows
    assert e.value.code == na._lib.ERR_TOO_SHORT


def test_oracle_tone(na):
    fs, off = 1_200_000, 37_000
    s = na.iq.IqSettings(fs, offset_hz=off)
    n = 120_000
    t = np.arange(n, dtype=np.float64)
    x = np.exp(2j * np.pi * (off + 1000.0) * t / fs).astype(np.complex64)
    a = oracle_for(x, "cf32", s)
    settle = 337 // 25 + 2
    assert np.max(np.abs(a[settle:] - 1000.0)) < 0.05


def test_oracle_frequency_steps(na):
    fs = 1_200_000
    s = na.iq.IqSettings(fs)
    steps = [-15000.0, 4000.0, 12000.0]
    seg = 60_000
    freq = np.repeat(steps, seg)
    ph = np.cumsum(2 * np.pi * freq / fs) - 2 * np.pi * freq / fs
    x = np.exp(1j * ph).astype(np.complex64)
    a = oracle_for(x, "cf32", s)
    D = s.decimation
    for k, f in enumerate(steps):
        lo, hi = (k * seg) // D + 20, ((k + 1) * seg) // D - 1
        assert np.max(np.abs(a[lo:hi] - f)) < 0.05, k


def test_oracle_formats_agree(na):
    rng = np.random.default_rng(3)
    u = rng.integers(0, 256, size=2 * 30_000).astype(np.uint8)
    cs = (u.astype(np.int16) * 2 - 255)                    # 2u - 255 = 2 (u - 127.5): exact in every format
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    a8 = oracle_for(u, "cu8", s)
    a16 = oracle_for(cs.astype(np.int16), "cs16", s)
    af = oracle_for(cs.astype(np.float32), "cf32", s)
    # the cu8 values are half the others: a power-of-two scale is exact through every product, so the audio is identical
    assert np.array_equal(a16, af)
    assert np.array_equal(a8, a16)
    half = (cs.astype(np.float32) / 2).astype(np.float32)
    assert np.array_equal(a8, oracle_for(half, "cf32", s))


def _write_wav(path, data, rate, channels, bits, fmt_tag=1):
    raw = data.tobytes()
    block = channels * bits // 8
    hdr = b"RIFF" + struct.pack("<I", 36 + len(raw)) + b"WAVE"
    hdr += b"fmt " + struct.pack("<IHHIIHH", 16, fmt_tag, channels, rate, rate * block, block, bits)
    hdr += b"data" + struct.pack("<I", len(raw))
    with open(path, "wb") as f:
        f.write(hdr + raw)


def test_wav_load_iq_roundtrip(na, tmp_path):
    iq = np.array([1, -2, 300, -32768, 32767, 0, 5, 6], dtype=np.int16)
    p = tmp_path / "iq.wav"
    _write_wav(p, iq, 2_048_000, 2, 16)
    got, rate = na.wav.load_iq(p)
    assert rate == 2_048_000 and got.dtype == np.int16 and np.array_equal(got, iq)
    mono = tmp_path / "mono.wav"
    _write_wav(mono, iq, 48_000, 1, 16)
    with pytest.raises(na.err.Io):
        na.wav.load_iq(mono)
    fl = tmp_path / "float.wav"
    _write_wav(fl, iq.astype(np.float32), 48_000, 2, 32, fmt_tag=3)
    with pytest.raises(na.err.Io):
        na.wav.load_iq(fl)


def test_synthetic_iq_is_deterministic(na):
    from noaa_apt_b200 import synth
    a = synth.apt_iq(250_000, n_samples=50_000, seed=4, offset_hz=20_000, fmt="cu8")
    b = synth.apt_iq(250_000, n_samples=50_000, seed=4, offset_hz=20_000, fmt="cu8")
    assert a.dtype == np.uint8 and a.size == 100_000 and np.array_equal(a, b)
    # the phase is carried across generation chunks: without noise the chunk size changes nothing but float64 rounding
    a = synth.apt_iq(250_000, n_samples=50_000, seed=4, offset_hz=20_000, fmt="cu8", chunk=1 << 14, noise_rel=0)
    b = synth.apt_iq(250_000, n_samples=50_000, seed=4, offset_hz=20_000, fmt="cu8", noise_rel=0)
    assert np.max(np.abs(a.astype(int) - b.astype(int))) <= 1
    c = synth.apt_iq(250_000, n_samples=1000, seed=4, fmt="cf32")
    assert c.dtype == np.complex64 and c.size == 1000


@pytest.mark.parametrize("iq_rate,max_push", [(1_200_000, 240_000), (2_400_000, 1_200_000), (250_000, 7)])
@pytest.mark.parametrize("sync", [True, False])
def test_stream_geometry_iq(na, iq_rate, max_push, sync):
    s = na.iq.IqSettings(iq_rate)
    g = na.stream_geometry_iq(s, sync=sync, max_push=max_push)
    D = s.decimation
    audio = na.stream_geometry(s.audio_rate, sync=sync, max_push=max_push // D + 1)
    assert g["max_push"] == max_push and g["latency_work"] == audio["latency_work"]
    # the audio stream's buffers, plus the cf32 window, one push's raw samples and the I/Q tables
    extra = g["device_bytes"] - audio["device_bytes"]
    N = TABLE[iq_rate][2]
    qpad = -(-(-(-N // D)) // 16) * 16
    window = 2 * (N + 2 * D) + max_push + 64
    assert extra == window * 8 + max_push * 8 + (D * qpad + 2 * B) * 4


def test_stream_geometry_iq_errors(na):
    s = na.iq.IqSettings(1_200_000)
    for mp in (0, (1 << 28) + 1):
        with pytest.raises(na.err.InvalidInput):
            na.stream_geometry_iq(s, max_push=mp)
    s.audio_rate = 47_000
    with pytest.raises(na.err.InvalidInput):
        na.stream_geometry_iq(s)

