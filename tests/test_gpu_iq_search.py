"""Finding carriers on the device (DESIGN.md §10, "Finding carriers"): the spectrum against numpy, carrier accuracy with
and without Doppler, rejections, several channels decoded from one upload equal to one apt_decode_iq each, and the
whole search-and-decode on a recording with three carriers at unknown offsets."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


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


def _load(x, fmt):
    if fmt == "cu8":
        v = x.astype(np.float32) - np.float32(127.5)
        return (v[0::2] + 1j * v[1::2]).astype(np.complex128)
    if fmt == "cs16":
        v = x.astype(np.float64)
        return v[0::2] + 1j * v[1::2]
    return x.astype(np.complex128)


def _ref_spectrum(x, fmt, nfft, max_segments):
    z = _load(x, fmt)
    S = z.size // nfft
    K = min(S, max_segments)
    t = np.arange(nfft)
    w = (0.5 - 0.5 * np.cos(2 * np.pi * t / nfft)).astype(np.float32).astype(np.float64)
    acc = np.zeros(nfft)
    for k in range(K):
        a = (k * S // K) * nfft
        acc += np.abs(np.fft.fft(z[a:a + nfft] * w)) ** 2
    return np.fft.fftshift(acc / K), K


def _signal(n, fmt, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    z = 0.6 * np.exp(2j * np.pi * 0.1234567 * t) + 0.05 * np.exp(-2j * np.pi * 0.31 * t) \
        + 0.02 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "cf32":
        return z.astype(np.complex64)
    scale = 100.0 if fmt == "cu8" else 20000.0
    inter = np.empty(2 * n)
    inter[0::2], inter[1::2] = z.real * scale, z.imag * scale
    if fmt == "cu8":
        return np.clip(np.rint(inter + 127.5), 0, 255).astype(np.uint8)
    return np.rint(inter).astype(np.int16)


@pytest.mark.parametrize("fmt", ["cu8", "cs16", "cf32"])
@pytest.mark.parametrize("nfft", [256, 4096, 16384])
@pytest.mark.parametrize("segs", ["below", "at"])
def test_spectrum_against_numpy(na, fmt, nfft, segs):
    S = 37
    max_segments = 2048 if segs == "below" else 11       # K = S = 37 < 2048, or K = 11 spread over 37
    n = S * nfft + nfft // 3
    x = _signal(n, fmt, nfft + len(fmt))
    freqs, got = na.iq.spectrum(x, 1_000_000, nfft=nfft, max_segments=max_segments)
    ref, K = _ref_spectrum(x, fmt, nfft, max_segments)
    assert freqs[nfft // 2] == 0.0 and freqs[0] == -500_000.0
    m = ref.max()
    assert np.max(np.abs(got - ref)) <= 2e-5 * m
    big = ref > m / 1e4
    assert np.max(np.abs(got[big] - ref[big]) / ref[big]) <= 1e-3
    again = na.iq.spectrum(x, 1_000_000, nfft=nfft, max_segments=max_segments)[1]
    assert np.array_equal(again.view(np.uint32), got.view(np.uint32))
    for chunk in (1, 3 * nfft + 5, 10 * nfft):
        c = _with_chunk(chunk, lambda: na.iq.spectrum(x, 1_000_000, nfft=nfft, max_segments=max_segments)[1])
        assert np.array_equal(c.view(np.uint32), got.view(np.uint32)), chunk


def _true_mean(offset, doppler, tca, width, seconds):
    t = np.linspace(0, seconds, 10001)
    return offset + np.mean(-doppler * (t - tca) / np.sqrt((t - tca) ** 2 + width ** 2))


@pytest.mark.parametrize("fs", [1_200_000, 2_400_000])
@pytest.mark.parametrize("where", ["+37000", "-120000", "+251313", "edge"])
@pytest.mark.parametrize("doppler", [0.0, 3000.0])
def test_carrier_accuracy(na, fs, where, doppler):
    from noaa_apt_b200 import synth
    offset = fs // 2 - 22_000 - 25_000 if where == "edge" else int(where)
    seconds, tca, width = 6.0, 2.5, 1.0
    x = synth.apt_iq_multi(fs, seconds, carriers=[(offset, 4, doppler, tca, width)], fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(x, fs)
    apt = [c for c in found if c.is_apt]
    assert len(apt) == 1, found
    err = apt[0].centre_hz - _true_mean(offset, doppler, tca, width, seconds)
    print(f"carrier error fs={fs} offset={where} doppler={doppler}: {err:+.1f} Hz, snr {apt[0].snr_db:.1f} dB, "
          f"apt_score {apt[0].apt_score:.3f}; all scores {[round(c.apt_score, 3) for c in found]}")
    assert abs(err) <= 300.0


def test_rejections(na):
    from noaa_apt_b200 import synth
    fs = 2_400_000
    noise = synth.apt_iq_multi(fs, 5.0, carriers=[], fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(noise, fs)
    print("pure noise:", [(c.offset_hz, round(c.snr_db, 1), round(c.apt_score, 3)) for c in found])
    assert not any(c.is_apt for c in found)
    band = synth.apt_iq_multi(fs, 5.0, carriers=[], extra_bands=[(200_000, 120_000, 1.0)], fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(band, fs)
    print("120 kHz band:", [(c.offset_hz, round(c.snr_db, 1), round(c.apt_score, 3)) for c in found])
    assert any(abs(c.centre_hz - 200_000) < 60_000 for c in found)
    assert not any(c.is_apt for c in found)
    two = synth.apt_iq_multi(fs, 6.0, carriers=[(-100_000, 1, 0.0, None, 20.0), (190_000, 2, 0.0, None, 20.0)],
                             fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(two, fs)
    print("two carriers:", [(c.offset_hz, round(c.snr_db, 1), round(c.apt_score, 3)) for c in found])
    apt = sorted(c.offset_hz for c in found if c.is_apt)
    assert len(apt) == 2 and abs(apt[0] + 100_000) < 300 and abs(apt[1] - 190_000) < 300


@pytest.fixture(scope="module")
def three(na):
    from noaa_apt_b200 import synth
    fs = 1_200_000
    s = na.iq.IqSettings(fs)
    x = synth.apt_iq_multi(fs, 12.0, carriers=[(37_000, 21, 0.0, None, 20.0), (-180_000, 22, 0.0, None, 20.0)],
                           fmt="cu8", noise_rel=0.03)
    return s, x


@pytest.mark.parametrize("chunk", [None, 1_000_003])
def test_decode_channels_equal_decode_iq(na, three, chunk):
    s, x = three
    offsets = [37_000, -180_000, 300_000]          # the third holds noise only
    run = (lambda f: f()) if chunk is None else (lambda f: _with_chunk(chunk, f))
    rows, sts = run(lambda: na.iq.decode_iq_channels(x, s, offsets))
    for c, off in enumerate(offsets):
        so = na.iq.IqSettings(s.iq_rate, offset_hz=off)
        try:
            want, wst = run(lambda: na.iq.decode_iq(x, so)), na._lib.OK
        except na.err.Error as e:
            want, wst = np.empty(0, np.float32), e.code
        assert sts[c] == wst, (c, sts)
        assert np.array_equal(rows[c], want), c
        if wst == na._lib.OK:
            audio = na.iq.fm_demod(x, so)
            with na.Decoder(s.audio_rate, max_samples=audio.size) as dec:
                assert np.array_equal(dec.decode(audio, sync=True), rows[c])
                assert dec.last_sync().size >= 5      # the sync positions behind these rows
    # the noise-only channel gets whatever apt_decode_iq gives it (the peak picker finds a row sync in noise too)
    print(f"channel statuses (chunk {chunk}): {sts}")
    assert sts[0] == na._lib.OK and sts[1] == na._lib.OK
    # a channel that fails keeps its own status and the others still decode
    import ctypes as C
    lib = na._lib.load()
    L = na._lib
    xs, fmt, n = na.iq.iq_format(x)
    qs, st = s.to_c(), na.Settings().to_c()
    bufs = [np.empty(max(r.size, 1) + 2080, np.float32) for r in rows]
    bufs[1] = np.empty(16, np.float32)                 # too small for channel 1
    k = len(offsets)
    outs = (C.c_void_p * k)(*[b.ctypes.data for b in bufs])
    caps = (C.c_uint64 * k)(*[b.size for b in bufs])
    nouts, stc = (C.c_uint64 * k)(), (C.c_int * k)()
    rc = run(lambda: lib.apt_decode_iq_channels(xs.ctypes.data, fmt, n, C.byref(qs), (C.c_int32 * k)(*offsets), k,
                                                C.byref(st), 1, outs, caps, nouts, stc))
    assert rc == L.ERR_CAPACITY and stc[1] == L.ERR_CAPACITY and nouts[1] == 0
    for c in (0, 2):
        assert stc[c] == sts[c] and np.array_equal(bufs[c][: nouts[c]], rows[c])


def test_end_to_end_three_carriers(na):
    from noaa_apt_b200 import synth
    fs, seconds = 1_200_000, 60.0
    car = [(37_000, 31, 0.0, None, 20.0), (-180_000, 32, 3000.0, 30.0, 20.0), (260_000, 33, 0.0, None, 20.0)]
    x = synth.apt_iq_multi(fs, seconds, carriers=car, fmt="cu8", noise_rel=0.03)
    carriers, rows = na.iq.decode_iq_auto(x, fs)
    print("end to end:", [(c.offset_hz, round(c.snr_db, 1), round(c.apt_score, 3)) for c in carriers])
    assert len(carriers) == 3 and all(r is not None for r in rows)
    s = na.iq.IqSettings(fs)
    for c, r in zip(carriers, rows):
        k = int(np.argmin([abs(c.offset_hz - o) for o, *_ in car]))
        seed = car[k][1]
        assert abs(c.centre_hz - car[k][0]) <= 300.0
        clean = synth.apt_signal(s.audio_rate, seconds, seed=seed)
        want = na.decode(None, None, clean, s.audio_rate)
        with na.Decoder(s.audio_rate, max_samples=clean.size) as dec:
            dec.decode(na.iq.fm_demod(x, na.iq.IqSettings(fs, offset_hz=c.offset_hz)), sync=True)
            n_iq = dec.last_sync().size
            dec.decode(clean, sync=True)
            n_clean = dec.last_sync().size
        assert n_iq == n_clean, (c, n_iq, n_clean)
        assert r.size == want.size
        g, w = r.reshape(-1, 2080), want.reshape(-1, 2080)
        cols = np.r_[86:995, 1126:2035]
        corr = np.corrcoef(g[:, cols].ravel(), w[:, cols].ravel())[0, 1]
        print(f"carrier {car[k][0]:+d} (doppler {car[k][2]}): found {c.centre_hz:+.1f} Hz, image correlation {corr:.4f}")
        assert corr >= 0.98, corr
