"""The carrier-finding spectrum on the device (k_spectrum / k_spectrum_finish, DESIGN.md §10 "Finding carriers") against
its CPU restatement tests/_spectrum_oracle.py bit for bit: every nfft (radix-2 first stage or not, every B4) and I/Q
format, one to 2048 segments and up to eight per partial-spectrum slot, every way of splitting the segments into
launches, the staging ring, pinned input and the unstaged copy.  Then against float64 and analytic spectra, and
apt_iq_find_carriers composed from apt_iq_spectrum, apt_find_carriers_psd, apt_fm_demod and the restated APT score."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import _spectrum_oracle as so
from test_spectrum_oracle_cpu import C_MEAN, SIZES, _white, f64_spectrum, sweep

pytestmark = pytest.mark.gpu

FORMATS = ["cu8", "cs16", "cf32"]


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


def _device(na, x, nfft, max_segments=0, ptr=None):
    """(psd, nseg) of apt_iq_spectrum through the C ABI; ptr: the same samples at another host address."""
    xs, fmt, n = na.iq.iq_format(x)
    psd = np.empty(nfft, np.float32)
    nseg = C.c_uint32(0)
    ss = na._lib.CSpectrumSettings(nfft, max_segments)
    na.err.raise_for(na._lib.load().apt_iq_spectrum(xs.ctypes.data if ptr is None else ptr, fmt, n, 1_000_000,
                                                    C.byref(ss), psd.ctypes.data, psd.size, C.byref(nseg)))
    return psd, nseg.value


def _assert_bits(got, want, what):
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, f"{what}: {bad.size} bins differ, first {bad[:4].tolist()}: {got[bad[:4]]} vs {want[bad[:4]]}"


def _recording(n, fmt, seed):
    """Two tones 22 dB apart over noise 30 dB below the stronger, quantised to `fmt`."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    z = 0.6 * np.exp(2j * np.pi * 0.1234567 * t) + 0.05 * np.exp(-2j * np.pi * 0.31 * t) \
        + 0.02 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "cf32":
        return z.astype(np.complex64)
    inter = np.empty(2 * n)
    inter[0::2], inter[1::2] = z.real, z.imag
    if fmt == "cu8":
        return np.clip(np.rint(inter * 100.0 + 127.5), 0, 255).astype(np.uint8)
    return np.rint(inter * 20000.0).astype(np.int16)


def _head(x, n):
    return x[:n] if x.dtype == np.complex64 else x[: 2 * n]


def _classes(nfft):
    """(n, max_segments, K): one segment (n = nfft and 2 nfft - 1), K = S = 255, K = 256 of S = 300, K = S = 257, and
    below nfft 16384 K = 2048 of S = 2051 (test_staging_ring_and_pinned_input runs that class at 16384)."""
    c = [(nfft, 0, 1), (2 * nfft - 1, 0, 1), (255 * nfft + nfft // 3, 0, 255), (300 * nfft, 256, 256),
         (257 * nfft + 5, 257, 257)]
    if nfft < 16384:
        c.append((2051 * nfft + 7, 0, 2048))
    return c


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("nfft", SIZES)
def test_bit_identical(na, nfft, fmt):
    classes = _classes(nfft)
    x = _recording(max(n for n, _, _ in classes), fmt, nfft + len(fmt))
    for n, ms, K in classes:
        xn = _head(x, n)
        got, nseg = _device(na, xn, nfft, ms)
        want, k = so.spectrum(xn, nfft, ms)
        assert nseg == k == K, (n, ms, nseg, k)
        _assert_bits(got, want, f"nfft {nfft} {fmt} n {n} K {K}")


@pytest.mark.parametrize("nfft,fmt", [(1024, "cf32"), (8192, "cs16")])
def test_chunks_bit_identical(na, monkeypatch, nfft, fmt):
    # APTB200_IQ_CHUNK / nfft segments per launch: 1 (2048 launches of one CTA), 255 (k0 not a multiple of 256, a grid
    # below 256), 257 (one CTA of each launch takes two segments), all 2048 in one launch.  nfft 16384 is split into
    # launches in test_staging_ring_and_pinned_input.
    x = _recording(2051 * nfft + 7, fmt, 3 * nfft)
    want, K = so.spectrum(x, nfft)
    assert K == 2048
    for per in (1, 255, 257, 2048):
        monkeypatch.setenv("APTB200_IQ_CHUNK", str(per * nfft))
        got, nseg = _device(na, x, nfft)
        assert nseg == K
        _assert_bits(got, want, f"nfft {nfft} {fmt}, {per} segments per launch")


def test_staging_ring_and_pinned_input(na, monkeypatch):
    # 2048 of 2051 segments of 16384 cu8: 64 MB packed, four fills of the staging ring's three 16 MB buffers
    import torch
    nfft = 16384
    x = _recording(2051 * nfft + 100, "cu8", 5)
    want, K = so.spectrum(x, nfft)
    got, nseg = _device(na, x, nfft)
    assert nseg == K == 2048
    _assert_bits(got, want, "pageable, one launch")
    monkeypatch.setenv("APTB200_IQ_CHUNK", str(700 * nfft))      # three launches of up to 22 MB each
    _assert_bits(_device(na, x, nfft)[0], want, "pageable, 700 segments per launch")
    monkeypatch.delenv("APTB200_IQ_CHUNK")
    pinned = torch.from_numpy(x).pin_memory()                    # one copy per run of adjacent segments: three runs
    _assert_bits(_device(na, x, nfft, ptr=pinned.data_ptr())[0], want, "pinned")
    monkeypatch.setenv("APTB200_NO_STAGER", "1")
    na._lib.load().apt_cache_clear()                             # a fresh workspace: it gets no staging ring
    _assert_bits(_device(na, x, nfft)[0], want, "pageable without the staging ring")


@pytest.mark.parametrize("nfft", SIZES)
def test_against_float64(na, nfft):
    for fmt in ("cf32", "cu8"):
        x = _white(37 * nfft + nfft // 3, fmt, 7 * nfft)
        got, _ = _device(na, x, nfft, 37)
        ref = f64_spectrum(x, nfft, 37)
        err = np.max(np.abs(got.astype(np.float64) - ref)) / ref.mean()
        print(f"nfft {nfft} {fmt} K 37: max |error| / mean power {err:.2e}")
        assert err <= C_MEAN


@pytest.mark.parametrize("nfft", SIZES)
def test_zero_and_constant(na, nfft):
    got, _ = _device(na, np.zeros(3 * nfft, np.complex64), nfft)
    assert not np.any(got.view(np.uint32))                       # +0.0 in every bin
    # I = Q = 127 - 127.5: the window's sum at DC (N/2 after the shift), -N/4 at DC +- 1, nothing elsewhere
    got, _ = _device(na, np.full(2 * 3 * nfft, 127, np.uint8), nfft)
    w = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(nfft) / nfft)).astype(np.float32).astype(np.float64)
    dc, b = 2.0 * (0.5 * w.sum()) ** 2, nfft // 2
    assert abs(got[b] / dc - 1.0) <= 1e-6
    assert abs(got[b - 1] / (dc / 4) - 1.0) <= 1e-6 and abs(got[b + 1] / (dc / 4) - 1.0) <= 1e-6
    assert np.max(np.delete(got, [b - 1, b, b + 1])) <= dc * 1e-10     # 100 dB below DC


@pytest.mark.parametrize("nfft", [256, 512, 1024, 2048])
def test_flat_sweep(na, nfft):
    # segment k a unit tone at bin k: every output of every stage carries a tone's whole power once, and the Hann
    # leakage makes the average 3N/8 in every bin (tests/test_spectrum_oracle_cpu.py::test_flat_sweep)
    got, K = _device(na, sweep(nfft), nfft, nfft)
    assert K == nfft
    assert np.max(np.abs(got / (3.0 * nfft / 8.0) - 1.0)) <= 1e-5


# iq_rate: (carriers of synth.apt_iq_multi, a search window (lo, hi) in Hz).  Default nfft 2048, 8192, 8192, 16384.
SEARCH = {
    250_000: ([(31_000, 41, 0.0, None, 20.0)], (0, 90_000)),
    1_024_000: ([(-200_000, 42, 0.0, None, 20.0), (150_000, 43, 0.0, None, 20.0)], (-300_000, 0)),
    1_200_000: ([(37_000, 44, 0.0, None, 20.0)], (-100_000, 100_000)),
    2_400_000: ([(-450_000, 45, 0.0, None, 20.0), (251_313, 46, 0.0, None, 20.0)], (100_000, 400_000)),
}


@pytest.fixture(scope="module")
def searched():
    """iq_rate -> (recording, restated search spectrum), made once per rate."""
    cache = {}

    def get(rate):
        if rate not in cache:
            from noaa_apt_b200 import synth
            x = synth.apt_iq_multi(rate, 5.0, carriers=SEARCH[rate][0], fmt="cu8", noise_rel=0.03)
            cache[rate] = x, so.spectrum(x, so.search_nfft(rate), 2048)[0]
        return cache[rate]
    return get


def _restated_score(na, x, rate, offset):
    """apt_test restated: the middle min(len, 4 s) of apt_fm_demod's audio at `offset`, scored by the restatement; 0
    when the offset is too near the band edge to demodulate."""
    s = dataclasses.replace(na.iq.IqSettings(rate), offset_hz=offset)
    try:
        audio = na.iq.fm_demod(x, s)
    except na.err.InvalidInput as e:
        assert e.code == na._lib.ERR_BAD_ARG
        return np.float32(0)
    L = min(audio.size, 4 * s.audio_rate)
    m0 = (audio.size - L) // 2
    return so.apt_score(audio[m0:m0 + L], s.audio_rate)


def _check_scores(na, x, rate, found):
    for c in found:
        want = _restated_score(na, x, rate, c.offset_hz)
        assert np.float32(c.apt_score).view(np.uint32) == want.view(np.uint32), (c, want)
        assert c.is_apt == (want >= np.float32(0.5)), (c, want)


@pytest.mark.parametrize("window", [False, True])
@pytest.mark.parametrize("rate", list(SEARCH))
def test_find_carriers_composed(na, searched, rate, window):
    x, restated = searched(rate)
    carriers, (lo, hi) = SEARCH[rate][0], SEARCH[rate][1] if window else (None, None)
    nfft = so.search_nfft(rate)
    found = na.iq.find_carriers(x, rate, lo=lo, hi=hi)
    _, psd = na.iq.spectrum(x, rate, nfft=nfft, max_segments=2048)
    _assert_bits(psd, restated, f"search spectrum at {rate}")
    want = na.iq.find_carriers_psd(psd, rate, cutout=na.iq.IqSettings(rate).cutout, lo=lo, hi=hi)
    assert [(c.offset_hz, c.centre_hz, c.snr_db) for c in found] == [(c.offset_hz, c.centre_hz, c.snr_db) for c in want]
    _check_scores(na, x, rate, found)
    placed = sorted(o for o, *_ in carriers if lo is None or lo <= o <= hi)
    assert sorted(c.offset_hz for c in found if c.is_apt) == pytest.approx(placed, abs=300), found


def test_apt_score_edges(na):
    from noaa_apt_b200 import synth
    rate, cutout = 250_000, na.iq.IqSettings(250_000).cutout
    # 2 s: less than the 4 s window, so the score takes all the audio
    x = synth.apt_iq_multi(rate, 2.0, carriers=[(31_000, 47, 0.0, None, 20.0)], fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(x, rate)
    assert any(c.is_apt for c in found), found
    _check_scores(na, x, rate, found)
    # 20 000 samples: 4000 samples of audio at 50 kHz, fewer than one 4096-point segment, so the score is 0
    x = synth.apt_iq_multi(rate, n_samples=20_000, carriers=[(31_000, 47, 0.0, None, 20.0)], fmt="cu8", noise_rel=0.03)
    found = na.iq.find_carriers(x, rate)
    assert found and all(c.apt_score == 0.0 and not c.is_apt for c in found), found
    _check_scores(na, x, rate, found)
    # a carrier 4 kHz past the usable band's edge: the peak is the window's last bin, and the centroid around it lands
    # beyond |offset| + cutout < iq_rate / 2, where the channel filter cannot be made: score 0
    x = synth.apt_iq_multi(rate, 3.0, carriers=[(rate // 2 - int(cutout) + 4000, 48, 0.0, None, 20.0)], fmt="cu8",
                           noise_rel=0.03)
    found = na.iq.find_carriers(x, rate)
    edge = [c for c in found if abs(c.offset_hz) + cutout >= rate / 2]
    assert edge and all(c.apt_score == 0.0 and not c.is_apt for c in edge), found
    _check_scores(na, x, rate, found)
