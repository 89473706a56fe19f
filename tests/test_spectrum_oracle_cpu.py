"""The CPU restatement of the carrier-finding spectrum (tests/_spectrum_oracle.py) against float64, without a device.

test_gpu_spectrum.py holds the device to this restatement bit for bit, so the error measured here against a float64
FFT average is the device's own error."""
import math

import numpy as np
import pytest

import _spectrum_oracle as so

SIZES = [256, 512, 1024, 2048, 4096, 8192, 16384]

# |restatement - float64| <= C_MEAN * mean(float64 spectrum) in every bin.  Measured on the cases below: at most 2.3e-6
# (K = 1: one segment's rounding is not averaged down), 1.2e-6 at K = 300; the bound keeps about 9x margin.
C_MEAN = 2e-5


def _white(n, fmt, seed):
    rng = np.random.default_rng(seed)
    if fmt == "cu8":
        return rng.integers(0, 256, 2 * n, dtype=np.uint8)
    return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)


def _f64_load(x):
    if x.dtype == np.uint8:
        v = x.astype(np.float64) - 127.5
        return v[0::2] + 1j * v[1::2]
    return x.astype(np.complex128)


def f64_spectrum(x, nfft, max_segments=0):
    """The same average in float64: np.fft.fft of each segment times the float32 window, fftshifted."""
    z = _f64_load(x)
    _, K, starts = so.segment_starts(z.size, nfft, max_segments)
    w = so.tables(nfft)[0].astype(np.float64)
    acc = np.zeros(nfft)
    for a in starts:
        acc += np.abs(np.fft.fft(z[a:a + nfft] * w)) ** 2
    return np.fft.fftshift(acc / K)


@pytest.mark.parametrize("K", [1, 37, 300])
@pytest.mark.parametrize("fmt", ["cf32", "cu8"])
@pytest.mark.parametrize("nfft", SIZES)
def test_restatement_against_float64(nfft, fmt, K):
    n = K * nfft + nfft // 3                              # a partial segment at the end, never used
    x = _white(n, fmt, nfft + K)
    got, k = so.spectrum(x, nfft, K)
    ref = f64_spectrum(x, nfft, K)
    assert k == K and got.dtype == np.float32
    err = np.max(np.abs(got.astype(np.float64) - ref)) / ref.mean()
    print(f"nfft {nfft} {fmt} K {K}: max |error| / mean power {err:.2e}")
    assert err <= C_MEAN


@pytest.mark.parametrize("nfft", SIZES)
def test_tables(nfft):
    win, twr, twi = so.tables(nfft)
    ang = 2.0 * np.pi * np.arange(nfft) / nfft
    assert np.array_equal(win, (0.5 - 0.5 * np.cos(ang)).astype(np.float32))
    assert np.array_equal(twr, np.cos(ang).astype(np.float32))
    assert np.array_equal(twi, (-np.sin(ang)).astype(np.float32))
    assert win[0] == 0.0 and win[nfft // 2] == 1.0 and twr[0] == 1.0 and twi[0] == 0.0 and twi[nfft // 4] == -1.0


def test_segment_starts():
    for nfft in (256, 16384):
        S, K, starts = so.segment_starts(300 * nfft + 7, nfft, 0)
        assert S == K == 300 and starts == [k * nfft for k in range(300)]
        assert so.segment_starts(2 * nfft - 1, nfft) == (1, 1, [0])
        assert so.segment_starts(nfft - 1, nfft)[:2] == (0, 0)
    # the formula of tests/test_gpu_iq_search.py::_ref_spectrum at S = 37, K = 11
    S, K, starts = so.segment_starts(37 * 4096 + 4096 // 3, 4096, 11)
    assert (S, K) == (37, 11) and starts == [(k * 37 // 11) * 4096 for k in range(11)]
    # S not a multiple of K, at the size the carrier search uses: every segment inside the recording, in order
    S, K, starts = so.segment_starts(2051 * 16384 + 100, 16384, 2048)
    assert (S, K) == (2051, 2048) and starts[0] == 0 and starts[-1] == 2049 * 16384     # floor(2047 * 2051 / 2048)
    assert all(b - a in (16384, 2 * 16384) for a, b in zip(starts, starts[1:]))
    assert sum(b - a == 2 * 16384 for a, b in zip(starts, starts[1:])) == 2       # the third unused one is the last


def test_search_nfft():
    assert [so.search_nfft(r) for r in (48_000, 250_000, 1_024_000, 1_200_000, 2_048_000, 2_400_000, 10_000_000)] == \
        [256, 2048, 8192, 8192, 16384, 16384, 16384]


def sweep(nfft):
    """S = K = nfft segments, segment k a unit tone at exact bin k (cf32)."""
    t = np.arange(nfft, dtype=np.int64)
    k = t[:, None]
    return np.exp(2j * np.pi * ((k * t) % nfft) / nfft).astype(np.complex64).ravel()


@pytest.mark.parametrize("nfft", [256, 512, 1024, 2048])
def test_flat_sweep(nfft):
    # the periodic Hann window spreads a bin-centred tone over its bin (N/2 in amplitude) and the two neighbours (-N/4):
    # over all N tones every bin collects N^2/4 + 2 N^2/16, an average of 3N/8
    got, K = so.spectrum(sweep(nfft), nfft, nfft)
    assert K == nfft
    assert np.max(np.abs(got / (3.0 * nfft / 8.0) - 1.0)) <= 1e-5


@pytest.mark.parametrize("freq,want", [(2400.0, 1.0), (12_000.0, 0.0), (150.0, 0.0)])
def test_apt_score(freq, want):
    rate = 48_000
    t = np.arange(3 * rate)
    audio = (1000.0 * np.cos(2 * np.pi * freq * t / rate)).astype(np.float32)
    score = so.apt_score(audio, rate)
    assert score.dtype == np.float32 and abs(float(score) - want) <= 1e-3, score
    # in float64: the score of the float64 spectrum of the same K = S segments
    h = f64_spectrum(audio.astype(np.complex64), so.APT_NFFT, audio.size // so.APT_NFFT)
    f = np.abs((np.arange(so.APT_NFFT) - so.APT_NFFT // 2) * rate / so.APT_NFFT)
    inside = (f >= so.APT_LO_HZ) & (f <= so.APT_HI_HZ)
    assert math.isclose(float(score), h[inside].sum() / h.sum(), rel_tol=1e-5, abs_tol=1e-7)
    assert so.apt_score(audio[: so.APT_NFFT - 1], rate) == 0.0
    assert so.apt_score(np.zeros(2 * so.APT_NFFT, np.float32), rate) == 0.0
