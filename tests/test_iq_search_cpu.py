"""Finding carriers without a GPU (DESIGN.md §10, "Finding carriers"): the new entry points are exported, their argument
errors come back before any device is touched, the host search (floor, band power, peaks, suppression, centroid) agrees
with a plain-numpy oracle on crafted spectra, and apt_iq_multi is deterministic and chunk-invariant."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as entry

NEW = ("apt_iq_spectrum", "apt_iq_find_carriers", "apt_find_carriers_psd", "apt_decode_iq_channels", "apt_decode_iq_auto")


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def test_abi_exports_the_search(na):
    lib = C.CDLL(na.library_path())
    for name in NEW:
        assert hasattr(lib, name) and name in na._lib.SIGNATURES
    assert lib.apt_abi_version() == 1
    assert C.sizeof(na._lib.CCarrier) == 20 and C.sizeof(na._lib.CCarrierSearch) == 20
    assert C.sizeof(na._lib.CSpectrumSettings) == 8


def _iq(n):
    return np.full(2 * n, 128, np.uint8)


def test_argument_errors_before_the_device(na):
    """Every one of these would be APT_ERR_CUDA without a device if it reached one."""
    lib = na._lib.load()
    L = na._lib
    x = _iq(100_000)
    psd = np.empty(16384, np.float32)
    nseg = C.c_uint32(0)
    for nfft in (0, 128, 1000, 32768):
        ss = L.CSpectrumSettings(nfft, 0)
        assert lib.apt_iq_spectrum(x.ctypes.data, L.CU8, 100_000, 2_400_000, C.byref(ss), psd.ctypes.data, psd.size,
                                   C.byref(nseg)) == L.ERR_BAD_ARG
    ss = L.CSpectrumSettings(4096, 0)
    assert lib.apt_iq_spectrum(x.ctypes.data, L.CU8, 4095, 2_400_000, C.byref(ss), psd.ctypes.data, psd.size,
                               C.byref(nseg)) == L.ERR_BAD_ARG                       # fewer than nfft samples
    assert lib.apt_iq_spectrum(None, L.CU8, 100_000, 2_400_000, C.byref(ss), psd.ctypes.data, psd.size,
                               C.byref(nseg)) == L.ERR_BAD_ARG
    assert lib.apt_iq_spectrum(x.ctypes.data, L.F32, 100_000, 2_400_000, C.byref(ss), psd.ctypes.data, psd.size,
                               C.byref(nseg)) == L.ERR_BAD_ARG
    assert lib.apt_iq_spectrum(x.ctypes.data, L.CU8, 100_000, 2_400_000, C.byref(ss), psd.ctypes.data, 4095,
                               C.byref(nseg)) == L.ERR_CAPACITY
    s = na.iq.IqSettings(2_400_000).to_c()
    out = (L.CCarrier * 8)()
    cnt = C.c_uint32(0)
    inverted = L.CCarrierSearch(50_000, -50_000, 0, 0, 0.0)
    assert lib.apt_iq_find_carriers(x.ctypes.data, L.CU8, 100_000, C.byref(s), C.byref(inverted), out, 8,
                                    C.byref(cnt)) == L.ERR_BAD_ARG
    cs = L.CCarrierSearch(0, 0, 16384, 0, 0.0)
    assert lib.apt_iq_find_carriers(x.ctypes.data, L.CU8, 16383, C.byref(s), C.byref(cs), out, 8,
                                    C.byref(cnt)) == L.ERR_BAD_ARG
    assert lib.apt_iq_find_carriers(x.ctypes.data, L.CU8, 100_000, None, C.byref(cs), out, 8, C.byref(cnt)) == L.ERR_BAD_ARG
    assert lib.apt_iq_find_carriers(x.ctypes.data, L.CU8, 100_000, C.byref(s), C.byref(cs), None, 8,
                                    C.byref(cnt)) == L.ERR_BAD_ARG

    # channels: count < 1, NULL pointers, an offset past the band edge, too short: every status set, no device
    n = 2_400_000 * 12
    big = np.zeros(1, np.uint8)   # never read: the errors come first
    st = na.Settings().to_c()
    rows = np.empty(16, np.float32)
    k = 3
    outs = (C.c_void_p * k)(*([rows.ctypes.data] * k))
    caps = (C.c_uint64 * k)(*([1 << 40] * k))
    nouts = (C.c_uint64 * k)()
    sts = (C.c_int * k)()
    offs = (C.c_int32 * k)(37_000, -120_000, 2_400_000 // 2 - 22_000)       # |offset| + cutout == iq_rate / 2
    assert lib.apt_decode_iq_channels(big.ctypes.data, L.CU8, n, C.byref(s), offs, 0, C.byref(st), 1, outs, caps, nouts,
                                      sts) == L.ERR_BAD_ARG
    assert lib.apt_decode_iq_channels(big.ctypes.data, L.CU8, n, C.byref(s), None, k, C.byref(st), 1, outs, caps, nouts,
                                      sts) == L.ERR_BAD_ARG
    assert lib.apt_decode_iq_channels(big.ctypes.data, L.CU8, n, C.byref(s), offs, k, C.byref(st), 1, outs, caps, nouts,
                                      sts) == L.ERR_BAD_ARG
    assert list(sts) == [L.ERR_BAD_ARG] * k
    offs[2] = 251_313
    assert lib.apt_decode_iq_channels(big.ctypes.data, L.CU8, 2_400_000 * 4, C.byref(s), offs, k, C.byref(st), 1, outs,
                                      caps, nouts, sts) == L.ERR_TOO_SHORT
    assert list(sts) == [L.ERR_TOO_SHORT] * k
    # auto: the search's and the decode's argument errors
    found = (L.CCarrier * 4)()
    nf = C.c_uint32(0)
    assert lib.apt_decode_iq_auto(big.ctypes.data, L.CU8, n, C.byref(s), C.byref(inverted), C.byref(st), 1, found, 3,
                                  C.byref(nf), outs, caps, nouts, sts) == L.ERR_BAD_ARG
    assert lib.apt_decode_iq_auto(big.ctypes.data, L.CU8, 2_400_000 * 4, C.byref(s), None, C.byref(st), 1, found, 3,
                                  C.byref(nf), outs, caps, nouts, sts) == L.ERR_TOO_SHORT
    assert lib.apt_decode_iq_auto(big.ctypes.data, L.CU8, n, C.byref(s), None, C.byref(st), 1, None, 3,
                                  C.byref(nf), outs, caps, nouts, sts) == L.ERR_BAD_ARG


def oracle_search(psd, fs, cutout, lo=None, hi=None, min_snr_db=6.0):
    """The search of apt_iq_find_carriers in plain numpy (float64): [(offset_hz, centre_hz, snr_db)] by descending SNR."""
    N = psd.size
    p = psd.astype(np.float64)
    f = (np.arange(N) - N // 2) * (fs / N)
    inside = np.abs(f) + cutout < fs / 2
    if lo is not None:
        inside &= (f >= lo) & (f <= hi)
    win = np.nonzero(inside)[0]
    if win.size == 0:
        return []
    wa, wb = win[0], win[-1]
    floor = np.median(p[wa:wb + 1])
    if not floor > 0:
        return []
    hb = (20000 * N) // fs
    P = np.concatenate([[0.0], np.cumsum(p)])
    a = np.maximum(np.arange(N) - hb, 0)
    c = np.minimum(np.arange(N) + hb, N - 1)
    E = P[c + 1] - P[a]
    nb = c - a + 1
    cands = []
    i = wa
    while i <= wb:
        j = i
        while j < wb and E[j + 1] == E[i]:
            j += 1
        if (i == wa or E[i - 1] < E[i]) and (j == wb or E[j + 1] < E[j]):
            snr = 10 * np.log10(E[i] / (floor * nb[i]))
            if snr >= min_snr_db:
                cands.append((i, snr))
        i = j + 1
    cands.sort(key=lambda t: -E[t[0]])          # stable: ties keep the lower bin first
    kept = []
    for b, snr in cands:
        if all(abs(b - k) * (fs / N) > 40000 for k, _ in kept):
            kept.append((b, snr))
    kept.sort(key=lambda t: -t[1])
    out = []
    for b, snr in kept:
        sl = slice(max(0, b - hb), min(N - 1, b + hb) + 1)
        w = p[sl] - floor
        w = np.where(w > 0, w, 0.0)
        centre = float(np.sum(w * f[sl]) / np.sum(w)) if np.sum(w) > 0 else float(f[b])
        out.append((int(np.floor(centre + 0.5)) if centre >= 0 else -int(np.floor(-centre + 0.5)), centre, snr))
    return out


def _compare(na, psd, fs, cutout=22000.0, **kw):
    got = na.iq.find_carriers_psd(psd, fs, cutout, **kw)
    kw2 = dict(kw)
    if kw2.get("min_snr_db", 0.0) == 0.0:
        kw2["min_snr_db"] = 6.0
    want = oracle_search(psd, fs, cutout, **kw2)
    assert len(got) == len(want), (got, want)
    for g, (off, centre, snr) in zip(got, want):
        assert g.offset_hz == off
        assert abs(g.centre_hz - centre) <= 1e-6 * max(1.0, abs(centre)) + 1e-3
        assert abs(g.snr_db - snr) <= 1e-5
        assert not g.is_apt and g.apt_score == 0.0
    return got


def _bump(N, fs, centre, width, height):
    f = (np.arange(N) - N // 2) * (fs / N)
    return height * (np.abs(f - centre) <= width)


def test_search_matches_numpy_oracle(na):
    rng = np.random.default_rng(3)
    for fs, N in ((2_400_000, 16384), (1_200_000, 8192), (250_000, 2048)):
        for trial in range(6):
            base = rng.uniform(0.8, 1.2, N)
            psd = base.copy()
            k = int(rng.integers(1, 4))
            for _ in range(k):
                c = rng.uniform(-0.4, 0.4) * fs
                psd += _bump(N, fs, c, rng.uniform(5000, 17000), rng.uniform(2, 50))
            got = _compare(na, psd.astype(np.float32), fs)
            assert len(got) >= 1
            _compare(na, psd.astype(np.float32), fs, lo=-fs // 4, hi=fs // 4)
            _compare(na, psd.astype(np.float32), fs, min_snr_db=3.0)
    # pure flat noise floor: nothing
    assert na.iq.find_carriers_psd(np.ones(16384, np.float32), 2_400_000) == []
    # all zero: no floor, nothing
    assert na.iq.find_carriers_psd(np.zeros(4096, np.float32), 1_200_000) == []


def test_search_ties_edges_and_suppression(na):
    fs, N = 2_400_000, 16384
    bw = fs / N
    # integer-valued spectra: prefix sums are exact, so plateaus of E are exact ties (the first bin of a run wins)
    psd = np.ones(N)
    psd += _bump(N, fs, 100_000, 15_000, 20.0)
    got = _compare(na, psd.astype(np.float32), fs)
    assert len(got) == 1 and abs(got[0].centre_hz - 100_000) < bw
    # two carriers 30 kHz apart: the weaker one is suppressed; 50 kHz apart: both kept
    for sep, n_keep in ((30_000, 1), (50_000, 2)):
        psd = np.ones(N) + _bump(N, fs, 0, 8000, 30.0) + _bump(N, fs, sep, 8000, 20.0)
        got = _compare(na, psd.astype(np.float32), fs)
        assert len(got) == n_keep
    # two equal carriers far apart: both kept, the tie in E broken by the lower bin
    psd = np.ones(N) + _bump(N, fs, -300_000, 10_000, 10.0) + _bump(N, fs, 300_000, 10_000, 10.0)
    got = _compare(na, psd.astype(np.float32), fs)
    assert len(got) == 2
    # a carrier at the window edge and one cut by the usable band's edge
    edge = fs // 2 - 22_000 - 30_000
    psd = np.ones(N) + _bump(N, fs, edge, 12_000, 25.0)
    _compare(na, psd.astype(np.float32), fs)
    _compare(na, psd.astype(np.float32), fs, lo=edge - 5000, hi=edge + 5000)
    _compare(na, psd.astype(np.float32), fs, lo=-200_000, hi=edge - 20_000)
    # a window that holds no bin
    assert na.iq.find_carriers_psd(psd.astype(np.float32), fs, lo=fs, hi=fs + 1000) == []
    # capacity: the full count comes back with APT_ERR_CAPACITY
    psd = np.ones(N)
    for c in (-600_000, -300_000, 0, 300_000, 600_000):
        psd += _bump(N, fs, c, 10_000, 10.0)
    lib = na._lib.load()
    p = psd.astype(np.float32)
    out = (na._lib.CCarrier * 2)()
    cnt = C.c_uint32(0)
    assert lib.apt_find_carriers_psd(p.ctypes.data, N, fs, 22000.0, None, out, 2, C.byref(cnt)) == na._lib.ERR_CAPACITY
    assert cnt.value == 5
    assert lib.apt_find_carriers_psd(p.ctypes.data, N, fs, 22000.0, None, None, 0, C.byref(cnt)) == na._lib.ERR_CAPACITY
    assert cnt.value == 5


def test_apt_iq_multi_deterministic_and_chunk_invariant():
    from noaa_apt_b200 import synth
    fs = 250_000
    car = [(37_000, 3, 3000.0, 0.2, 0.5), (-60_000, 5, 0.0, None, 20.0)]
    bands = [(10_000, 40_000, 0.5)]
    for fmt in ("cu8", "cs16", "cf32"):
        a = synth.apt_iq_multi(fs, 1.0, carriers=car, extra_bands=bands, fmt=fmt)
        b = synth.apt_iq_multi(fs, 1.0, carriers=car, extra_bands=bands, fmt=fmt)
        c = synth.apt_iq_multi(fs, 1.0, carriers=car, extra_bands=bands, fmt=fmt, chunk=70_001)
        assert np.array_equal(a, b) and np.array_equal(a, c), fmt
        assert a.size == (fs if fmt == "cf32" else 2 * fs)
    # one carrier without Doppler or bands: the signal of apt_iq (the noise differs in its generator only)
    x = synth.apt_iq_multi(fs, 0.5, carriers=[(20_000, 7, 0.0, None, 10.0)], fmt="cf32", noise_rel=0.0)
    y = synth.apt_iq(fs, 0.5, seed=7, offset_hz=20_000, fmt="cf32", noise_rel=0.0)
    assert np.max(np.abs(x - y)) < 1e-5
    # the Doppler shape: the instantaneous frequency crosses offset_hz at tca and swings by +-doppler
    z = synth.apt_iq_multi(fs, 1.0, carriers=[(0, 1, 3000.0, 0.5, 0.05)], fmt="cf32", noise_rel=0.0,
                           deviation_hz=0.0).astype(np.complex128)
    inst = np.angle(z[1:] * np.conj(z[:-1])) * fs / (2 * np.pi)
    assert abs(inst[1000] - 3000.0 * 0.5 / np.hypot(0.5, 0.05)) < 5
    assert abs(inst[-1000] + 3000.0 * 0.5 / np.hypot(0.5, 0.05)) < 5
