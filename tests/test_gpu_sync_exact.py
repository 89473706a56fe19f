"""The fused back half on the GPU, pinned bit for bit against its float32 restatement (_sync_oracle.py) on the device's
own envelope: the low-passed signal, the correlation, every tile's record counts, maximum and records (what
k_lowpass_records wrote, read back with Decoder.last_records), the roots, the positions and the rows.

Every kind that decodes with the fused low-pass is held to the same bits: the Records kind (f and corr never written,
rows gathered straight from the envelope), the Hbm kind (APTB200_LEGACY_SYNC=1, and the redo after a record-pool
overflow) and the stream.  A comparison to within 1e-5 of the oracle cannot see a dropped edge tap, a reassociated box
sum or a weak record test made strict; these can.

The recordings carry a zero gap of about one work sample at six places, so that the sync positions take all four
alignments of the row gather's 16-byte staging.  A decode needs ten rows (decode.rs:79-83), so the correlation always
spans more than one tile and more than min_distance; the shortest decodable recording is among the length edges.
"""
import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import synth
from noaa_apt_b200.err import InvalidInput
import _sync_oracle as so

pytestmark = pytest.mark.gpu

CASES = [(48000, "standard"), (48000, "fast"), (48000, "slow"), (11025, "standard")]
IDS = [f"{r}-{p}" for r, p in CASES]
REGION = 640                     # kRegion (back.cu): records a tile keeps in its own region of the pool


def recording(rate, s, seconds=16, seed=61, cuts=6):
    """synth.apt_signal with a zero gap of about one work sample at `cuts` places: every gap moves the sync phase."""
    x = synth.apt_signal(rate, seconds, seed=seed)
    gap = max(1, round(rate / s.work_rate))
    parts = np.split(x, [x.size * (i + 1) // (cuts + 1) for i in range(cuts)])
    out = []
    for i, p in enumerate(parts):
        out.append(p)
        if i < cuts:
            out.append(np.zeros(gap, np.float32))
    return np.concatenate(out)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(bits(got) != bits(want))
    assert bad.size == 0, f"{what}: {bad.size} of {want.size} values differ, first at {bad[:8].tolist()}"


def decode(rate, s, x, sync):
    """One decode and everything the decoder reads back about it."""
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        got = {"rows": dec.decode(x, sync=sync), "e": dec.read_stage("demodulated")}
        if sync:
            got["pos"] = dec.last_sync()
            try:
                got["tiles"], got["records"] = dec.last_records()
            except InvalidInput:
                pass                                     # the job did not end on the record kernel's output
            roots = dec.last_roots()
        got["f"] = dec.read_stage("filtered")
        if sync:
            got["corr"] = dec.read_stage("correlation")
            got["roots"] = dec.last_roots()
            assert np.array_equal(got["roots"], roots)  # read_stage leaves the job's roots where they are
            if "tiles" in got:                           # ... and its records
                t2, r2 = dec.last_records()
                assert np.array_equal(t2, got["tiles"]) and np.array_equal(r2, got["records"])
    return got


def assert_records(got, ref):
    gt, rt = got["tiles"], ref["tiles"]
    assert gt.size == rt.size, ("tiles", gt.size, rt.size)
    for k in ("n_suffix", "n_prefix"):
        bad = np.flatnonzero(gt[k] != rt[k])
        assert bad.size == 0, f"{k} differs in tiles {bad[:8].tolist()}: {gt[k][bad[:4]]} vs {rt[k][bad[:4]]}"
    assert_bits(gt["max"], rt["max"], "tile maxima")
    gr, rr = got["records"], ref["records"]
    assert gr.size == rr.size, ("records", gr.size, rr.size)
    bad = np.flatnonzero(gr["pos"] != rr["pos"])
    assert bad.size == 0, f"record positions differ at {bad[:8].tolist()}"
    assert_bits(gr["val"], rr["val"], "record values")


def check(rate, s, x, sync, records):
    """Decode x and compare every output with the restatement; returns (device outputs, restatement)."""
    got = decode(rate, s, x, sync)
    ref = so.back_half(got["e"], s.work_rate, s.demodulation_atten, sync)
    assert_bits(got["f"], ref["f"], "f")
    if sync:
        assert_bits(got["corr"], ref["corr"], "correlation")
        assert np.array_equal(got["roots"], ref["roots"]), "roots"
        assert np.array_equal(got["pos"], ref["positions"]), "positions"
        assert ("tiles" in got) == records
        if records:
            assert_records(got, ref)
    assert_bits(got["rows"], ref["rows"], "rows")
    return got, ref


def alignments(pos, s, nrows):
    """(pos - EOFF) mod 4 of the gathered rows: the compute variant of both half rows (the second half starts
    PW * 1040 samples later, a multiple of 4)."""
    eoff = (so.lowpass_taps(s.work_rate, s.demodulation_atten).size - 1 + 3) // 4 * 4
    return set(((pos[:nrows].astype(np.int64) - eoff) % 4).tolist())


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_records_kind_with_sync(rate, profile):
    s = na.Settings.profile(profile)
    got, ref = check(rate, s, recording(rate, s), True, True)
    assert alignments(got["pos"], s, got["rows"].size // 2080) == {0, 1, 2, 3}


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_records_kind_without_sync(rate, profile):
    s = na.Settings.profile(profile)
    check(rate, s, recording(rate, s), False, False)


@pytest.mark.parametrize("sync", [True, False], ids=["sync", "nosync"])
@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_hbm_kind(rate, profile, sync, monkeypatch):
    monkeypatch.setenv("APTB200_LEGACY_SYNC", "1")
    s = na.Settings.profile(profile)
    check(rate, s, recording(rate, s, seed=62), sync, False)


def length_edges(rate, s, x):
    """Input lengths (prefixes of x) whose correlation leaves ncorr mod W in {0, 1, 31, 32, 33, W-1}, and the shortest
    decodable length (ten rows).  A remainder no input length reaches at the first tile count is taken a tile earlier."""
    pw = so.pixel_width(s.work_rate)
    w = so.tile_width(pw)
    g = 38 * pw
    full = so.work_len(x.size, rate, s)
    out = {}
    for r in (0, 1, 31, 32, 33, w - 1):
        tiles = (full - g - 1) // w - 1
        while r not in out and tiles > 0:
            n = so.input_len_for(tiles * w + r + g, rate, s)
            if n is not None:
                out[r] = n
            tiles -= 1
    assert len(out) == 6, sorted(out)
    shortest = next(n for k in range(8) if (n := so.input_len_for(10 * 2080 * pw + k, rate, s)) is not None)
    return out, shortest


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_tile_and_length_edges(rate, profile):
    s = na.Settings.profile(profile)
    x = recording(rate, s, seconds=12, seed=63)
    pw = so.pixel_width(s.work_rate)
    w = so.tile_width(pw)
    edges, shortest = length_edges(rate, s, x)
    for r, n in edges.items():
        got, ref = check(rate, s, x[:n], True, True)
        ncorr = got["corr"].size
        assert ncorr % w == r and got["tiles"].size == -(-ncorr // w)
    got, ref = check(rate, s, x[:shortest], True, True)
    assert got["rows"].size // 2080 >= 8
    check(rate, s, x[:shortest], False, False)


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_last_row_close_to_the_end(rate, profile):
    """The recording ends just after the correlation reaches the row after row k: row k is the last one gathered, and it
    ends 38*PW + d samples before the end of the envelope, the least a regular signal allows (the last position is
    never gathered, and it needs 38*PW samples of correlation after it)."""
    s = na.Settings.profile(profile)
    x = recording(rate, s, seed=64)
    pw = so.pixel_width(s.work_rate)
    row = 2080 * pw
    pos = decode(rate, s, x, True)["pos"].astype(np.int64)
    gaps = []
    for k in (pos.size - 4, pos.size - 7):
        for d in (1, 7, 20):
            n = next(n for j in range(4) if (n := so.input_len_for(int(pos[k]) + row + 38 * pw + d + j, rate, s)))
            got, _ = check(rate, s, x[:n], True, True)
            nr = got["rows"].size // 2080
            gaps.append(got["f"].size - (int(got["pos"][nr - 1]) + row))
    assert min(gaps) <= 38 * pw + 24, gaps


@pytest.mark.parametrize("where", ["inside", "end"])
@pytest.mark.parametrize("region", [None, "8"], ids=["regions", "region8"])
@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_exact_ties_of_silence(rate, profile, where, region, monkeypatch):
    """Zero input gives an exact 0.0 correlation plateau away from the filter edges: equal values decide the weak and
    strict records and the picker's strict `>`.  At the end of the recording every plateau position is a weak suffix
    record, more than a tile's region holds: those tiles take their records from the shared overflow area (with a
    region of 8 records, most tiles do)."""
    if region:
        monkeypatch.setenv("APTB200_RECORD_REGION", region)
    s = na.Settings.profile(profile)
    x = recording(rate, s, seconds=11 if region else 16, seed=65)   # 11 s: the slow profile's records fit the overflow area
    k = int(0.3 * rate)
    if where == "inside":
        x[x.size // 2: x.size // 2 + k] = 0.0
    else:
        x[-k:] = 0.0
    got, ref = check(rate, s, x, True, True)
    zeros = np.flatnonzero(ref["corr"] == 0)
    assert zeros.size > so.tile_width(so.pixel_width(s.work_rate))
    big = got["tiles"]["n_suffix"] + got["tiles"]["n_prefix"]
    if where == "end":
        assert big.max() > REGION
    if region:
        assert np.count_nonzero(big > 8) > big.size // 2


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_pool_overflow_redo(rate, profile, monkeypatch):
    s = na.Settings.profile(profile)
    x = recording(rate, s, seed=66)
    plain = decode(rate, s, x, True)
    assert "tiles" in plain
    monkeypatch.setenv("APTB200_RECORD_POOL", "4096")
    got, _ = check(rate, s, x, True, False)              # redone by the Hbm kernels: no records to read back
    assert np.array_equal(got["pos"], plain["pos"])
    assert_bits(got["rows"], plain["rows"], "rows after the redo")


def test_seed15_tie_same_positions_in_every_kind(monkeypatch):
    """Seed 15 of the bench's recordings holds two neighbouring sync candidates 1 ulp apart: apt_decode (Records),
    APTB200_LEGACY_SYNC=1 (Hbm) and the stream in 1 s pushes must pick the same one, since all three compute the same
    correlation bits."""
    rate = 48000
    x = synth.apt_pcm16(rate, 900, seed=15).astype(np.float32)
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        rows_rec = dec.decode(x, sync=True)
        pos_rec = dec.last_sync()
        dec.last_records()                               # the Records kind ran, without a redo
    monkeypatch.setenv("APTB200_LEGACY_SYNC", "1")
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        rows_hbm = dec.decode(x, sync=True)
        pos_hbm = dec.last_sync()
    monkeypatch.delenv("APTB200_LEGACY_SYNC")
    with na.Stream(rate, sync=True, max_push=rate) as strm:
        parts = [strm.push(x[t:t + rate]) for t in range(0, x.size, rate)]
        parts.append(strm.finish())
        pos_str = strm.positions()
    rows_str = np.concatenate(parts).ravel()
    assert np.array_equal(pos_hbm, pos_rec)
    assert np.array_equal(pos_str, pos_rec)
    assert_bits(rows_hbm, rows_rec, "Hbm rows")
    assert_bits(rows_str, rows_rec, "stream rows")


def test_last_records_refuses_jobs_without_records(monkeypatch):
    rate = 48000
    s = na.Settings()
    x = recording(rate, s, seconds=12, seed=67)
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        with pytest.raises(InvalidInput):
            dec.last_records()                           # no job yet
        dec.decode(x, sync=False)
        with pytest.raises(InvalidInput):
            dec.last_records()
        dec.decode(x, sync=True)
        tiles, recs = dec.last_records()
        assert tiles.size and recs.size == int(tiles["n_suffix"].sum() + tiles["n_prefix"].sum())
    monkeypatch.setenv("APTB200_LEGACY_SYNC", "1")
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        dec.decode(x, sync=True)
        with pytest.raises(InvalidInput):
            dec.last_records()
