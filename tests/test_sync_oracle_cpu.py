"""The float32 restatement of the fused back half (_sync_oracle.py), checked without a GPU.

- fma32 is the correctly rounded float32 FMA: equal to the exact rational value rounded to nearest-even on random
  operands, and on constructed operands where rounding through float64 first lands on a float32 midpoint and rounds the
  wrong way.
- The restated low-pass and correlation are within float32 rounding of the C oracle's sequential sums.
- The per-tile records rebuild exactly the roots of the definition, with the k_resolve_roots rule, on real, silent,
  monotone, integer-valued and plateau signals (plateaus are where weak and strict records differ).
- The restated picker gives oracle.find_sync's positions on the golden excerpts (one holds a duplicate push), and the
  restated rows are the oracle's decode.
- The tile widths are the record kernel's.
"""
import os
from fractions import Fraction

import numpy as np
import pytest

import __graft_entry__ as entry
import noaa_apt_b200 as na
from noaa_apt_b200 import synth
import _sync_oracle as so
import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -24


@pytest.fixture(scope="module", autouse=True)
def built():
    entry.build()


def exact_fma(a, b, c):
    """float32 nearest-even rounding of the exact a*b + c."""
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    x = np.float32(float(v))
    best = None
    for cand in (np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))):
        if not np.isfinite(cand):
            continue
        d = abs(Fraction(float(cand)) - v)
        key = (d, int(np.array(cand, np.float32).view(np.uint32)) & 1)    # ties: even significand
        if best is None or key < best[0]:
            best = (key, cand)
    return np.float32(best[1])


def test_fma32_random_operands():
    rng = np.random.default_rng(1)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * 2.0 ** rng.integers(-30, 0, n))).astype(np.float32)
    c[::3] = (rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n)).astype(np.float32)[::3]
    got = so.fma32(a, b, c)
    want = np.array([exact_fma(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def double_rounding_cases():
    """(a, b, c): the exact sum lies 2^-70 relative off a float32 midpoint, on the side opposite to the even neighbour;
    float64 rounds it onto the midpoint, and the float32 tie then goes to the wrong (even) side."""
    one_up = np.float32(1 + 2.0 ** -23)                  # odd significand
    b = np.float32(2.0 ** -24 * (1 - 2.0 ** -23))        # (1 + 2^-23) b = 2^-24 - 2^-70
    cases = []
    for scale in (1.0, 2.0 ** 10, 2.0 ** -10):
        s = np.float32(scale)
        cases += [(one_up, b * s, one_up * s), (one_up, -b * s, one_up * s),
                  (-one_up, b * s, -one_up * s), (-one_up, -b * s, -one_up * s)]
    return cases


def test_fma32_where_float64_double_rounding_fails():
    for a, b, c in double_rounding_cases():
        want = exact_fma(a, b, c)
        naive = np.float32(np.float64(a) * np.float64(b) + np.float64(c))
        assert naive != want, (a, b, c)                   # the construction really defeats float64
        assert so.fma32(a, b, c) == want, (a, b, c)


def test_fma32_signed_zeros():
    z = so.fma32(np.float32([0.5, -0.5, 0.0]), np.float32([0.0, 0.0, -1.0]), np.float32([0.0, 0.0, -0.0]))
    assert list(np.signbit(z)) == [False, False, True]


@pytest.fixture(scope="module")
def steps():
    out = {}
    for rate, profile, seconds, seed in ((48000, "standard", 14, 3), (48000, "fast", 12, 4), (48000, "slow", 12, 5),
                                         (11025, "standard", 14, 6)):
        s = na.Settings.profile(profile)
        o = oracle.default_settings()
        for k in ("work_rate", "resample_atten", "resample_delta_freq", "resample_cutout", "demodulation_atten"):
            setattr(o, k, getattr(s, k))
        x = synth.apt_signal(rate, seconds, seed=seed)
        ref, st = oracle.decode_steps(x, rate, o)
        out[(rate, profile)] = (s, x, ref, st)
    return out


CASES = [(48000, "standard"), (48000, "fast"), (48000, "slow"), (11025, "standard")]
IDS = [f"{r}-{p}" for r, p in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_taps_are_the_oracle_design(steps, case):
    s = steps[case][0]
    c = np.float32(so.FINAL_RATE) / np.float32(s.work_rate)
    want = oracle.design(1, float(c), s.demodulation_atten, float(c / np.float32(5)))
    got = so.lowpass_taps(s.work_rate, s.demodulation_atten)
    assert got.size in (37, 43, 61) and np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_lowpass_and_correlation_within_rounding_of_the_oracle(steps, case):
    s, _, _, st = steps[case]
    e, fref = st["demodulated"], st["filtered"]
    taps = so.lowpass_taps(s.work_rate, s.demodulation_atten)
    f = so.lowpass(e, taps)
    nt = taps.size
    ep = np.concatenate([np.zeros(nt, np.float64), np.abs(e.astype(np.float64))])
    ep[nt] = 0.0                                         # e[0] is never read
    mag = sum(abs(float(taps[t])) * ep[nt - t: nt - t + e.size] for t in range(nt))
    assert np.all(np.abs(f.astype(np.float64) - fref) <= 2 * nt * EPS * mag + 1e-30)
    # the correlation of the oracle's own f, in the kernels' order and in the reference's
    pw = so.pixel_width(s.work_rate)
    corr = so.correlation(fref, pw)
    _, cref = oracle.find_sync(fref, s.work_rate, want_corr=True)
    g = 38 * pw
    af = np.concatenate([[0.0], np.cumsum(np.abs(fref.astype(np.float64)))])
    cmag = af[g: g + cref.size] - af[: cref.size]
    assert corr.size == cref.size
    assert np.all(np.abs(corr.astype(np.float64) - cref) <= 2 * g * EPS * cmag + 1e-30)
    assert np.any(corr != cref)                           # the orders really differ


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_rows_are_the_oracle_decode(steps, case):
    s, _, ref, st = steps[case]
    pw = so.pixel_width(s.work_rate)
    got = so.rows(st["filtered"], st["sync_pos"], pw)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    _, o = steps[case][1], oracle.default_settings()
    for k in ("work_rate", "resample_atten", "resample_delta_freq", "resample_cutout", "demodulation_atten"):
        setattr(o, k, getattr(s, k))
    ref_nosync = oracle.decode(steps[case][1], case[0], o, sync=False)
    assert np.array_equal(so.rows(st["filtered"], None, pw).view(np.uint32), ref_nosync.view(np.uint32))


def resolve_roots(tiles, recs, w, dist, ncorr):
    """k_resolve_roots on the records: p is a root iff it is a suffix record of its tile, no tile strictly inside
    (p, p+D] has a larger maximum, and the first prefix record of the window's last tile that exceeds corr[p] lies
    beyond p+D."""
    off = np.concatenate([[0], np.cumsum(tiles["n_suffix"].astype(np.int64) + tiles["n_prefix"])])
    out = []
    for t in range(tiles.size):
        suf = recs[off[t]: off[t] + tiles["n_suffix"][t]]
        for p, v in zip(suf["pos"].astype(np.int64), suf["val"]):
            end = min(p + dist, ncorr - 1)
            te = end // w
            if te > t + 1 and np.max(tiles["max"][t + 1: te]) > v:
                continue
            if te > t:
                pre = recs[off[te] + tiles["n_suffix"][te]: off[te + 1]]
                big = np.nonzero(pre["val"] > v)[0]
                if big.size and pre["pos"][big[0]] <= end:
                    continue
            out.append(p)
    return np.array(out, np.uint64)


def records_brute(c, w):
    """Records by their definitions, position by position."""
    tiles, pos = [], []
    for t in range(0, c.size, w):
        x = c[t: t + w]
        suf = [i for i in range(x.size) if not np.any(x[i + 1:] > x[i])]
        pre = [i for i in range(x.size) if np.all(x[i] > x[:i])]
        tiles.append((len(suf), len(pre), x.max()))
        pos += [t + i for i in suf] + [t + i for i in pre]
    return tiles, np.array(pos, np.int64)


def signals(steps):
    rng = np.random.default_rng(7)
    real = so.correlation(steps[(48000, "standard")][3]["filtered"], 3)
    n = 40_000
    plateau = np.repeat(rng.integers(0, 6, n // 300 + 1), 300)[:n].astype(np.float32)
    plateau[n // 2: n // 2 + 9000] = 5.0                  # one plateau wider than the window, across tiles
    return {
        "real": real,
        "silent": np.zeros(n, np.float32),
        "rising": np.arange(n, dtype=np.float32),
        "falling": np.arange(n, 0, -1).astype(np.float32),
        "integers": rng.integers(-3, 4, n).astype(np.float32),
        "plateau": plateau,
        "real_then_silent": np.concatenate([real[:30_000], np.zeros(12_000, np.float32)]),
    }


@pytest.mark.parametrize("name", ["real", "silent", "rising", "falling", "integers", "plateau", "real_then_silent"])
@pytest.mark.parametrize("pw", [3, 4, 5])
def test_records_rebuild_the_roots(steps, name, pw):
    c = signals(steps)[name]
    w = so.tile_width(pw)
    dist = so.min_distance(pw * so.FINAL_RATE)
    tiles, recs = so.tile_records(c, w)
    assert tiles.size == -(-c.size // w)
    assert np.array_equal(resolve_roots(tiles, recs, w, dist, c.size), so.roots_direct(c, dist))
    # records by definition on a few tiles (first, middle, last)
    off = np.concatenate([[0], np.cumsum(tiles["n_suffix"].astype(np.int64) + tiles["n_prefix"])])
    for t in sorted({0, tiles.size // 2, tiles.size - 1}):
        bt, bpos = records_brute(c[t * w: (t + 1) * w], w)
        assert tuple(tiles[t]) == bt[0]
        assert np.array_equal(recs["pos"][off[t]: off[t + 1]].astype(np.int64) - t * w, bpos)
        assert np.array_equal(recs["val"][off[t]: off[t + 1]], c[recs["pos"][off[t]: off[t + 1]]])


def test_plateaus_separate_weak_and_strict_records(steps):
    c = signals(steps)["silent"]
    tiles, _ = so.tile_records(c, 1920)
    assert np.all(tiles["n_suffix"][:-1] == 1920) and np.all(tiles["n_prefix"] == 1)


@pytest.mark.parametrize("key", ["pcm_start", "pcm_dup"])
def test_positions_on_the_golden_excerpts(key):
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_11025hz_excerpts.npz"))
    x = z[key].astype(np.float32)
    _, st = oracle.decode_steps(x, 11025)
    pos, cref = oracle.find_sync(st["filtered"], 12480, want_corr=True)
    assert np.array_equal(so.positions(cref, 12480), pos)
    assert np.array_equal(so.positions(so.correlation(st["filtered"], 3), 12480), pos)
    if key == "pcm_dup":
        assert np.any(np.diff(pos.astype(np.int64)) == 0)


def test_tile_widths():
    assert [so.tile_width(pw) for pw in (3, 4, 5)] == [1920, 1888, 1856]
    for pw in (3, 4, 5):
        w = so.tile_width(pw)
        # the tile's correlation needs W + 36 PW + 2 PW - 1 low-passed samples of the 32 x 64 it stages
        assert w % 32 == 0 and w + 38 * pw - 1 <= 32 * so.REC_TB < w + 32 + 38 * pw - 1


@pytest.mark.parametrize("rate,profile", CASES, ids=IDS)
def test_input_length_search(rate, profile):
    s = na.Settings.profile(profile)
    nw = 10 * 2080 * so.pixel_width(s.work_rate) + 777
    n = so.input_len_for(nw, rate, s)
    if n is not None:
        assert so.work_len(n, rate, s) == nw and so.work_len(n - 1, rate, s) < nw
    _, st = oracle.decode_steps(synth.apt_signal(rate, 12, seed=1)[: rate * 11], rate,
                                _oracle_settings(s))
    assert so.work_len(rate * 11, rate, s) == st["demodulated"].size


def _oracle_settings(s):
    o = oracle.default_settings()
    for k in ("work_rate", "resample_atten", "resample_delta_freq", "resample_cutout", "demodulation_atten"):
        setattr(o, k, getattr(s, k))
    return o
