"""The exact first-stage inputs of _impulse.py, checked without a GPU.

- Which kernel and loop shape make_front picks for each representative input rate: a plan change that moves a rate to
  another kernel or shape fails here first, and the list must keep covering every shape the kernels branch on.
- The impulse trains keep their promises: at most two impulses per output window, every tap of the filter met by some
  output, the forced impulses present.
- The oracle's fast_resampling equals the index-arithmetic restatement bit for bit, for f32 and PCM16 input.
- The checks can fail: a zeroed small tap or swapped phases change the restated values, and a wrong previous sample at
  a tile boundary leaves the envelope bound.
"""
import numpy as np
import pytest

import __graft_entry__ as entry
import _impulse as imp
import oracle

IDS = [f"{r}-{p}" for r, p, *_ in imp.REPRESENTATIVES]


@pytest.fixture(scope="module", autouse=True)
def built():
    entry.build()


def choice(rate, profile):
    return imp.front_choice(rate, imp.settings(profile))


@pytest.mark.parametrize("rate,profile,kind,shape,groups,rows_per_copy", imp.REPRESENTATIVES, ids=IDS)
def test_kernel_choice(rate, profile, kind, shape, groups, rows_per_copy):
    c = choice(rate, profile)
    assert c["kind"] == kind
    assert c["shape"] == shape
    if kind == "tiled":
        t = c["info"]
        assert (t.groups, t.rows_per_copy) == (groups, rows_per_copy)
        assert c["unit_out"] * c["m"] == c["unit_in"] * c["l"]


def test_representatives_cover_every_branch():
    fixed = {(7, 1, 6, 2), (11, 11, 11, 1), (3, 0, 3, 2)}      # the shapes launch.cu unrolls
    tiled = [r for r in imp.REPRESENTATIVES if r[2] == "tiled"]
    shapes = {r[3] for r in tiled}
    assert fixed <= shapes
    runtime = shapes - fixed
    assert any(s[3] == 1 for s in runtime) and any(s[3] == 2 for s in runtime)
    assert any(0 < bb < ae < it for it, bb, ae, _ in runtime)
    assert {1, 3, 5, 13} <= {r[4] for r in tiled}
    assert {1, 2} == {r[5] for r in tiled}
    assert {"tiled", "uniform-tap", "phase-major", "generic", "decimate"} == {r[2] for r in imp.REPRESENTATIVES}


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("rate,profile", [r[:2] for r in imp.REPRESENTATIVES], ids=IDS)
def test_train_invariants(rate, profile, dtype):
    c = choice(rate, profile)
    l, m, h = c["l"], c["m"], c["taps"]
    x = imp.representative_train(c, dtype)
    n, w = x.size, imp.window(l, m, h.size)
    pos = np.flatnonzero(x)
    # values: +-2^e, e in 0..14, and -32768 for PCM16
    mag = np.abs(x[pos].astype(np.float64))
    allowed = {2.0 ** e for e in range(15)} | ({32768.0} if dtype == np.int16 else set())
    assert set(mag.tolist()) <= allowed
    # at most two impulses in any window of w samples, hence in any output window
    assert (pos[2:] - pos[:-2] >= w).all()
    ks, taps, _, count = imp.contributions(n, pos, l, m, h.size)
    assert np.bincount(ks, minlength=count).max() <= 2
    # every tap the filter can use meets an impulse at some output
    last = h.size - 1 if l == 1 else 2 * ((h.size - 1) // 2)
    nz = np.flatnonzero(h[: last + 1])
    assert np.setdiff1d(nz, np.unique(taps)).size == 0
    # the impulses every train has, and both sides of every unit boundary away from the ends
    force = imp.unit_force(n, c["unit_in"], w)
    assert {0, 1, n - 1}.issubset(pos.tolist()) and np.intersect1d(pos, [n - 4, n - 3, n - 2]).size == 1
    assert set(force) <= set(pos.tolist())
    if c["unit_in"]:
        assert len(force) >= 4


def test_train_rejects_three_forced_impulses_in_one_window():
    with pytest.raises(ValueError):
        imp.impulse_train(10000, 13, 50, 959, seed=0, force=(5000, 5010, 5020))


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("rate,profile", [r[:2] for r in imp.REPRESENTATIVES], ids=IDS)
def test_oracle_equals_restatement(rate, profile, dtype):
    s = imp.settings(profile)
    c = choice(rate, profile)
    x = imp.representative_train(c, dtype)
    xf = oracle.pcm16_to_f32(x) if dtype == np.int16 else x
    ref = oracle.resample_with_filter(xf, rate, s.work_rate, oracle.FILTER_LOWPASS_DC,
                                      oracle.freq_hz(s.resample_cutout, rate), s.resample_atten,
                                      oracle.freq_hz(s.resample_delta_freq, rate))
    got = imp.exact_resample(x, c["l"], c["m"], c["taps"])
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), np.flatnonzero(got != ref)[:8]
    assert np.count_nonzero(got) > got.size // 4


@pytest.mark.parametrize("rate,profile", [r[:2] for r in imp.REPRESENTATIVES], ids=IDS)
def test_restatement_sees_a_wrong_tap(rate, profile):
    c = choice(rate, profile)
    l, m, h = c["l"], c["m"], c["taps"]
    x = imp.representative_train(c)
    r = imp.exact_resample(x, l, m, h)
    last = h.size - 1 if l == 1 else 2 * ((h.size - 1) // 2)
    nz = np.flatnonzero(h[: last + 1])
    small = nz[np.argmin(np.abs(h[nz]))]
    dropped = h.copy()
    dropped[small] = 0
    assert not np.array_equal(imp.exact_resample(x, l, m, dropped), r), f"tap {small} ({h[small]:.3e})"
    swapped = h.copy()
    if l > 1:                                            # phase 0 and phase 1 of the polyphase filter trade taps
        k = min(swapped[0::l].size, swapped[1::l].size)
        swapped[0:k * l:l], swapped[1:k * l:l] = h[1:k * l:l], h[0:k * l:l]
    else:
        swapped[small], swapped[small ^ 1] = h[small ^ 1], h[small]
    assert not np.array_equal(imp.exact_resample(x, l, m, swapped), r)


@pytest.mark.parametrize("rate,profile", [r[:2] for r in imp.REPRESENTATIVES if r[2] != "generic" and r[2] != "decimate"],
                         ids=[i for i, r in zip(IDS, imp.REPRESENTATIVES) if r[2] not in ("generic", "decimate")])
def test_envelope_bound_sees_a_wrong_previous_sample(rate, profile):
    s = imp.settings(profile)
    c = choice(rate, profile)
    r = imp.exact_resample(imp.representative_train(c), c["l"], c["m"], c["taps"])
    e = oracle.demodulate(r, oracle.freq_hz(imp.CARRIER_HZ, s.work_rate))
    assert imp.envelope_misses(e, r, s.work_rate).size == 0
    carrier = oracle.freq_hz(imp.CARRIER_HZ, s.work_rate)
    bounds = np.arange(c["unit_out"], r.size, c["unit_out"])
    shifted = e.copy()
    for k in bounds:                                     # each unit's first output paired with r[k-2] instead of r[k-1]
        shifted[k] = oracle.demodulate(np.array([r[k - 2], r[k]], np.float32), carrier)[1]
    want = [int(k) for k in bounds if r[k - 2] != r[k - 1]]
    assert len(want) >= 2
    assert set(want) <= set(imp.envelope_misses(shifted, r, s.work_rate).tolist())
    # and output 0 must be exactly 0
    e0 = e.copy()
    e0[0] = np.float32(1e-30)
    assert 0 in imp.envelope_misses(e0, r, s.work_rate)
