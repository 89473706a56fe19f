"""apt_stream on the GPU: rows, sync positions and status of any split of a recording into pushes equal apt_decode's on
the whole recording, bit for bit; rows leave as the emission rule says; device memory stays what create allocated."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, synth
from noaa_apt_b200.err import Error as AptError
import oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_PUSH = 24000


def settings(profile):
    return na.Settings() if profile == "standard" else na.Settings.profile(profile)


def schedules(n, rate, seed=0):
    rng = np.random.default_rng(seed)
    out = {"one": [n], "fixed4800": [4800] * (n // 4800) + ([n % 4800] if n % 4800 else [])}
    sizes, t = [], 0
    while t < n:
        k = int(min(n - t, rng.integers(1, 3 * MAX_PUSH + 1)))
        sizes.append(k)
        t += k
    out["random"] = sizes
    sizes, t = [], 0
    while t < min(n, 2 * rate):    # 1-7-sample pushes over the first 2 s, then large ones
        k = int(min(n - t, rng.integers(1, 8)))
        sizes.append(k)
        t += k
    while t < n:
        k = min(n - t, 5 * MAX_PUSH)
        sizes.append(k)
        t += k
    out["tiny_then_large"] = sizes
    return out


def reference(x, rate, s, sync):
    """rows, positions and status of apt_decode on the whole recording."""
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        try:
            rows = dec.decode(x, sync=sync)
            st = _lib.OK
        except AptError as e:
            rows, st = None, e.code
        pos = dec.last_sync() if sync and st == _lib.OK else None
    return rows, pos, st


def run_stream(stream, pieces):
    got = [stream.push(p) for p in pieces]
    try:
        got.append(stream.finish())
        st = _lib.OK
    except AptError as e:
        st = e.code
    return np.concatenate(got).ravel() if got else np.zeros(0, np.float32), stream.positions(), st


def split(x, sizes, fmt="f32"):
    pieces, t = [], 0
    for i, k in enumerate(sizes):
        p = x[t:t + k]
        if fmt == "pcm16" or (fmt == "mixed" and i % 2):
            p = p.astype(np.int16)
        pieces.append(p)
        t += k
    return pieces


def check_equal(x, rate, s, sync, fmt="f32", which=None, max_push=MAX_PUSH):
    xin = x.astype(np.int16) if fmt == "pcm16" else x
    ref, pos, st = reference(xin, rate, s, sync)
    with na.Stream(rate, s, sync=sync, max_push=max_push) as strm:
        bytes0 = strm.info()["device_bytes"]
        for name, sizes in schedules(x.size, rate).items():
            if which and name not in which:
                continue
            strm.reset()
            rows, spos, sst = run_stream(strm, split(x, sizes, fmt))
            assert sst == st, (name, sst, st)
            if st == _lib.OK:
                assert rows.size == ref.size, (name, rows.size, ref.size)
                assert np.array_equal(rows.view(np.uint32), ref.view(np.uint32)), name
                if sync:
                    assert np.array_equal(spos, pos), name
            assert strm.info()["device_bytes"] == bytes0
    return ref, pos


def apt(rate, seconds=20, seed=3):
    return synth.apt_pcm16(rate, seconds=seconds, seed=seed).astype(np.float32)


@pytest.mark.parametrize("rate", [48000, 96000, 11025, 24960])
@pytest.mark.parametrize("sync", [True, False])
def test_rates_all_schedules(rate, sync):
    check_equal(apt(rate), rate, na.Settings(), sync)


@pytest.mark.parametrize("rate,profile", [(48000, "fast"), (48000, "slow"), (11025, "fast"), (11025, "slow"),
                                          (24960, "slow"), (96000, "fast")])
@pytest.mark.parametrize("sync", [True, False])
def test_profiles(rate, profile, sync):
    check_equal(apt(rate, 16), rate, settings(profile), sync, which=("random", "tiny_then_large"))


@pytest.mark.parametrize("fmt", ["pcm16", "mixed"])
@pytest.mark.parametrize("rate", [48000, 11025, 24960])
def test_pcm16_and_mixed_pushes(rate, fmt):
    check_equal(apt(rate, 16), rate, na.Settings(), True, fmt=fmt, which=("fixed4800", "random"))


def test_generic_resampler():
    code = ("import numpy as np, sys; sys.path.insert(0, %r); import test_gpu_stream as t; "
            "t.check_equal(t.apt(48000, 16), 48000, t.na.Settings(), True, which=('random', 'tiny_then_large')); print('ok')"
            % os.path.join(ROOT, "tests"))
    env = dict(os.environ, APTB200_GENERIC_RESAMPLER="1")
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("rate", [48000, 11025, 24960])
def test_oracle(rate):
    x = apt(rate, 14)
    rows = run_stream(na.Stream(rate, sync=True, max_push=MAX_PUSH), split(x, [7777] * (x.size // 7777 + 1)))[0]
    ref = oracle.decode(x, rate)
    assert rows.shape == ref.shape
    assert float(np.max(np.abs(rows - ref))) / float(np.max(np.abs(ref))) <= 1e-5


@pytest.mark.parametrize("name", ["start", "dup"])
def test_golden_excerpts(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_11025hz_excerpts.npz"))
    pcm = z["pcm_" + name]
    ref, pos = check_equal(pcm.astype(np.float32), 11025, na.Settings(), True, which=("fixed4800", "random"))
    assert np.array_equal(pos.astype(np.int64), z["sync_" + name].astype(np.int64))


def test_emission_rule():
    rate = 48000
    x = apt(rate, 30)
    s = na.Settings()
    _, steps = oracle.decode_steps(x, rate)
    pos = steps["sync_pos"].astype(np.int64)
    wr, row = 12480, 6240
    G, D = 38 * 3, row * 8 // 10
    geom = na.stream_geometry(rate, s, True, MAX_PUSH)
    assert geom["latency_work"] <= D + G
    fu_out = 13 * 8 * 64   # generous bound on one first-stage unit (outputs)
    with na.Stream(rate, s, sync=True, max_push=MAX_PUSH) as strm:
        t, out = 0, 0
        while t < x.size:
            k = min(24000, x.size - t)
            out += strm.push(x[t:t + k]).shape[0]
            t += k
            inf = strm.info()
            wf = inf["work_final"]
            due = 0
            for k_ in range(pos.size - 1):
                if max(pos[k_] + row, pos[k_ + 1] + G) + inf["latency_work"] <= wf:
                    due = k_ + 1
                else:
                    break
            assert inf["rows_out"] == out >= due
            complete = (t * wr) // rate
            assert complete - wf <= fu_out + 64, (complete, wf)


def test_memory_constant_and_long():
    rate = 48000
    b60 = na.stream_geometry(rate, None, True, 48000)["device_bytes"]
    x = apt(rate, 3600, seed=5)
    ref, pos, st = reference(x, rate, na.Settings(), True)
    with na.Stream(rate, sync=True, max_push=48000) as strm:
        assert strm.info()["device_bytes"] == b60
        rows, spos, sst = run_stream(strm, split(x, [48000] * (x.size // 48000 + 1)))
        assert strm.info()["device_bytes"] == b60
    assert sst == st == _lib.OK
    assert np.array_equal(rows.view(np.uint32), ref.view(np.uint32))
    assert np.array_equal(spos, pos)


def fade_out(rate, before, fade, after):
    """APT, a carrier fading out (a rising correlation without roots: hundreds of duplicate sync positions), APT."""
    a = synth.apt_pcm16(rate, seconds=before, seed=6).astype(np.float32)
    n = rate * fade
    t = np.arange(n, dtype=np.float64) / rate
    carrier = (np.linspace(1.0, 0.01, n) * 12000 * np.sin(2 * np.pi * 2400 * t)).astype(np.float32)
    b = synth.apt_pcm16(rate, seconds=after, seed=7).astype(np.float32)
    return np.concatenate([a, carrier, b])


def test_silence_and_fade_out():
    rate = 48000
    check_equal(np.zeros(rate * 40, np.float32), rate, na.Settings(), True, which=("fixed4800", "random"))
    x = fade_out(rate, 10, 150, 10)
    ref, pos = check_equal(x, rate, na.Settings(), True, which=("fixed4800", "random"))
    assert np.max(np.unique(pos, return_counts=True)[1]) > 256   # a duplicate run longer than the run ring


@pytest.mark.parametrize("step", [1000, 11025])
def test_fade_out_small_pushes(step):
    """10 s of APT, a 200 s fade-out, 10 s of APT at 11 025 Hz: the duplicate run is pushed long before its rows are
    final; every push returns, memory stays, and the result is apt_decode's."""
    rate = 11025
    x = fade_out(rate, 10, 200, 10)
    ref, pos, st = reference(x, rate, na.Settings(), True)
    assert st == _lib.OK
    with na.Stream(rate, sync=True, max_push=MAX_PUSH) as strm:
        b0 = strm.info()["device_bytes"]
        rows, spos, sst = run_stream(strm, split(x, [step] * (x.size // step + 1)))
        assert strm.info()["device_bytes"] == b0
    assert sst == _lib.OK
    assert np.array_equal(rows.view(np.uint32), ref.view(np.uint32))
    assert np.array_equal(spos, pos)


def test_errors():
    rate = 48000
    s = na.Settings()
    with na.Stream(rate, s, sync=True, max_push=MAX_PUSH) as strm:
        strm.push(apt(rate, 2))
        with pytest.raises(AptError) as e:
            strm.finish()
        assert e.value.code == _lib.ERR_TOO_SHORT
        with pytest.raises(AptError) as e:
            strm.push(np.zeros(10, np.float32))
        assert e.value.code == _lib.ERR_BAD_ARG
        strm.reset()
        noise = (np.random.default_rng(1).standard_normal(rate * 12) * 3000).astype(np.float32)
        _, _, st = reference(noise, rate, s, True)
        assert run_stream(strm, [noise])[2] == st
        # APT_ERR_CAPACITY leaves the stream unchanged: the same push then succeeds
        strm.reset()
        x = apt(rate, 14)
        lib = _lib.load()
        import ctypes as C
        got = C.c_uint64(0)
        out = np.empty(2080, np.float32)
        rc = lib.apt_stream_push(strm._h, x.ctypes.data, _lib.F32, x.size, out.ctypes.data, 0, C.byref(got))
        assert rc == _lib.ERR_CAPACITY
        assert strm.info()["samples_in"] == 0
        rows, pos, st = run_stream(strm, [x])
        ref, rpos, rst = reference(x, rate, s, True)
        assert st == rst == _lib.OK and np.array_equal(rows.view(np.uint32), ref.view(np.uint32))


def test_concurrent_streams():
    rate = 48000
    xs = [apt(rate, 14, seed=i) for i in range(4)]
    refs = [reference(x, rate, na.Settings(), True) for x in xs]
    # round-robin on one thread
    strms = [na.Stream(rate, sync=True, max_push=MAX_PUSH) for _ in xs]
    outs = [[] for _ in xs]
    for t in range(0, xs[0].size, 9600):
        for i, x in enumerate(xs):
            if t < x.size:
                outs[i].append(strms[i].push(x[t:t + 9600]))
    for i, s_ in enumerate(strms):
        outs[i].append(s_.finish())
        got = np.concatenate(outs[i]).ravel()
        assert np.array_equal(got.view(np.uint32), refs[i][0].view(np.uint32))
        assert np.array_equal(s_.positions(), refs[i][1])
        s_.close()
    # one stream per thread
    res = [None] * 4

    def work(i):
        with na.Stream(rate, sync=True, max_push=MAX_PUSH) as s_:
            res[i] = run_stream(s_, split(xs[i], [12345] * (xs[i].size // 12345 + 1)))
    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t_ in th:
        t_.start()
    for t_ in th:
        t_.join()
    for i in range(4):
        assert np.array_equal(res[i][0].view(np.uint32), refs[i][0].view(np.uint32))
