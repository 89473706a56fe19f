"""Deterministic synthetic NOAA APT recordings (2.4 kHz AM sub-carrier).

Used by the tests and by bench.py to build the workloads BASELINE.json names
(there are no recordings on the GPU box and no network).  The line layout
follows the constants of the reference (decode.rs:16-35: sync 39 px, space 47,
image 909, telemetry 45, two channels = 2080 px at 4160 px/s) and the sync-A
pattern of `generate_sync_frame` (decode.rs:188-198) at 1-px resolution.

Samples are quantised to int16 and handed out either as int16 (what a WAV
holds) or as the f32 cast `wav::load_wav` performs (wav.rs:37) -- raw integer
values, not normalised.  Gaussian noise from a counter-based generator
(numpy Philox, keyed by the seed) is mandatory: a clean signal has exact
correlation ties that the sync picker resolves by first-wins (decode.rs:250).
"""
import numpy as np

PX_PER_ROW = 2080
FINAL_RATE = 4160
CARRIER_HZ = 2400.0
_WEDGES = np.array([31, 63, 95, 127, 159, 191, 224, 255, 0, 60, 120, 180, 90, 150, 210, 30], dtype=np.float64)


def _sync_a():
    # 2 low, 7 x (2 low, 2 high), 8 low = 38 px, +1 low px to fill PX_SYNC_FRAME = 39
    px = [0, 0]
    for _ in range(7):
        px += [0, 0, 1, 1]
    px += [0] * 8 + [0]
    return np.array(px, dtype=np.float64) * 255.0


def _sync_b():
    # 7 pulses at 832 Hz => 5-px period (3 high, 2 low), padded with low px to 39
    px = [0, 0, 0, 0]
    for _ in range(7):
        px += [1, 1, 1, 0, 0]
    return np.array(px[:39] + [0] * max(0, 39 - len(px)), dtype=np.float64) * 255.0


_SYNC_A = _sync_a()
_SYNC_B = _sync_b()


def _row_template(seed):
    """Column-only part of a row: sync + space; image/telemetry filled per line."""
    t = np.zeros(PX_PER_ROW, dtype=np.float64)
    t[0:39] = _SYNC_A
    t[39:86] = 8.0          # space A (dark)
    t[1040:1079] = _SYNC_B
    t[1079:1126] = 245.0    # space B (bright)
    return t


def pixels(line, col, seed):
    """Pixel value 0..255 for (line, col) arrays of equal shape (vectorised)."""
    line = np.asarray(line)
    col = np.asarray(col)
    tmpl = _row_template(seed)
    out = tmpl[col]
    ph = 0.37 * (seed % 97)
    # image A: cols 86..994, image B: cols 1126..2034
    in_a = (col >= 86) & (col < 995)
    in_b = (col >= 1126) & (col < 2035)
    ca = col - 86
    cb = col - 1126
    img_a = 127.5 + 70.0 * np.sin(ca / 57.0 + ph) * np.cos(line / 83.0 + 0.5 * ph) \
        + 40.0 * np.sin((ca + 2.0 * line) / 19.0)
    img_b = 127.5 + 85.0 * np.cos(cb / 41.0 - ph) * np.sin(line / 61.0 + ph) \
        + 25.0 * np.cos((cb - line) / 13.0)
    out = np.where(in_a, img_a, out)
    out = np.where(in_b, img_b, out)
    # telemetry: 16 wedges of 8 lines each (telemetry.rs:129-133)
    wedge = _WEDGES[(line // 8) % 16]
    in_t = ((col >= 995) & (col < 1040)) | (col >= 2035)
    out = np.where(in_t, wedge, out)
    return np.clip(out, 0.0, 255.0)


def apt_pcm16(rate_hz, seconds=None, seed=0, n_samples=None, start=0, amplitude=20000.0,
              noise_sigma=200.0, chunk=1 << 22):
    """int16 samples [start, start + n) of the synthetic recording `seed` at `rate_hz`."""
    if n_samples is None:
        n_samples = int(round(rate_hz * seconds))
    out = np.empty(n_samples, dtype=np.int16)
    theta = 0.1 + 0.01 * (seed % 50)
    done = 0
    while done < n_samples:
        m = min(chunk - (start + done) % chunk, n_samples - done)
        n = np.arange(start + done, start + done + m, dtype=np.int64)
        pix = (n * FINAL_RATE) // rate_hz
        line = pix // PX_PER_ROW
        col = pix % PX_PER_ROW
        px = pixels(line, col, seed)
        # phase kept small: (n mod rate) keeps the argument exact in f64
        phase = 2.0 * np.pi * CARRIER_HZ * ((n % rate_hz).astype(np.float64) / rate_hz) + theta
        env = amplitude * (0.05 + 0.87 * px / 255.0)
        # counter-based noise: one Philox stream per (seed, chunk index) so any
        # [start, start+n) slice aligned to `chunk` reproduces the same samples
        rng = np.random.Generator(np.random.Philox(key=[0xA97 + seed, (start + done) // chunk]))
        skip = (start + done) % chunk
        noise = rng.standard_normal(skip + m)[skip:] * noise_sigma if noise_sigma > 0 else 0.0
        v = np.rint(env * np.sin(phase) + noise)
        out[done:done + m] = np.clip(v, -32768, 32767).astype(np.int16)
        done += m
    return out


def apt_signal(rate_hz, seconds=None, seed=0, **kw):
    """The same recording as the f32 `Signal` wav::load_wav would return (wav.rs:37)."""
    return apt_pcm16(rate_hz, seconds, seed, **kw).astype(np.float32)


_IQ_SCALE = {"cu8": 100.0, "cs16": 20000.0, "cf32": 1.0}


def apt_iq(iq_rate, seconds=None, seed=0, offset_hz=0, deviation_hz=17000.0, fmt="cu8", n_samples=None,
           noise_rel=0.03, audio_amplitude=20000.0, chunk=1 << 22):
    """The synthetic APT audio of `seed` (apt_pcm16 at iq_rate, no audio noise) FM-modulated onto a carrier at offset_hz:
    instantaneous frequency offset_hz + deviation_hz * audio / audio_amplitude, phase accumulated in float64 and carried
    across generation chunks, complex Gaussian noise of noise_rel times the carrier amplitude (counter-based, keyed by the
    seed), quantised to `fmt`: "cu8" (interleaved uint8 around 127.5), "cs16" (interleaved int16) or "cf32" (complex64)."""
    if n_samples is None:
        n_samples = int(round(iq_rate * seconds))
    scale = _IQ_SCALE[fmt]
    out = np.empty(n_samples, dtype=np.complex128)
    phase = 0.3 + 0.1 * (seed % 17)
    done = 0
    while done < n_samples:
        m = min(chunk, n_samples - done)
        audio = apt_pcm16(iq_rate, seed=seed, n_samples=m, start=done, noise_sigma=0.0, chunk=chunk).astype(np.float64)
        inc = 2.0 * np.pi * (offset_hz + deviation_hz * audio / audio_amplitude) / iq_rate
        ph = phase + np.cumsum(inc) - inc        # phase of sample k: sum of the increments before it
        phase = ph[-1] + inc[-1]
        rng = np.random.Generator(np.random.Philox(key=[0x1B5 + seed, done // chunk]))
        noise = rng.standard_normal((2, m)) * noise_rel if noise_rel > 0 else np.zeros((2, m))
        out[done:done + m] = np.exp(1j * ph) + (noise[0] + 1j * noise[1])
        done += m
    if fmt == "cf32":
        return out.astype(np.complex64)
    inter = np.empty(2 * n_samples, dtype=np.float64)
    inter[0::2], inter[1::2] = out.real * scale, out.imag * scale
    if fmt == "cu8":
        return np.clip(np.rint(inter + 127.5), 0, 255).astype(np.uint8)
    return np.clip(np.rint(inter), -32768, 32767).astype(np.int16)


_BLOCK = 1 << 16   # noise block of apt_iq_multi: sample i comes from block i // _BLOCK, whatever the chunk size


def _noise_blocks(key, a, b):
    """Complex standard Gaussian noise (each part N(0, 1)) for absolute sample indices [a, b), a >= 0: counter-based,
    one Philox stream per (key, block), so any slice is the same numbers."""
    out = np.empty(b - a, dtype=np.complex128)
    i = a
    while i < b:
        blk = i // _BLOCK
        lo, hi = i - blk * _BLOCK, min(b - blk * _BLOCK, _BLOCK)
        v = np.random.Generator(np.random.Philox(key=[key, blk])).standard_normal((2, _BLOCK))
        out[i - a:i - a + hi - lo] = v[0, lo:hi] + 1j * v[1, lo:hi]
        i += hi - lo
    return out


def _band_taps(width_hz, iq_rate, ntaps=255):
    """Hann-windowed sinc low-pass with cut-off width_hz / 2: the shape of an extra band."""
    k = np.arange(ntaps) - (ntaps - 1) / 2
    fc = 0.5 * width_hz / iq_rate
    return 2 * fc * np.sinc(2 * fc * k) * np.hanning(ntaps + 2)[1:-1]


def apt_iq_multi(iq_rate, seconds=None, carriers=((0, 0, 0.0, None, 60.0),), extra_bands=(), fmt="cu8", noise_rel=0.03,
                 n_samples=None, deviation_hz=17000.0, audio_amplitude=20000.0, chunk=1 << 22):
    """Several signals in one synthetic I/Q recording, as an SDR tuned near 137 MHz sees them.

    carriers: (offset_hz, seed, doppler_hz, tca_s, width_s) per APT carrier of amplitude 1, FM-modulated like apt_iq by the
      audio of `seed`, whose carrier frequency is offset_hz + doppler_hz * -(t - tca) / sqrt((t - tca)^2 + width^2), the
      shape of a pass with its closest approach at tca_s (None: the middle of the recording).
    extra_bands: (offset_hz, width_hz, rel_power) per band of Gaussian noise width_hz wide centred at offset_hz, of power
      rel_power relative to a carrier (an LRPT-like wideband signal).
    Complex Gaussian noise of noise_rel per part is added and the sum quantised to `fmt` as apt_iq does, scaled down by the
    number of signals.  Every sample is a function of its index alone (the audio phase is an exact integer running sum,
    the Doppler phase its closed-form integral, the noise counter-based per fixed block), so the output does not depend
    on `chunk`."""
    if n_samples is None:
        n_samples = int(round(iq_rate * seconds))
    nsig = len(carriers) + len(extra_bands)
    scale = _IQ_SCALE[fmt] / max(nsig, 1)
    out = np.empty(n_samples, dtype=np.complex128)
    acc = [0] * len(carriers)                 # running sum of each carrier's int16 audio before the chunk
    bands = [(_band_taps(w, iq_rate), off, p) for off, w, p in extra_bands]
    done = 0
    while done < n_samples:
        m = min(chunk, n_samples - done)
        idx = np.arange(done, done + m, dtype=np.int64)
        t = idx / float(iq_rate)
        y = np.zeros(m, dtype=np.complex128)
        for c, (off, seed, dop, tca, width) in enumerate(carriers):
            tca = 0.5 * n_samples / iq_rate if tca is None else tca
            audio = apt_pcm16(iq_rate, seed=seed, n_samples=m, start=done, noise_sigma=0.0, chunk=chunk).astype(np.int64)
            s_audio = acc[c] + np.cumsum(audio) - audio
            acc[c] += int(audio.sum())
            ph = (0.3 + 0.1 * (seed % 17)
                  + 2.0 * np.pi * ((idx * int(off)) % iq_rate).astype(np.float64) / iq_rate
                  + 2.0 * np.pi * deviation_hz / (audio_amplitude * iq_rate) * s_audio.astype(np.float64)
                  - 2.0 * np.pi * dop * (np.sqrt((t - tca) ** 2 + width ** 2) - np.sqrt(tca ** 2 + width ** 2)))
            y += np.exp(1j * ph)
        for b, (h, off, p) in enumerate(bands):
            raw = _noise_blocks(0x3D1 + b, done, done + m + h.size - 1)
            shaped = np.convolve(raw, h, mode="valid") * np.sqrt(p / (2.0 * np.sum(h * h)))
            y += shaped * np.exp(2j * np.pi * ((idx * int(off)) % iq_rate).astype(np.float64) / iq_rate)
        if noise_rel > 0:
            y += _noise_blocks(0x2C7, done, done + m) * noise_rel
        out[done:done + m] = y
        done += m
    if fmt == "cf32":
        return (out * scale).astype(np.complex64)
    inter = np.empty(2 * n_samples, dtype=np.float64)
    inter[0::2], inter[1::2] = out.real * scale, out.imag * scale
    if fmt == "cu8":
        return np.clip(np.rint(inter + 127.5), 0, 255).astype(np.uint8)
    return np.clip(np.rint(inter), -32768, 32767).astype(np.int16)


def _iq_pass_spans(iq_rate, passes):
    return [(int(off), int(seed), int(round(on * iq_rate)), int(round(off_s * iq_rate))) for off, seed, on, off_s in passes]


def apt_iq_passes_truth(iq_rate, passes, fade_s=10.0):
    """(offset_hz, fade-in midpoint, fade-out midpoint) in I/Q samples of every pass of apt_iq_passes."""
    h = int(round(0.5 * fade_s * iq_rate))
    return [(off, a + h, b - h) for off, _seed, a, b in _iq_pass_spans(iq_rate, passes)]


def apt_iq_passes(iq_rate, seconds=None, passes=(), extra_bands=(), fmt="cu8", noise_rel=0.03, fade_s=10.0, n_samples=None,
                  deviation_hz=17000.0, audio_amplitude=20000.0, chunk=1 << 22):
    """A continuous I/Q feed of one SDR in which each satellite's carrier is on only during its own passes.

    passes: (offset_hz, seed, on_s, off_s) per pass: from on_s to off_s the carrier at offset_hz carries the APT audio of
      `seed` (from its first sample, FM-modulated as apt_iq_multi does), its amplitude rising linearly from 0 over the first
      fade_s seconds and falling to 0 over the last; outside, the carrier is off.  Passes may overlap in time.
    extra_bands, noise_rel, fmt: as apt_iq_multi (receiver noise everywhere, the sum scaled down by the number of distinct
      carrier offsets plus bands).  Every sample is a function of its index alone, so the output does not depend on `chunk`."""
    if n_samples is None:
        n_samples = int(round(iq_rate * seconds))
    spans = _iq_pass_spans(iq_rate, passes)
    nsig = len({off for off, _s, _a, _b in spans}) + len(extra_bands)
    scale = _IQ_SCALE[fmt] / max(nsig, 1)
    out = np.empty(n_samples, dtype=np.complex128)
    bands = [(_band_taps(w, iq_rate), off, p) for off, w, p in extra_bands]
    fade = max(fade_s * iq_rate, 1.0)
    acc = [0] * len(spans)                    # running sum of each pass's int16 audio before the chunk
    done = 0
    while done < n_samples:
        m = min(chunk, n_samples - done)
        idx = np.arange(done, done + m, dtype=np.int64)
        y = np.zeros(m, dtype=np.complex128)
        for p, (off, seed, a, b) in enumerate(spans):
            lo, hi = max(a, done), min(b, done + m)
            if lo >= hi:
                continue
            audio = apt_pcm16(iq_rate, seed=seed, n_samples=hi - lo, start=lo - a, noise_sigma=0.0, chunk=chunk).astype(np.int64)
            s_audio = acc[p] + np.cumsum(audio) - audio
            acc[p] += int(audio.sum())
            k = idx[lo - done:hi - done]
            rel = (k - a).astype(np.float64)
            gain = np.clip(np.minimum(rel / fade, (b - a - rel) / fade), 0.0, 1.0)
            ph = (0.3 + 0.1 * (seed % 17)
                  + 2.0 * np.pi * ((k * off) % iq_rate).astype(np.float64) / iq_rate
                  + 2.0 * np.pi * deviation_hz / (audio_amplitude * iq_rate) * s_audio.astype(np.float64))
            y[lo - done:hi - done] += gain * np.exp(1j * ph)
        for bi, (h, off, pw) in enumerate(bands):
            raw = _noise_blocks(0x3D1 + bi, done, done + m + h.size - 1)
            shaped = np.convolve(raw, h, mode="valid") * np.sqrt(pw / (2.0 * np.sum(h * h)))
            y += shaped * np.exp(2j * np.pi * ((idx * int(off)) % iq_rate).astype(np.float64) / iq_rate)
        if noise_rel > 0:
            y += _noise_blocks(0x2C7, done, done + m) * noise_rel
        out[done:done + m] = y
        done += m
    if fmt == "cf32":
        return (out * scale).astype(np.complex64)
    inter = np.empty(2 * n_samples, dtype=np.float64)
    inter[0::2], inter[1::2] = out.real * scale, out.imag * scale
    if fmt == "cu8":
        return np.clip(np.rint(inter + 127.5), 0, 255).astype(np.uint8)
    return np.clip(np.rint(inter), -32768, 32767).astype(np.int16)


def _real_noise(key, a, b):
    """Real standard Gaussian noise for absolute sample indices [a, b): one Philox stream per (key, block of _BLOCK)."""
    out = np.empty(b - a, dtype=np.float64)
    i = a
    while i < b:
        blk = i // _BLOCK
        lo, hi = i - blk * _BLOCK, min(b - blk * _BLOCK, _BLOCK)
        out[i - a:i - a + hi - lo] = np.random.Generator(np.random.Philox(key=[key, blk])).standard_normal(_BLOCK)[lo:hi]
        i += hi - lo
    return out


def _segments(rate_hz, layout):
    """[(kind, first sample, end sample, pass seed)] of a layout of (kind, seconds[, pass seed]) entries."""
    out, t = [], 0.0
    for entry in layout:
        kind, seconds = entry[0], float(entry[1])
        if kind not in ("noise", "silence", "pass"):
            raise ValueError(f"unknown segment kind {kind!r}")
        a, b = int(round(t * rate_hz)), int(round((t + seconds) * rate_hz))
        out.append((kind, a, b, int(entry[2]) if len(entry) > 2 else 0))
        t += seconds
    return out


def apt_passes_len(rate_hz, layout):
    return _segments(rate_hz, layout)[-1][2] if layout else 0


def apt_passes_truth(rate_hz, layout, fade_s=10.0):
    """(fade-in midpoint, fade-out midpoint) in samples of every "pass" segment of apt_passes."""
    h = int(round(0.5 * fade_s * rate_hz))
    return [(a + h, b - h) for kind, a, b, _ in _segments(rate_hz, layout) if kind == "pass"]


def apt_passes(rate_hz, layout, seed=0, start=0, n_samples=None, noise_sigma=2000.0, fade_s=10.0, amplitude=20000.0):
    """int16 samples [start, start + n) of a long recording made of segments, as a station recording all day sees it.

    layout: (kind, seconds) or ("pass", seconds, pass_seed) entries, one after the other:
      "noise"    Gaussian receiver noise of noise_sigma;
      "silence"  exact zeros (the receiver off or squelched);
      "pass"     the synthetic APT recording of pass_seed (apt_pcm16 without its own noise, from its first sample), its
                 amplitude rising linearly from 0 over the first fade_s seconds and falling to 0 over the last, over the
                 same receiver noise.
    Every sample depends only on its index, so any slice, and so a 96 kHz x 10 h recording generated chunk by chunk,
    gives the same numbers."""
    segs = _segments(rate_hz, layout)
    total = segs[-1][2] if segs else 0
    if n_samples is None:
        n_samples = total - start
    if start < 0 or start + n_samples > total:
        raise ValueError("slice outside the recording")
    out = np.zeros(n_samples, dtype=np.float64)
    fade = max(fade_s * rate_hz, 1.0)
    for kind, a, b, pseed in segs:
        lo, hi = max(a, start), min(b, start + n_samples)
        if lo >= hi or kind == "silence":
            continue
        x = _real_noise(0x5A7 + seed, lo, hi) * noise_sigma if noise_sigma > 0 else np.zeros(hi - lo)
        if kind == "pass":
            k = np.arange(lo - a, hi - a, dtype=np.float64)
            gain = np.clip(np.minimum(k / fade, (b - a - k) / fade), 0.0, 1.0)
            sig = apt_pcm16(rate_hz, seed=pseed, n_samples=hi - lo, start=lo - a, noise_sigma=0.0, amplitude=amplitude)
            x += gain * sig.astype(np.float64)
        out[lo - start:hi - start] = x
    return np.clip(np.rint(out), -32768, 32767).astype(np.int16)
