"""CPU restatement of the averaged power spectrum behind finding carriers (k_spectrum / k_spectrum_finish,
DESIGN.md §10 "Finding carriers") and of the APT test's score, for the tests of apt_iq_spectrum and
apt_iq_find_carriers.  Test infrastructure only.

The kernel rounds every f32 operation on its own and fixes its summation order, so this restatement does the same
operations in the same order on float32 arrays and gives the device's result bit for bit:

  1. tables   -- angle 2*pi*t/N in double, window 0.5 - 0.5 cos, twiddle (cos, -sin), each rounded once to f32
  2. segments -- S = n // N whole segments, K = min(S, max_segments or 2048), segment k at floor(k S / K) * N
  3. load     -- cu8: f32(v) - 127.5; cs16: f32(v); cf32 as is; times the window, per component
  4. FFT      -- Stockham autosort: a radix-2 stage first when log2 N is odd, then radix-4 stages
  5. sums     -- |X|^2 = x*x + y*y of segment k added into slot k mod 256, in ascending k, each slot from 0
  6. finish   -- the slots added in slot order, fftshifted by (b + N/2) & (N - 1), divided by f32(K)

No np.sum / np.add.reduce (they add pairwise) and no float64 intermediates: every operation below is one elementwise
float32 operation, as on the device.
"""
import functools
import math

import numpy as np

F32 = np.float32
TWO_PI = 2 * math.pi
assert TWO_PI == 6.283185307179586      # kTwoPi of spectrum.cu

SLOTS = 256                             # kSpecSlots
MIN_NFFT, MAX_NFFT = 256, 16384
DEFAULT_SEGMENTS = 2048
BATCH = 256                             # segments transformed at once: K = 2048 at nfft 16384 fits in memory

APT_NFFT = 4096
APT_LO_HZ, APT_HI_HZ = 300.0, 4800.0


@functools.lru_cache(maxsize=None)
def tables(nfft):
    """(win, tw_re, tw_im), float32 arrays of nfft: math.cos / math.sin are the libm of std::cos / std::sin."""
    ang = [TWO_PI * t / nfft for t in range(nfft)]
    win = np.array([0.5 - 0.5 * math.cos(a) for a in ang], dtype=np.float64).astype(F32)
    twr = np.array([math.cos(a) for a in ang], dtype=np.float64).astype(F32)
    twi = np.array([-math.sin(a) for a in ang], dtype=np.float64).astype(F32)
    for a in (win, twr, twi):
        a.setflags(write=False)
    return win, twr, twi


def search_nfft(iq_rate):
    """make_search's default nfft: the smallest power of two from 256 to 16384 whose bins are at most 200 Hz wide."""
    n = MIN_NFFT
    while n < MAX_NFFT and iq_rate / n > 200.0:
        n *= 2
    return n


def segment_starts(n, nfft, max_segments=0):
    """(S, K, starts): the first sample of each of the K segments, in Python ints (the __int128 product)."""
    S = n // nfft
    K = min(S, max_segments or DEFAULT_SEGMENTS)
    return S, K, [(k * S // K) * nfft for k in range(K)]


def _pairs(iq):
    """(format, (n, 2) view of I and Q): uint8 is cu8, int16 cs16, complex64 or interleaved float32 cf32."""
    x = np.ascontiguousarray(iq)
    if x.dtype == np.complex64:
        x = x.view(F32)
    fmt = {np.dtype(np.uint8): "cu8", np.dtype(np.int16): "cs16", np.dtype(F32): "cf32"}.get(x.dtype)
    if fmt is None or x.size % 2:
        raise TypeError("I/Q must be interleaved uint8, int16 or float32, or complex64")
    return fmt, x.reshape(-1, 2)


def _load(fmt, raw):
    """iq_load: (B, N, 2) raw samples to float32."""
    if fmt == "cu8":
        return np.subtract(raw.astype(F32), F32(127.5))
    return raw.astype(F32)


def _cmul(ar, ai, br, bi):
    """cmul_rn: (ar br - ai bi, ar bi + ai br), every product and sum rounded to f32."""
    return ar * br - ai * bi, ar * bi + ai * br


def segment_power(re, im, nfft):
    """|X|^2 of the windowed FFT of each row of re + i im ((B, nfft) float32), in natural bin order."""
    win, twr, twi = tables(nfft)
    B, N = re.shape
    assert N == nfft and re.dtype == F32 and im.dtype == F32
    xr, xi = re * win, im * win
    q4 = N // 4
    Ns = 1
    if (N.bit_length() - 1) & 1:
        # y[2j] = x[j] + x[j + N/2], y[2j + 1] = x[j] - x[j + N/2]
        ar, ai, br, bi = xr[:, : N // 2], xi[:, : N // 2], xr[:, N // 2:], xi[:, N // 2:]
        xr = np.stack([ar + br, ar - br], axis=-1).reshape(B, N)
        xi = np.stack([ai + bi, ai - bi], axis=-1).reshape(B, N)
        Ns = 2
    while True:
        # butterfly j = g Ns + kk (kk = j mod Ns) takes x[j + r N/4]; its output r goes to g 4Ns + r Ns + kk
        G = q4 // Ns
        v = [(xr[:, r * q4:(r + 1) * q4].reshape(B, G, Ns), xi[:, r * q4:(r + 1) * q4].reshape(B, G, Ns))
             for r in range(4)]
        if Ns > 1:
            kk = np.arange(Ns)
            stride = N // (Ns * 4)
            for r in range(1, 4):
                t = r * kk * stride
                v[r] = _cmul(v[r][0], v[r][1], twr[t], twi[t])
        a0 = (v[0][0] + v[2][0], v[0][1] + v[2][1])
        a1 = (v[0][0] - v[2][0], v[0][1] - v[2][1])
        a2 = (v[1][0] + v[3][0], v[1][1] + v[3][1])
        d = (v[1][0] - v[3][0], v[1][1] - v[3][1])
        a3 = (d[1], -d[0])                          # -i (v1 - v3)
        y = [(a0[0] + a2[0], a0[1] + a2[1]), (a1[0] + a3[0], a1[1] + a3[1]),
             (a0[0] - a2[0], a0[1] - a2[1]), (a1[0] - a3[0], a1[1] - a3[1])]
        if Ns * 4 == N:                             # G == 1: output r of butterfly j is bin j + r N/4
            return np.concatenate([(yr * yr + yi * yi).reshape(B, q4) for yr, yi in y], axis=1)
        xr = np.stack([yr for yr, _ in y], axis=2).reshape(B, N)
        xi = np.stack([yi for _, yi in y], axis=2).reshape(B, N)
        Ns *= 4


def spectrum(iq, nfft, max_segments=0):
    """(psd, K): apt_iq_spectrum's fftshifted average of |X|^2 over the K segments, float32."""
    if not (MIN_NFFT <= nfft <= MAX_NFFT and nfft & (nfft - 1) == 0):
        raise ValueError(f"nfft {nfft} is not a power of two in [{MIN_NFFT}, {MAX_NFFT}]")
    fmt, raw = _pairs(iq)
    S, K, starts = segment_starts(raw.shape[0], nfft, max_segments)
    if K == 0:
        raise ValueError(f"{raw.shape[0]} samples hold no segment of {nfft}")
    slots = np.zeros((min(K, SLOTS), nfft), dtype=F32)
    for k0 in range(0, K, BATCH):                   # BATCH divides SLOTS: batch k0 fills slots 0 .. k1 - k0 - 1
        k1 = min(K, k0 + BATCH)
        idx = np.asarray(starts[k0:k1], dtype=np.int64)[:, None] + np.arange(nfft, dtype=np.int64)
        z = _load(fmt, raw[idx])
        s0 = k0 % SLOTS
        slots[s0:s0 + k1 - k0] += segment_power(z[..., 0], z[..., 1], nfft)
    total = slots[0].copy()
    for s in range(1, slots.shape[0]):
        total += slots[s]
    shift = (np.arange(nfft) + nfft // 2) & (nfft - 1)
    return total[shift] / F32(K), K


def apt_score(audio, audio_rate):
    """The APT test's score of demodulated audio (the window apt_test takes): the fraction of the power of the nfft-4096
    spectrum of audio + 0i (K = S) between 300 Hz and 4.8 kHz, summed in double in bin order; 0 when there is no
    segment or no power."""
    a = np.ascontiguousarray(audio, dtype=F32)
    S = a.size // APT_NFFT
    if S == 0:
        return F32(0)
    z = np.zeros(a.size, dtype=np.complex64)
    z.real = a
    h, _ = spectrum(z, APT_NFFT, S)
    inside = everything = 0.0
    for b in range(APT_NFFT):
        f = abs((b - APT_NFFT // 2) * audio_rate / APT_NFFT)
        everything += float(h[b])
        if APT_LO_HZ <= f <= APT_HI_HZ:
            inside += float(h[b])
    return F32(inside / everything) if everything > 0.0 else F32(0)
