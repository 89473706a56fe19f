"""Decoding straight from SDR I/Q (DESIGN.md §10): FM demodulation on the device.

The format comes from the array's dtype:

    uint8      interleaved I, Q: rtl_sdr / librtlsdr (u - 127.5)
    int16      interleaved I, Q: the 16-bit baseband WAVs of SDR# and SDR++ (wav.load_iq)
    complex64  or interleaved float32: GQRX I/Q recordings, the GNU Radio file sink

    s = IqSettings(2_400_000, offset_hz=37_000)     # audio_rate 48 kHz, channel filter 22 kHz / 8 kHz / 40 dB
    audio = fm_demod(iq, s)                         # instantaneous frequency in Hz at s.audio_rate
    a0, a1 = fm_demod_channels(iq, s, [-400_000, 120_000])   # several channels, one launch per chunk
    rows = decode_iq(iq, s)                         # == decode(None, None, audio, s.audio_rate); the audio stays on the GPU

Without knowing where the carriers are (DESIGN.md §10, "Finding carriers"):

    freqs, psd = spectrum(iq, 2_400_000)            # averaged Hann-windowed power spectrum, fftshifted
    found = find_carriers(iq, 2_400_000)            # [Carrier(offset_hz, centre_hz, snr_db, apt_score, is_apt), ...]
    carriers, rows = decode_iq_auto(iq, 2_400_000)  # every APT carrier decoded from one upload of the recording
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib
from .config import Settings
from .err import raise_for


@dataclass
class IqSettings:
    """apt_iq_settings.  audio_rate / cutout / delta_freq / atten left as None take apt_iq_default_settings' values."""
    iq_rate: int
    offset_hz: int = 0
    audio_rate: int = None
    cutout: float = None
    delta_freq: float = None
    atten: float = None

    def to_c(self):
        c = _lib.CIqSettings()
        st = _lib.load().apt_iq_default_settings(int(self.iq_rate), int(self.offset_hz), C.byref(c))
        if st != _lib.OK and self.audio_rate is None:
            raise_for(st)   # no default audio rate for this iq_rate
        for name in ("audio_rate", "cutout", "delta_freq", "atten"):
            v = getattr(self, name)
            if v is not None:
                setattr(c, name, v)
        c.iq_rate = int(self.iq_rate)
        c.offset_hz = int(self.offset_hz)
        return c

    def __post_init__(self):
        c = self.to_c()
        for name in ("audio_rate", "cutout", "delta_freq", "atten"):
            if getattr(self, name) is None:
                setattr(self, name, getattr(c, name))

    @property
    def decimation(self):
        return self.iq_rate // self.audio_rate


def iq_format(iq):
    """(contiguous array, apt_sample_format, complex sample count) of an I/Q array."""
    x = np.ascontiguousarray(iq)
    if x.dtype == np.complex64:
        return x, _lib.CF32, x.size
    fmt = {np.dtype(np.uint8): _lib.CU8, np.dtype(np.int16): _lib.CS16, np.dtype(np.float32): _lib.CF32}.get(x.dtype)
    if fmt is None:
        raise TypeError("I/Q must be interleaved uint8 (cu8), interleaved int16 (cs16), complex64 or interleaved float32 (cf32)")
    if x.size % 2:
        raise ValueError("interleaved I/Q needs an even number of values")
    return x, fmt, x.size // 2


def fm_demod_len(n, settings):
    out = C.c_uint64(0)
    raise_for(_lib.load().apt_fm_demod_len(int(n), C.byref(settings.to_c()), C.byref(out)))
    return out.value


def fm_demod(iq, settings):
    """The I/Q stage alone: ceil(n / D) f32 audio samples (Hz of deviation) at settings.audio_rate."""
    x, fmt, n = iq_format(iq)
    s = settings.to_c()
    out = np.empty(max(fm_demod_len(n, settings), 1), dtype=np.float32)
    got = C.c_uint64(0)
    raise_for(_lib.load().apt_fm_demod(x.ctypes.data, fmt, n, C.byref(s), out.ctypes.data, out.size, C.byref(got)))
    return out[: got.value].copy()


def _offsets(offsets):
    offs = [int(o) for o in offsets]
    return offs, (C.c_int32 * max(len(offs), 1))(*offs)


def fm_demod_channels(iq, iq_settings, offsets):
    """fm_demod at every offset of `offsets` (1..8 channels; iq_settings.offset_hz is ignored), demodulated together in one
    kernel launch per chunk: [audio of channel c], each equal to fm_demod with offset_hz = offsets[c], bit for bit."""
    x, fmt, n = iq_format(iq)
    s = iq_settings.to_c()
    s.offset_hz = 0   # ignored: the channels are `offsets`
    offs, c_offs = _offsets(offsets)
    na = C.c_uint64(0)
    raise_for(_lib.load().apt_fm_demod_len(n, C.byref(s), C.byref(na)))
    outs = [np.empty(max(na.value, 1), dtype=np.float32) for _ in offs]
    ptrs = (C.c_void_p * max(len(offs), 1))(*[o.ctypes.data for o in outs])
    got = C.c_uint64(0)
    raise_for(_lib.load().apt_fm_demod_channels(x.ctypes.data if n else None, fmt, n, C.byref(s), c_offs, len(offs), ptrs,
                                                na.value, C.byref(got)))
    return [o[: got.value].copy() for o in outs]


def decode_iq(iq, iq_settings, settings=None, sync=True, context=None):
    """noaa_apt::decode of the FM-demodulated I/Q at iq_settings.audio_rate, audio produced on the device."""
    lib = _lib.load()
    x, fmt, n = iq_format(iq)
    s = (settings or Settings()).to_c()
    qs = iq_settings.to_c()
    bound = C.c_uint64(0)
    raise_for(lib.apt_decode_len_bound(fm_demod_len(n, iq_settings), int(qs.audio_rate), C.byref(s), C.byref(bound)))
    out = np.empty(max(bound.value, 1), dtype=np.float32)
    got = C.c_uint64(0)

    def _cb(progress, desc, _user):
        if context is not None:
            context.status(progress, desc.decode())

    cb = _lib.STATUS_CB(_cb)
    raise_for(lib.apt_decode_iq(x.ctypes.data, fmt, n, C.byref(qs), C.byref(s), int(bool(sync)), out.ctypes.data, out.size,
                                C.byref(got), cb, None))
    return out[: got.value].copy()


@dataclass
class Carrier:
    """apt_carrier: a carrier found in the spectrum; offset_hz is ready for IqSettings.offset_hz."""
    offset_hz: int
    centre_hz: float
    snr_db: float
    apt_score: float
    is_apt: bool

    @classmethod
    def from_c(cls, c):
        return cls(int(c.offset_hz), float(c.centre_hz), float(c.snr_db), float(c.apt_score), bool(c.is_apt))


def spectrum(iq, iq_rate, nfft=16384, max_segments=2048):
    """(freqs, psd): the average of |FFT|^2 of Hann-windowed segments of nfft samples (at most max_segments of them,
    spread evenly over the recording), fftshifted, and each bin's frequency in Hz relative to the tuned centre."""
    x, fmt, n = iq_format(iq)
    ss = _lib.CSpectrumSettings(int(nfft), int(max_segments))
    psd = np.empty(int(nfft), dtype=np.float32)
    nseg = C.c_uint32(0)
    raise_for(_lib.load().apt_iq_spectrum(x.ctypes.data, fmt, n, int(iq_rate), C.byref(ss), psd.ctypes.data, psd.size,
                                          C.byref(nseg)))
    freqs = (np.arange(int(nfft), dtype=np.float64) - int(nfft) // 2) * (float(iq_rate) / int(nfft))
    return freqs, psd


def _search(lo, hi, nfft, max_segments, min_snr_db):
    if (lo is None) != (hi is None):
        raise ValueError("give both lo and hi, or neither")
    return _lib.CCarrierSearch(int(lo or 0), int(hi or 0), int(nfft), int(max_segments), float(min_snr_db))


def _iq_settings(iq_rate, iq_settings):
    if iq_settings is None:
        return IqSettings(int(iq_rate))
    if iq_rate is not None and int(iq_rate) != iq_settings.iq_rate:
        raise ValueError("iq_rate differs from iq_settings.iq_rate")
    return iq_settings


def find_carriers(iq, iq_rate=None, lo=None, hi=None, nfft=0, max_segments=0, min_snr_db=0.0, iq_settings=None,
                  max_carriers=64):
    """The carriers in an I/Q recording by descending SNR.  lo / hi: search window in Hz relative to the tuned centre
    (default: the whole usable band); zero nfft / max_segments / min_snr_db take the defaults (<= 200 Hz bins, 2048
    segments, 6 dB).  iq_settings (optional) gives the channel filter of the APT test."""
    x, fmt, n = iq_format(iq)
    s = _iq_settings(iq_rate, iq_settings).to_c()
    cs = _search(lo, hi, nfft, max_segments, min_snr_db)
    out = (_lib.CCarrier * max(int(max_carriers), 1))()
    count = C.c_uint32(0)
    raise_for(_lib.load().apt_iq_find_carriers(x.ctypes.data, fmt, n, C.byref(s), C.byref(cs), out, len(out),
                                               C.byref(count)))
    return [Carrier.from_c(out[i]) for i in range(count.value)]


def find_carriers_psd(psd, iq_rate, cutout=22000.0, lo=None, hi=None, min_snr_db=0.0, max_carriers=64):
    """The search of find_carriers on a spectrum in spectrum()'s order, on the host (no APT test: is_apt is False)."""
    p = np.ascontiguousarray(psd, dtype=np.float32)
    cs = _search(lo, hi, 0, 0, min_snr_db)
    out = (_lib.CCarrier * max(int(max_carriers), 1))()
    count = C.c_uint32(0)
    raise_for(_lib.load().apt_find_carriers_psd(p.ctypes.data, p.size, int(iq_rate), float(cutout), C.byref(cs), out,
                                                len(out), C.byref(count)))
    return [Carrier.from_c(out[i]) for i in range(count.value)]


def _row_buffers(lib, n, qs, s, count):
    q0 = _lib.CIqSettings(qs.iq_rate, qs.audio_rate, 0, qs.cutout, qs.delta_freq, qs.atten)
    na, bound = C.c_uint64(0), C.c_uint64(0)
    raise_for(lib.apt_fm_demod_len(int(n), C.byref(q0), C.byref(na)))
    raise_for(lib.apt_decode_len_bound(na.value, int(qs.audio_rate), C.byref(s), C.byref(bound)))
    bufs = [np.empty(max(bound.value, 1), dtype=np.float32) for _ in range(count)]
    return (bufs, (C.c_void_p * count)(*[b.ctypes.data for b in bufs]), (C.c_uint64 * count)(*[b.size for b in bufs]),
            (C.c_uint64 * count)(), (C.c_int * count)())


_BEFORE_DEVICE = (_lib.ERR_BAD_ARG, _lib.ERR_TOO_SHORT, _lib.ERR_WORK_RATE)


def decode_iq_channels(iq, iq_settings, offsets, settings=None, sync=True):
    """decode_iq at each offset in `offsets` (Hz), the recording uploaded once: (rows, statuses), rows[c] the image rows
    of channel c (empty when statuses[c] is not OK).  Raises for an error every channel shares (bad arguments, too short)."""
    lib = _lib.load()
    x, fmt, n = iq_format(iq)
    s = (settings or Settings()).to_c()
    qs = iq_settings.to_c()
    offs = [int(o) for o in offsets]
    k = len(offs)
    if k < 1:
        raise ValueError("give at least one offset")
    bufs, outs, caps, nouts, sts = _row_buffers(lib, n, qs, s, k)
    rc = lib.apt_decode_iq_channels(x.ctypes.data, fmt, n, C.byref(qs), (C.c_int32 * k)(*offs), k, C.byref(s),
                                    int(bool(sync)), outs, caps, nouts, sts)
    if rc in _BEFORE_DEVICE and all(sts[c] == rc for c in range(k)):
        raise_for(rc)
    return [bufs[c][: nouts[c]].copy() for c in range(k)], [int(sts[c]) for c in range(k)]


def decode_iq_auto(iq, iq_rate=None, settings=None, sync=True, lo=None, hi=None, nfft=0, max_segments=0, min_snr_db=0.0,
                   iq_settings=None, max_channels=8):
    """find_carriers, then decode_iq_channels on the APT carriers: (carriers, rows), rows[i] the image of carriers[i]
    (None if that channel failed to decode)."""
    lib = _lib.load()
    x, fmt, n = iq_format(iq)
    qset = _iq_settings(iq_rate, iq_settings)
    qs = qset.to_c()
    s = (settings or Settings()).to_c()
    cs = _search(lo, hi, nfft, max_segments, min_snr_db)
    k = max(int(max_channels), 1)
    bufs, outs, caps, nouts, sts = _row_buffers(lib, n, qs, s, k)
    found = (_lib.CCarrier * k)()
    nfound = C.c_uint32(0)
    rc = lib.apt_decode_iq_auto(x.ctypes.data, fmt, n, C.byref(qs), C.byref(cs), C.byref(s), int(bool(sync)), found, k,
                                C.byref(nfound), outs, caps, nouts, sts)
    m = nfound.value
    if rc != _lib.OK and (m == 0 or (rc in _BEFORE_DEVICE and all(sts[c] == rc for c in range(m)))):
        raise_for(rc)
    carriers = [Carrier.from_c(found[i]) for i in range(m)]
    rows = [bufs[i][: nouts[i]].copy() if sts[i] == _lib.OK else None for i in range(m)]
    return carriers, rows
