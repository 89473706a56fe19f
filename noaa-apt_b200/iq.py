"""Decoding straight from SDR I/Q (DESIGN.md §10): FM demodulation on the device.

The format comes from the array's dtype:

    uint8      interleaved I, Q: rtl_sdr / librtlsdr (u - 127.5)
    int16      interleaved I, Q: the 16-bit baseband WAVs of SDR# and SDR++ (wav.load_iq)
    complex64  or interleaved float32: GQRX I/Q recordings, the GNU Radio file sink

    s = IqSettings(2_400_000, offset_hz=37_000)     # audio_rate 48 kHz, channel filter 22 kHz / 8 kHz / 40 dB
    audio = fm_demod(iq, s)                         # instantaneous frequency in Hz at s.audio_rate
    rows = decode_iq(iq, s)                         # == decode(None, None, audio, s.audio_rate); the audio stays on the GPU
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
