"""wav.rs (load_wav / write_wav) and resample.rs (the WAV -> WAV resample tool) over the C ABI."""
import ctypes as C
import os

import numpy as np

from . import _lib
from .err import raise_for


def info(path):
    wi = _lib.CWavInfo()
    raise_for(_lib.load().apt_wav_info_read(os.fsencode(path), C.byref(wi)))
    return {"sample_rate": wi.sample_rate, "channels": wi.channels, "bits_per_sample": wi.bits_per_sample,
            "is_float": bool(wi.is_float), "frames": int(wi.frames)}


def load_wav(path):
    """wav.rs:11-56 -> (Signal of channel 0 as f32, sample rate)"""
    i = info(path)
    out = np.empty(max(i["frames"], 1), dtype=np.float32)
    n, rate = C.c_uint64(0), C.c_uint32(0)
    raise_for(_lib.load().apt_wav_load(os.fsencode(path), out.ctypes.data, out.size, C.byref(n), C.byref(rate)))
    return out[: n.value], rate.value


def load_wav_pcm16(path):
    """The file's 16-bit samples (channel 0) as they are -- input of decode(..., int16) / apt_decode_pcm16."""
    i = info(path)
    out = np.empty(max(i["frames"], 1), dtype=np.int16)
    n, rate = C.c_uint64(0), C.c_uint32(0)
    raise_for(_lib.load().apt_wav_load_pcm16(os.fsencode(path), out.ctypes.data, out.size, C.byref(n), C.byref(rate)))
    return out[: n.value], rate.value


def load_iq(path):
    """A 2-channel 16-bit PCM WAV (SDR# / SDR++ baseband) -> (interleaved int16 I/Q, sample rate); input of iq.decode_iq."""
    i = info(path)
    out = np.empty(max(2 * i["frames"], 2), dtype=np.int16)
    n, rate = C.c_uint64(0), C.c_uint32(0)
    raise_for(_lib.load().apt_wav_load_iq16(os.fsencode(path), out.ctypes.data, out.size, C.byref(n), C.byref(rate)))
    return out[: 2 * n.value], rate.value


def write_wav_i16(path, samples, rate):
    x = np.ascontiguousarray(samples, dtype=np.int16)
    raise_for(_lib.load().apt_wav_write_i16(os.fsencode(path), x.ctypes.data, x.size, int(rate)))


def quantize_i16(signal):
    """wav.rs:71-85 on the device: (x / max * 32767) as i16"""
    x = np.ascontiguousarray(signal, dtype=np.float32)
    out = np.empty(x.size, dtype=np.int16)
    raise_for(_lib.load().apt_quantize_i16(x.ctypes.data, x.size, out.ctypes.data))
    return out


def resample_wav(input_path, output_path, output_rate, atten=40.0, delta_w_pi=0.1):
    """resample.rs:17-71 (defaults: default_settings.toml wav_resample_atten / wav_resample_delta_freq)"""
    n = C.c_uint64(0)
    raise_for(_lib.load().apt_resample_wav(os.fsencode(input_path), os.fsencode(output_path), int(output_rate), float(atten),
                                           float(delta_w_pi), C.byref(n)))
    return n.value
