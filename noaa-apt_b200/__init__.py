"""noaa-apt_b200 -- H100-native APT decode path behind the reference's own surface.

Mirrors the module layout of martinber/noaa-apt's hot path:

    noaa_apt_b200.decode(context, settings, signal, input_rate, sync)   # noaa_apt::decode
    noaa_apt_b200.dsp.{resample_with_filter, resample, demodulate, filter, Freq, Rate}
    noaa_apt_b200.filters.{NoFilter, Lowpass, LowpassDcRemoval}
    noaa_apt_b200.Context, noaa_apt_b200.Settings, noaa_apt_b200.err

Every compute call goes through the C ABI of libaptb200.so (include/aptb200.h) into hand-written
sm_90a CUDA kernels.  There is no CPU path: importing works anywhere, computing needs a GPU.
"""
from . import _lib, config, context, dsp, err, filters, frequency, image, iq, passes, wav  # noqa: F401
from . import decode as _decode_mod
from .config import Settings
from .context import Context
from .decode import (CARRIER_FREQ, FINAL_RATE, PX_PER_ROW, Decoder, Stream, decode, decode_batch, decode_len_bound,
                     find_sync, generate_sync_frame, stream_geometry, stream_geometry_iq)
from .frequency import Freq, Rate
from .iq import Carrier, decode_iq_auto, decode_iq_channels, find_carriers, spectrum
from .passes import IqWatch, Pass, PassTracker, Recording, Watch, decode_passes_png, find_passes_quality

__all__ = ["decode", "decode_batch", "decode_len_bound", "find_sync", "generate_sync_frame", "Decoder", "Stream",
           "stream_geometry", "stream_geometry_iq", "spectrum", "find_carriers", "decode_iq_channels", "decode_iq_auto",
           "Carrier", "Recording", "Pass", "find_passes_quality", "decode_passes_png", "PassTracker", "Watch", "IqWatch",
           "Settings", "Context", "Freq", "Rate", "dsp", "filters", "err", "config", "frequency", "image", "iq", "passes", "wav",
           "FINAL_RATE", "PX_PER_ROW", "CARRIER_FREQ"]


def library_path():
    return _lib.LIB_PATH


def device_count():
    return _lib.load().apt_device_count()
