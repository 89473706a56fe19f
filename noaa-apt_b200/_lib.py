"""ctypes loader for libaptb200.so -- the C ABI declared in include/aptb200.h.

The library is the product.  If it has not been built this module raises: there
is no Python or CPU fallback for any compute entry point.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("APTB200_LIB") or os.path.join(HERE, "libaptb200.so")   # APTB200_LIB: an experimental build

OK = 0
ERR_RESAMPLE_TO_ZERO = 1
ERR_TOO_SHORT = 2
ERR_FEW_SYNC_FRAMES = 3
ERR_WORK_RATE = 4
ERR_RATE_OVERFLOW = 5
ERR_CUDA = 6
ERR_BAD_ARG = 7
ERR_NOMEM = 8
ERR_CAPACITY = 9
ERR_EMPTY_RESULT = 10
ERR_IO = 11

FILTER_NONE, FILTER_LOWPASS, FILTER_LOWPASS_DC = 0, 1, 2
F32, PCM16 = 0, 1
CU8, CF32, CS16 = 2, 3, 4   # I/Q formats (apt_fm_demod / apt_decode_iq only)


class CSettings(C.Structure):
    _fields_ = [
        ("work_rate", C.c_uint32),
        ("resample_atten", C.c_float),
        ("resample_delta_freq", C.c_float),
        ("resample_cutout", C.c_float),
        ("demodulation_atten", C.c_float),
    ]


class CFilter(C.Structure):
    _fields_ = [
        ("kind", C.c_int),
        ("cutout_pi", C.c_float),
        ("atten", C.c_float),
        ("delta_w_pi", C.c_float),
    ]


class CTileInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("usable", "groups", "p_out", "p_in", "usteps", "row_len", "rows_per_tile",
                                          "smem_bytes", "slices", "slice_stride", "half_taps", "shift", "iters",
                                          "group_stride", "ctas_per_sm", "pair_pitch", "halves", "rows_per_copy")]


class CUtInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("usable", "l", "m", "np", "q", "rows_per_block", "vec", "back", "chunks",
                                          "slot_floats", "slot_stride", "nslot", "warps", "smem_bytes", "nvec",
                                          "stream_b", "halo_u0", "halo_n", "chunk_len")] + [("cs", C.c_uint32 * 8), ("ce", C.c_uint32 * 8)]


class CImageInfo(C.Structure):
    _fields_ = [("low", C.c_float), ("high", C.c_float), ("rows", C.c_uint64), ("telemetry_row", C.c_uint64),
                ("wedges_a", C.c_float * 16), ("wedges_b", C.c_float * 16)]


CONTRAST_MINMAX, CONTRAST_PERCENT, CONTRAST_TELEMETRY, CONTRAST_HISTOGRAM = 0, 1, 2, 3


class CProcessSettings(C.Structure):
    _fields_ = [("contrast", C.c_int), ("percent", C.c_float), ("rotate", C.c_int), ("palette", C.c_void_p),
                ("tune", C.c_float * 4), ("rgba", C.c_int)]


class CWavInfo(C.Structure):
    _fields_ = [("sample_rate", C.c_uint32), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("is_float", C.c_uint32),
                ("frames", C.c_uint64)]


class CPhInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("usable", "l", "m", "j", "jpad", "pitch", "row_len", "smem_bytes")]


class CStreamInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("samples_in", "work_final", "rows_out", "peaks", "latency_work", "max_push",
                                          "device_bytes")]


class CIqSettings(C.Structure):
    _fields_ = [("iq_rate", C.c_uint32), ("audio_rate", C.c_uint32), ("offset_hz", C.c_int32), ("cutout", C.c_float),
                ("delta_freq", C.c_float), ("atten", C.c_float)]


class CSpectrumSettings(C.Structure):
    _fields_ = [("nfft", C.c_uint32), ("max_segments", C.c_uint32)]


class CCarrierSearch(C.Structure):
    _fields_ = [("lo_hz", C.c_int32), ("hi_hz", C.c_int32), ("nfft", C.c_uint32), ("max_segments", C.c_uint32),
                ("min_snr_db", C.c_float)]


class CCarrier(C.Structure):
    _fields_ = [("offset_hz", C.c_int32), ("centre_hz", C.c_float), ("snr_db", C.c_float), ("apt_score", C.c_float),
                ("is_apt", C.c_int)]


class CTrackSettings(C.Structure):
    _fields_ = [("delta", C.c_uint32), ("lambda_", C.c_float)]


class CPngSettings(C.Structure):
    _fields_ = [("filter", C.c_int), ("matches", C.c_int), ("block_bytes", C.c_uint32), ("rgb_from_rgba", C.c_int)]


class CPngGroupImage(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("stream_offset", "stream_bytes", "out_offset", "out_bytes", "bound")] + \
               [(n, C.c_uint32) for n in ("first_row", "first_span", "first_block", "blocks", "first_chunk", "pad")]


class CPngGroupInfo(C.Structure):
    _fields_ = [("stream_bytes", C.c_uint64), ("out_bytes", C.c_uint64)] + \
               [(n, C.c_uint32) for n in ("rows", "spans", "blocks", "chunks")]


class CPassSearch(C.Structure):
    _fields_ = [("enter", C.c_float), ("exit", C.c_float), ("max_gap_s", C.c_float), ("min_length_s", C.c_float)]


class CPass(C.Structure):
    _fields_ = [("start", C.c_uint64), ("end", C.c_uint64), ("first_window", C.c_uint64), ("windows", C.c_uint64),
                ("mean_quality", C.c_float), ("peak_quality", C.c_float)]


class CRecordingInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("samples", "work_samples", "windows", "device_bytes")] + \
               [("input_rate", C.c_uint32), ("row_samples", C.c_uint32)]


PASS_AOS, PASS_LOS, PASS_SEGMENT = 1, 2, 3


class CPassEvent(C.Structure):
    _fields_ = [("kind", C.c_int), ("window", C.c_uint64), ("pass_", CPass)]


class CWatchSettings(C.Structure):
    _fields_ = [("sync", C.c_int), ("search", CPassSearch), ("ps", C.c_void_p), ("png", C.c_void_p), ("max_rows", C.c_uint64),
                ("max_push", C.c_uint64)]


class CWatchEvent(C.Structure):
    _fields_ = [("ev", CPassEvent), ("index", C.c_uint32), ("status", C.c_int), ("rows", C.c_uint64), ("info", CImageInfo),
                ("data", C.c_void_p), ("bytes", C.c_uint64)]


class CWatchInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("samples_in", "segment_start", "windows", "passes", "open", "device_bytes",
                                          "max_push", "latency_windows")]


STATUS_CB = C.CFUNCTYPE(None, C.c_float, C.c_char_p, C.c_void_p)
WATCH_CB = C.CFUNCTYPE(None, C.POINTER(CWatchEvent), C.c_void_p)
WATCH_IQ_CB = C.CFUNCTYPE(None, C.c_int, C.POINTER(CWatchEvent), C.c_void_p)
WATCH_IQ_MAX_CHANNELS = 8

# name -> (restype, argtypes); every symbol include/aptb200.h declares.
_u64p = C.POINTER(C.c_uint64)
_szp = C.POINTER(C.c_size_t)

SYNC_PEAKS, SYNC_TRACK = 0, 1   # apt_sync_mode
SIGNATURES = {
    "apt_strerror": (C.c_char_p, [C.c_int]),
    "apt_last_error": (C.c_char_p, []),
    "apt_abi_version": (C.c_int, []),
    "apt_device_count": (C.c_int, []),
    "apt_default_settings": (None, [C.POINTER(CSettings)]),
    "apt_profile_settings": (C.c_int, [C.c_char_p, C.POINTER(CSettings)]),
    "apt_freq_hz": (C.c_float, [C.c_float, C.c_uint32]),
    "apt_bessel_i0": (C.c_float, [C.c_float]),
    "apt_filter_resample": (None, [C.POINTER(CFilter), C.c_uint32, C.c_uint32]),
    "apt_filter_design": (C.c_int, [C.POINTER(CFilter), C.c_void_p, C.c_size_t, _szp]),
    "apt_resample_len": (C.c_int, [C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(CFilter), _u64p]),
    "apt_resample_with_filter": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(CFilter),
                                           C.c_void_p, C.c_uint64, _u64p]),
    "apt_resample": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_float, C.c_float,
                               C.c_void_p, C.c_uint64, _u64p]),
    "apt_demodulate": (C.c_int, [C.c_void_p, C.c_uint64, C.c_float, C.c_void_p]),
    "apt_filter_signal": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(CFilter), C.c_void_p]),
    "apt_filter_taps": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "apt_generate_sync_frame": (C.c_int, [C.c_uint32, C.c_void_p, C.c_size_t, _szp]),
    "apt_find_sync": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t, _szp, C.c_void_p]),
    "apt_decode_len_bound": (C.c_int, [C.c_uint64, C.c_uint32, C.POINTER(CSettings), _u64p]),
    "apt_decode": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(CSettings), C.c_int,
                             C.c_void_p, C.c_uint64, _u64p, STATUS_CB, C.c_void_p]),
    "apt_decode_pcm16": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(CSettings), C.c_int,
                                   C.c_void_p, C.c_uint64, _u64p, STATUS_CB, C.c_void_p]),
    "apt_wav_info_read": (C.c_int, [C.c_char_p, C.POINTER(CWavInfo)]),
    "apt_wav_load": (C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64, _u64p, C.POINTER(C.c_uint32)]),
    "apt_wav_load_pcm16": (C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64, _u64p, C.POINTER(C.c_uint32)]),
    "apt_wav_write_i16": (C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64, C.c_uint32]),
    "apt_quantize_i16": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "apt_resample_wav": (C.c_int, [C.c_char_p, C.c_char_p, C.c_uint32, C.c_float, C.c_float, _u64p]),
    "apt_decode_image_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CSettings), C.c_int, C.c_int,
                                      C.c_float, C.c_void_p, C.c_uint64, _u64p, C.POINTER(CImageInfo), STATUS_CB, C.c_void_p]),
    "apt_map_signal_u8": (C.c_int, [C.c_void_p, C.c_uint64, C.c_float, C.c_float, C.c_void_p]),
    "apt_contrast_bounds": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_float, C.POINTER(CImageInfo)]),
    "apt_telemetry_rows": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "apt_process": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(CProcessSettings), C.c_void_p, C.c_uint64, _u64p,
                              C.POINTER(CImageInfo)]),
    "apt_decode_image": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CSettings), C.c_int,
                                   C.POINTER(CProcessSettings), C.c_void_p, C.c_uint64, _u64p, C.POINTER(CImageInfo),
                                   STATUS_CB, C.c_void_p]),
    "apt_decoder_set_image_mode": (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    "apt_decoder_set_process_mode": (C.c_int, [C.c_void_p, C.POINTER(CProcessSettings)]),
    "apt_decoder_image_info": (C.c_int, [C.c_void_p, C.POINTER(CImageInfo)]),
    "apt_default_track_settings": (None, [C.POINTER(CTrackSettings)]),
    "apt_decoder_set_sync_mode": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(CTrackSettings)]),
    "apt_decoder_create": (C.c_int, [C.c_int, C.c_uint32, C.POINTER(CSettings), C.c_uint64, C.POINTER(C.c_void_p)]),
    "apt_decoder_destroy": (None, [C.c_void_p]),
    "apt_decoder_submit_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64]),
    "apt_decoder_submit_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64]),
    "apt_decoder_poll": (C.c_int, [C.c_void_p]),
    "apt_cache_clear": (None, []),
    "apt_bind_thread_to_device": (C.c_int, [C.c_int]),
    "apt_decoder_wait": (C.c_int, [C.c_void_p, _u64p]),
    "apt_decoder_last_sync": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _szp]),
    "apt_decoder_last_counts": (C.c_int, [C.c_void_p, _u64p, _u64p, _u64p]),
    "apt_decoder_last_root_count": (C.c_int, [C.c_void_p, _u64p]),
    "apt_decoder_last_roots": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _szp]),
    "apt_decoder_last_records": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _szp, C.c_void_p, C.c_size_t, _szp]),
    "apt_decoder_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, _u64p]),
    "apt_decoder_set_profiling": (C.c_int, [C.c_void_p, C.c_int]),
    "apt_decoder_kernel_count": (C.c_int, [C.c_void_p]),
    "apt_decoder_kernel_name": (C.c_char_p, [C.c_void_p, C.c_int]),
    "apt_decoder_kernel_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "apt_decoder_stream": (C.c_void_p, [C.c_void_p]),
    "apt_decoder_launch_count": (C.c_uint64, [C.c_void_p]),
    "apt_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "apt_host_free": (None, [C.c_void_p]),
    "apt_device_alloc": (C.c_int, [C.c_int, C.POINTER(C.c_void_p), C.c_size_t]),
    "apt_device_free": (None, [C.c_int, C.c_void_p]),
    "apt_memcpy_h2d": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "apt_memcpy_d2h": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "apt_ph_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(CPhInfo), C.c_void_p, C.c_size_t,
                              C.c_void_p, C.c_size_t]),
    "apt_ut_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(CUtInfo), C.c_void_p, C.c_size_t]),
    "apt_tile_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(CTileInfo), C.c_void_p,
                                C.c_size_t, C.c_void_p, C.c_size_t]),
    "apt_decode_batch": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, _u64p, C.c_int, C.c_uint32, C.POINTER(CSettings),
                                   C.c_int, C.POINTER(C.c_void_p), _u64p, _u64p, C.POINTER(C.c_int),
                                   C.POINTER(C.c_int), C.c_int, C.c_int]),
    "apt_stream_create": (C.c_int, [C.c_int, C.c_uint32, C.POINTER(CSettings), C.c_int, C.c_uint64, C.POINTER(C.c_void_p)]),
    "apt_stream_destroy": (None, [C.c_void_p]),
    "apt_stream_push_bound": (C.c_int, [C.c_void_p, C.c_uint64, _u64p]),
    "apt_stream_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, _u64p]),
    "apt_stream_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "apt_stream_reset": (C.c_int, [C.c_void_p]),
    "apt_stream_sync_positions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _szp]),
    "apt_stream_get_info": (C.c_int, [C.c_void_p, C.POINTER(CStreamInfo)]),
    "apt_stream_geometry": (C.c_int, [C.c_uint32, C.POINTER(CSettings), C.c_int, C.c_uint64, C.POINTER(CStreamInfo)]),
    "apt_iq_default_settings": (C.c_int, [C.c_uint32, C.c_int32, C.POINTER(CIqSettings)]),
    "apt_fm_demod_len": (C.c_int, [C.c_uint64, C.POINTER(CIqSettings), _u64p]),
    "apt_fm_demod": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.c_void_p, C.c_uint64, _u64p]),
    "apt_fm_demod_channels": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.POINTER(C.c_int32),
                                        C.c_int, C.POINTER(C.c_void_p), C.c_uint64, _u64p]),
    "apt_decode_iq": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.POINTER(CSettings), C.c_int,
                                C.c_void_p, C.c_uint64, _u64p, STATUS_CB, C.c_void_p]),
    "apt_stream_create_iq": (C.c_int, [C.c_int, C.POINTER(CIqSettings), C.POINTER(CSettings), C.c_int, C.c_uint64,
                                       C.POINTER(C.c_void_p)]),
    "apt_stream_geometry_iq": (C.c_int, [C.POINTER(CIqSettings), C.POINTER(CSettings), C.c_int, C.c_uint64,
                                         C.POINTER(CStreamInfo)]),
    "apt_wav_load_iq16":(C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64, _u64p, C.POINTER(C.c_uint32)]),
    "apt_iq_spectrum": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CSpectrumSettings), C.c_void_p,
                                  C.c_uint64, C.POINTER(C.c_uint32)]),
    "apt_iq_find_carriers": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.POINTER(CCarrierSearch),
                                       C.POINTER(CCarrier), C.c_uint32, C.POINTER(C.c_uint32)]),
    "apt_find_carriers_psd": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.POINTER(CCarrierSearch),
                                        C.POINTER(CCarrier), C.c_uint32, C.POINTER(C.c_uint32)]),
    "apt_decode_iq_channels": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.POINTER(C.c_int32),
                                         C.c_int, C.POINTER(CSettings), C.c_int, C.POINTER(C.c_void_p), _u64p, _u64p,
                                         C.POINTER(C.c_int)]),
    "apt_decode_iq_auto": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(CIqSettings), C.POINTER(CCarrierSearch),
                                     C.POINTER(CSettings), C.c_int, C.POINTER(CCarrier), C.c_uint32, C.POINTER(C.c_uint32),
                                     C.POINTER(C.c_void_p), _u64p, _u64p, C.POINTER(C.c_int)]),
    "apt_png_default_settings": (None, [C.POINTER(CPngSettings)]),
    "apt_png_bound": (C.c_int, [C.c_uint32, C.c_uint32, C.c_int, C.POINTER(CPngSettings), _u64p]),
    "apt_png_encode": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(CPngSettings), C.c_void_p,
                                 C.c_uint64, _u64p]),
    "apt_decode_png": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CSettings), C.c_int,
                                 C.POINTER(CProcessSettings), C.POINTER(CPngSettings), C.c_void_p, C.c_uint64, _u64p,
                                 C.POINTER(CImageInfo), STATUS_CB, C.c_void_p]),
    "apt_decoder_set_png_mode": (C.c_int, [C.c_void_p, C.POINTER(CPngSettings)]),
    "apt_decode_wav_png": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(CSettings), C.c_int, C.POINTER(CProcessSettings),
                                     C.POINTER(CPngSettings), C.POINTER(CImageInfo)]),
    "apt_decode_batch_image": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, _u64p, C.c_int, C.c_uint32, C.POINTER(CSettings),
                                         C.c_int, C.POINTER(CProcessSettings), C.POINTER(CPngSettings),
                                         C.POINTER(C.c_void_p), _u64p, _u64p, C.POINTER(CImageInfo), C.POINTER(C.c_int),
                                         C.POINTER(C.c_int), C.c_int, C.c_int]),
    "apt_png_encode_batch": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_int,
                                       C.POINTER(CPngSettings), C.POINTER(C.c_void_p), _u64p, _u64p]),
    "apt_png_group_plan": (C.c_int, [C.c_uint32, C.c_int, C.POINTER(CPngSettings), C.POINTER(C.c_uint32), C.c_uint32,
                                     C.POINTER(CPngGroupInfo), C.POINTER(CPngGroupImage), C.c_size_t]),
    "apt_stream_set_process_mode": (C.c_int, [C.c_void_p, C.POINTER(CProcessSettings), C.c_uint64]),
    "apt_stream_set_png_mode": (C.c_int, [C.c_void_p, C.POINTER(CPngSettings)]),
    "apt_stream_finish_image": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p, C.c_void_p, C.c_uint64, _u64p,
                                          C.POINTER(CImageInfo)]),
    "apt_recording_create": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CSettings),
                                       C.POINTER(C.c_void_p)]),
    "apt_recording_destroy": (None, [C.c_void_p]),
    "apt_recording_get_info": (C.c_int, [C.c_void_p, C.POINTER(CRecordingInfo)]),
    "apt_recording_quality": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "apt_find_passes_quality": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.POINTER(CPassSearch),
                                          C.POINTER(CPass), C.c_uint32, C.POINTER(C.c_uint32)]),
    "apt_recording_decode": (C.c_int, [C.c_void_p, C.POINTER(CPass), C.c_uint32, C.c_int, C.POINTER(CProcessSettings),
                                       C.POINTER(CPngSettings), C.POINTER(C.c_void_p), _u64p, _u64p, C.POINTER(CImageInfo),
                                       C.POINTER(C.c_int)]),
    "apt_pass_tracker_create": (C.c_int, [C.c_uint32, C.POINTER(CPassSearch), C.POINTER(C.c_void_p)]),
    "apt_pass_tracker_feed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(CPassEvent), C.c_uint64, _u64p]),
    "apt_pass_tracker_finish": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(CPassEvent), C.c_uint64, _u64p]),
    "apt_pass_tracker_destroy": (None, [C.c_void_p]),
    "apt_watch_create": (C.c_int, [C.c_int, C.c_uint32, C.POINTER(CSettings), C.POINTER(CWatchSettings), WATCH_CB, C.c_void_p,
                                   C.POINTER(C.c_void_p)]),
    "apt_watch_geometry": (C.c_int, [C.c_uint32, C.POINTER(CSettings), C.POINTER(CWatchSettings), C.POINTER(CWatchInfo)]),
    "apt_watch_push_bound": (C.c_int, [C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_reset": (C.c_int, [C.c_void_p]),
    "apt_watch_get_info": (C.c_int, [C.c_void_p, C.POINTER(CWatchInfo)]),
    "apt_watch_destroy": (None, [C.c_void_p]),
    "apt_watch_iq_geometry": (C.c_int, [C.POINTER(CIqSettings), C.POINTER(C.c_int32), C.c_int, C.POINTER(CSettings),
                                        C.POINTER(CWatchSettings), C.POINTER(CWatchInfo)]),
    "apt_watch_iq_create": (C.c_int, [C.c_int, C.POINTER(CIqSettings), C.POINTER(C.c_int32), C.c_int, C.POINTER(CSettings),
                                      C.POINTER(CWatchSettings), WATCH_IQ_CB, C.c_void_p, C.POINTER(C.c_void_p)]),
    "apt_watch_iq_push_bound": (C.c_int, [C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_iq_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_iq_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "apt_watch_iq_reset": (C.c_int, [C.c_void_p]),
    "apt_watch_iq_get_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(CWatchInfo)]),
    "apt_watch_iq_destroy": (None, [C.c_void_p]),
}

_lib = None


def load():
    """dlopen libaptb200.so and attach the prototypes.  Raises if the library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} has not been built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here means the ABI and the header have diverged
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib
