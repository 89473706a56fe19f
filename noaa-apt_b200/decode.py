"""decode.rs: decode(), find_sync(), generate_sync_frame() -- plus the explicit-state Decoder
(one CUDA stream, device workspaces) and the multi-device batch entry point."""
import ctypes as C

import numpy as np

from . import _lib
from .config import Settings
from .context import Context
from .err import InvalidInput, raise_for
from .frequency import _rate_hz

FINAL_RATE = 4160        # decode.rs:14
PX_PER_ROW = 2080        # decode.rs:35
CARRIER_FREQ = 2400      # decode.rs:38


def _fmt_of(arr):
    if arr.dtype == np.int16:
        return _lib.PCM16
    if arr.dtype == np.float32:
        return _lib.F32
    raise TypeError("signal must be float32 (Signal) or int16 (PCM16 of the WAV)")


def generate_sync_frame(work_rate):
    """decode.rs:171-199"""
    lib = _lib.load()
    n = C.c_size_t(0)
    raise_for(lib.apt_generate_sync_frame(_rate_hz(work_rate), None, 0, C.byref(n)))
    out = np.empty(n.value, dtype=np.int8)
    raise_for(lib.apt_generate_sync_frame(_rate_hz(work_rate), out.ctypes.data, out.size, C.byref(n)))
    return out


def find_sync(context, signal, work_rate, want_correlation=False):
    """decode.rs:204-263 -> positions of the sync frames (and the correlation if asked)."""
    lib = _lib.load()
    x = np.ascontiguousarray(signal, dtype=np.float32)
    wr = _rate_hz(work_rate)
    cap = x.size // max(1, PX_PER_ROW * wr // FINAL_RATE) + 4
    pos = np.empty(cap, dtype=np.uint64)
    n = C.c_size_t(0)
    corr = None
    if want_correlation:
        corr = np.empty(max(0, x.size - 38 * (wr // FINAL_RATE)), dtype=np.float32)
    raise_for(lib.apt_find_sync(x.ctypes.data, x.size, wr, pos.ctypes.data, cap, C.byref(n),
                                corr.ctypes.data if corr is not None else None))
    pos = pos[: n.value].copy()
    return (pos, corr) if want_correlation else pos


def decode_len_bound(n, input_rate, settings=None):
    s = (settings or Settings()).to_c()
    b = C.c_uint64(0)
    raise_for(_lib.load().apt_decode_len_bound(int(n), _rate_hz(input_rate), C.byref(s), C.byref(b)))
    return b.value


def decode(context, settings, signal, input_rate, sync=True):
    """noaa_apt::decode (decode.rs:43-162): Signal at input_rate -> rows*2080 f32 pixels.

    `signal` may also be the int16 PCM of the WAV (the `as f32` cast of wav.rs:37 is then done
    on the device).  sync="track" decodes with tracked sync (Decoder.set_sync_mode) through a decoder of its own."""
    x = np.ascontiguousarray(signal)
    if isinstance(sync, str):
        if sync != "track":
            raise ValueError(f"unknown sync mode {sync!r}: True, False or 'track'")
        with Decoder(input_rate, settings, max_samples=x.size) as dec:
            dec.set_sync_mode("track")
            return dec.decode(x, sync=True)
    lib = _lib.load()
    fmt = _fmt_of(x)
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    bound = C.c_uint64(0)
    raise_for(lib.apt_decode_len_bound(x.size, rate, C.byref(s), C.byref(bound)))
    out = np.empty(max(bound.value, 1), dtype=np.float32)
    n = C.c_uint64(0)

    def _cb(progress, desc, _user):
        if context is not None:
            context.status(progress, desc.decode())

    cb = _lib.STATUS_CB(_cb)
    fn = lib.apt_decode_pcm16 if fmt == _lib.PCM16 else lib.apt_decode
    raise_for(fn(x.ctypes.data, x.size, rate, C.byref(s), int(bool(sync)), out.ctypes.data, out.size, C.byref(n),
                 cb, None))
    return out[: n.value].copy()


# apt_tile_records and apt_record (Decoder.last_records)
TILE_RECORDS = np.dtype([("n_suffix", "<u4"), ("n_prefix", "<u4"), ("max", "<f4")])
RECORD = np.dtype([("pos", "<u4"), ("val", "<f4")])


class Decoder:
    """apt_decoder: plan + device workspaces + one stream; submit()/wait() keep one job in flight."""

    def __init__(self, input_rate, settings=None, max_samples=0, device=0):
        self._lib = _lib.load()
        self.settings = settings or Settings()
        self.input_rate = _rate_hz(input_rate)
        self.device = int(device)
        self.max_samples = int(max_samples)
        s = self.settings.to_c()
        h = C.c_void_p(None)
        raise_for(self._lib.apt_decoder_create(self.device, self.input_rate, C.byref(s), self.max_samples, C.byref(h)))
        self._h = h
        self._keep = None
        self._bpp = None       # bytes per pixel of the process mode's image; None: f32 rows
        self._png = None       # PNG mode: (filter, matches, block_bytes, rgb_from_rgba)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_decoder_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def out_bound(self, n):
        return decode_len_bound(n, self.input_rate, self.settings)

    # --- raw pointer interface (device-resident inputs: torch tensors' data_ptr(), apt_device_alloc) ---
    def submit_device(self, signal_ptr, fmt, n, sync, out_ptr, cap):
        raise_for(self._lib.apt_decoder_submit_device(self._h, signal_ptr, fmt, n, int(bool(sync)), out_ptr, cap))

    def submit_host_ptr(self, signal_ptr, fmt, n, sync, out_ptr, cap):
        raise_for(self._lib.apt_decoder_submit_host(self._h, signal_ptr, fmt, n, int(bool(sync)), out_ptr, cap))

    # --- process mode (image.process on every job) ---
    def set_process_mode(self, contrast=None, percent=0.98, rotate=False, palette=None, tune=(0, 0, 0, 0), rgba=None):
        """contrast=None: back to f32 rows.  Otherwise the numpy submit()/wait()/decode() return the image of
        image.process: (rows, 2080) u8 grey or (rows, 2080, 4) u8 RGBA; image_info() gives the contrast info."""
        from . import image
        if contrast is None:
            raise_for(self._lib.apt_decoder_set_process_mode(self._h, None))
            self._bpp = None
            self._png = None
            return
        ps, bpp, _pal = image.process_settings(contrast, percent, rotate, palette, tune, rgba)
        raise_for(self._lib.apt_decoder_set_process_mode(self._h, C.byref(ps)))   # the palette is copied here
        self._bpp = bpp

    def set_png_mode(self, enabled=True, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
        """In process mode: every job ends in the PNG of its image; submit()/wait()/decode() then return the file's
        bytes.  enabled=False goes back to the image arrays."""
        from . import image
        if not enabled:
            raise_for(self._lib.apt_decoder_set_png_mode(self._h, None))
            self._png = None
            return
        ps = image.png_settings(filter, matches, block_bytes, rgb_from_rgba)
        raise_for(self._lib.apt_decoder_set_png_mode(self._h, C.byref(ps)))
        self._png = (filter, matches, block_bytes, rgb_from_rgba)

    def set_sync_mode(self, mode="peaks", delta=2, lam=0.25):
        """Sync mode of the following sync jobs: "peaks" (the reference's picker, the default) or "track" (tracked sync
        with `delta` samples of period change per row and penalty `lam` per squared sample, DESIGN.md "Tracked sync")."""
        modes = {"peaks": _lib.SYNC_PEAKS, "track": _lib.SYNC_TRACK}
        if mode not in modes:
            raise ValueError(f"unknown sync mode {mode!r}: 'peaks' or 'track'")
        ts = _lib.CTrackSettings(int(delta), float(lam)) if mode == "track" else None
        raise_for(self._lib.apt_decoder_set_sync_mode(self._h, modes[mode], C.byref(ts) if ts is not None else None))

    def image_info(self):
        from . import image
        ci = _lib.CImageInfo()
        raise_for(self._lib.apt_decoder_image_info(self._h, C.byref(ci)))
        return image._info(ci)

    # --- numpy interface ---
    def submit(self, signal, sync=True, out=None):
        x = np.ascontiguousarray(signal)
        fmt = _fmt_of(x)
        bpp = self._bpp
        if out is None:
            if bpp:
                from . import image
                png = image.png_settings(*self._png) if self._png else None
                out = np.empty(max(image.output_bytes(self.out_bound(x.size), bpp, png), 1), dtype=np.uint8)
            else:
                out = np.empty(max(self.out_bound(x.size), 1), dtype=np.float32)
        self._keep = (x, out)
        self.submit_host_ptr(x.ctypes.data, fmt, x.size, sync, out.ctypes.data, out.size)
        return out

    def wait(self):
        n = C.c_uint64(0)
        st = self._lib.apt_decoder_wait(self._h, C.byref(n))
        keep, self._keep = self._keep, None
        raise_for(st)
        if keep is not None:
            bpp = self._bpp
            if bpp and self._png:
                return keep[1][: n.value].tobytes()
            if bpp:
                flat = keep[1][: n.value]
                return flat.reshape(-1, PX_PER_ROW, 4) if bpp == 4 else flat.reshape(-1, PX_PER_ROW)
            return keep[1][: n.value]
        return n.value

    def decode(self, signal, sync=True):
        self.submit(signal, sync)
        r = self.wait()
        return r if isinstance(r, bytes) else r.copy()

    # --- introspection ---
    def last_sync(self):
        n = C.c_size_t(0)
        raise_for(self._lib.apt_decoder_last_sync(self._h, None, 0, C.byref(n)))
        pos = np.empty(n.value, dtype=np.uint64)
        if n.value:
            raise_for(self._lib.apt_decoder_last_sync(self._h, pos.ctypes.data, pos.size, C.byref(n)))
        return pos

    def last_counts(self):
        a, b, c = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        raise_for(self._lib.apt_decoder_last_counts(self._h, C.byref(a), C.byref(b), C.byref(c)))
        r = C.c_uint64(0)
        raise_for(self._lib.apt_decoder_last_root_count(self._h, C.byref(r)))
        return {"n_work": a.value, "n_rows": b.value, "n_peaks": c.value, "n_roots": r.value}

    def last_roots(self):
        n = C.c_size_t(0)
        raise_for(self._lib.apt_decoder_last_roots(self._h, None, 0, C.byref(n)))
        out = np.empty(n.value, dtype=np.uint64)
        if n.value:
            raise_for(self._lib.apt_decoder_last_roots(self._h, out.ctypes.data, out.size, C.byref(n)))
        return out

    def last_records(self):
        """What the sync record kernel wrote for the last job (apt_decoder_last_records): (tiles, records), structured
        arrays -- tiles[t] = (n_suffix, n_prefix, max) of tile t; records = (pos, val) of every tile in tile order, its
        suffix list then its prefix list.  Raises unless the last job was a sync job that ran the record kernel and did
        not overflow its pool."""
        nt, nr = C.c_size_t(0), C.c_size_t(0)
        raise_for(self._lib.apt_decoder_last_records(self._h, None, 0, C.byref(nt), None, 0, C.byref(nr)))
        tiles = np.zeros(nt.value, dtype=TILE_RECORDS)
        recs = np.zeros(nr.value, dtype=RECORD)
        raise_for(self._lib.apt_decoder_last_records(self._h, tiles.ctypes.data if tiles.size else None, tiles.size,
                                                     C.byref(nt), recs.ctypes.data if recs.size else None, recs.size,
                                                     C.byref(nr)))
        return tiles, recs

    def read_stage(self, which):
        idx = {"demodulated": 0, "filtered": 1, "correlation": 2}[which] if isinstance(which, str) else int(which)
        n = C.c_uint64(0)
        raise_for(self._lib.apt_decoder_read_stage(self._h, idx, None, 0, C.byref(n)))
        out = np.empty(n.value, dtype=np.float32)
        if n.value:
            raise_for(self._lib.apt_decoder_read_stage(self._h, idx, out.ctypes.data, out.size, C.byref(n)))
        return out

    def set_profiling(self, enabled):
        raise_for(self._lib.apt_decoder_set_profiling(self._h, int(bool(enabled))))

    def kernel_times_ms(self):
        cnt = self._lib.apt_decoder_kernel_count(self._h)
        ms = (C.c_float * max(cnt, 1))()
        got = C.c_int(0)
        raise_for(self._lib.apt_decoder_kernel_ms(self._h, ms, cnt, C.byref(got)))
        return [(self._lib.apt_decoder_kernel_name(self._h, i).decode(), float(ms[i])) for i in range(got.value)]

    @property
    def stream(self):
        return self._lib.apt_decoder_stream(self._h)

    @property
    def launch_count(self):
        return int(self._lib.apt_decoder_launch_count(self._h))


def _stream_info(ci):
    return {n: int(getattr(ci, n)) for n, _ in _lib.CStreamInfo._fields_}


def stream_geometry(input_rate, settings=None, sync=True, max_push=48000):
    """apt_stream_geometry: latency_work, max_push and device_bytes of a stream, computed on the host (no device)."""
    s = (settings or Settings()).to_c()
    ci = _lib.CStreamInfo()
    raise_for(_lib.load().apt_stream_geometry(_rate_hz(input_rate), C.byref(s), int(bool(sync)), int(max_push), C.byref(ci)))
    return _stream_info(ci)


def stream_geometry_iq(iq_settings, settings=None, sync=True, max_push=1_200_000):
    """apt_stream_geometry_iq: the same for an I/Q stream (max_push in I/Q samples)."""
    s = (settings or Settings()).to_c()
    ci = _lib.CStreamInfo()
    raise_for(_lib.load().apt_stream_geometry_iq(C.byref(iq_settings.to_c()), C.byref(s), int(bool(sync)), int(max_push),
                                                 C.byref(ci)))
    return _stream_info(ci)


class Stream:
    """apt_stream: live decoding.  push() audio as it arrives and get back the image rows that became final; the rows
    of all pushes plus finish() are bit-identical to decode() on the whole recording.  Stream.for_iq(...) takes I/Q
    instead (uint8 / int16 interleaved, complex64 or interleaved float32, as iq.decode_iq), bit-identical to iq.decode_iq."""

    def __init__(self, input_rate, settings=None, sync=True, max_push=48000, device=0, _iq=None):
        self._lib = _lib.load()
        self._iq = _iq is not None
        s = (settings or Settings()).to_c()
        h = C.c_void_p(None)
        if self._iq:
            raise_for(self._lib.apt_stream_create_iq(int(device), C.byref(_iq.to_c()), C.byref(s), int(bool(sync)), int(max_push),
                                                     C.byref(h)))
        else:
            raise_for(self._lib.apt_stream_create(int(device), _rate_hz(input_rate), C.byref(s), int(bool(sync)), int(max_push),
                                                  C.byref(h)))
        self._h = h
        self._bpp = None       # image output: bytes per pixel of the process mode's image; None: off
        self._max_rows = 0
        self._png = None       # PNG output: (filter, matches, block_bytes, rgb_from_rgba)

    @classmethod
    def for_iq(cls, iq_settings, settings=None, sync=True, max_push=1_200_000, device=0):
        """apt_stream_create_iq: pushes are I/Q samples (max_push counts them)."""
        return cls(iq_settings.audio_rate, settings, sync, max_push, device, _iq=iq_settings)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_stream_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _rows(self, n, call):
        cap = C.c_uint64(0)
        raise_for(self._lib.apt_stream_push_bound(self._h, n, C.byref(cap)))
        out = np.empty(max(cap.value, PX_PER_ROW), dtype=np.float32)
        got = C.c_uint64(0)
        raise_for(call(out, got))
        return out[: got.value].reshape(-1, PX_PER_ROW).copy()

    def push(self, samples):
        """float32 or int16 samples -> (k, 2080) float32 rows that became final."""
        x = np.ascontiguousarray(samples).ravel()
        if self._iq:
            from .iq import iq_format
            x, fmt, n = iq_format(x)
        else:
            fmt, n = _fmt_of(x), x.size
        return self._rows(n, lambda out, got: self._lib.apt_stream_push(self._h, x.ctypes.data, fmt, n, out.ctypes.data,
                                                                        out.size, C.byref(got)))

    def finish(self):
        """The remaining rows; raises the error decode() would raise (too short, too few sync frames)."""
        return self._rows(0, lambda out, got: self._lib.apt_stream_finish(self._h, out.ctypes.data, out.size, C.byref(got)))

    def reset(self):
        """A new pass with the same plan, buffers and image / PNG output."""
        raise_for(self._lib.apt_stream_reset(self._h))

    # --- image output (apt_stream_set_process_mode / set_png_mode / finish_image) ---
    def set_process_mode(self, contrast=None, percent=0.98, rotate=False, palette=None, tune=(0, 0, 0, 0), rgba=None,
                         max_rows=2400):
        """Before the first push of a pass: keep the pass's rows (up to max_rows) on the device so that finish_image()
        returns the image of image.process, as image.decode_image would for the whole recording.  contrast=None switches
        image output (and PNG output) off and frees its device memory.  Setting a process mode switches PNG output off."""
        from . import image
        if contrast is None:
            raise_for(self._lib.apt_stream_set_process_mode(self._h, None, 0))
            self._bpp = None
            self._png = None
            return
        ps, bpp, _pal = image.process_settings(contrast, percent, rotate, palette, tune, rgba)
        raise_for(self._lib.apt_stream_set_process_mode(self._h, C.byref(ps), int(max_rows)))   # the palette is copied here
        self._bpp = bpp
        self._max_rows = int(max_rows)
        self._png = None

    def set_png_mode(self, enabled=True, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
        """In process mode, before the first push: finish_image() returns the PNG file's bytes (as image.decode_png)
        instead of the pixels.  The encoder workspace for max_rows rows is reserved here.  enabled=False: pixels again."""
        from . import image
        if not enabled:
            raise_for(self._lib.apt_stream_set_png_mode(self._h, None))
            self._png = None
            return
        ps = image.png_settings(filter, matches, block_bytes, rgb_from_rgba)
        raise_for(self._lib.apt_stream_set_png_mode(self._h, C.byref(ps)))
        self._png = (filter, matches, block_bytes, rgb_from_rgba)

    def finish_image(self):
        """finish() plus the image -> (rows, image, info): the remaining (k, 2080) float32 rows, the (h, 2080) / (h, 2080, 4)
        u8 image or the PNG bytes, and the contrast info.  Raises as finish() does, and when the pass has more rows than
        max_rows."""
        from . import image
        if self._bpp is None:
            raise InvalidInput(_lib.ERR_BAD_ARG, "the stream has no image output: call set_process_mode first")
        png = image.png_settings(*self._png) if self._png else None
        out = np.empty(max(image.output_bytes(self._max_rows * PX_PER_ROW, self._bpp, png), 1), dtype=np.uint8)
        n = C.c_uint64(0)
        ci = _lib.CImageInfo()
        rows = self._rows(0, lambda o, got: self._lib.apt_stream_finish_image(self._h, o.ctypes.data, o.size, C.byref(got),
                                                                             out.ctypes.data, out.size, C.byref(n), C.byref(ci)))
        if self._png:
            return rows, out[: n.value].tobytes(), image._info(ci)
        return rows, image._shape(out[: n.value].copy(), self._bpp), image._info(ci)

    def positions(self):
        n = C.c_size_t(0)
        raise_for(self._lib.apt_stream_sync_positions(self._h, None, 0, C.byref(n)))
        pos = np.empty(n.value, dtype=np.uint64)
        if n.value:
            raise_for(self._lib.apt_stream_sync_positions(self._h, pos.ctypes.data, pos.size, C.byref(n)))
        return pos

    def info(self):
        ci = _lib.CStreamInfo()
        raise_for(self._lib.apt_stream_get_info(self._h, C.byref(ci)))
        return _stream_info(ci)


def decode_batch(signals, input_rate, settings=None, sync=True, devices=None, streams_per_device=4):
    """Independent recordings sharded recording i -> devices[i % G], no collective (SURVEY §8e).
    Returns (list of row arrays or None, list of status codes)."""
    lib = _lib.load()
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    xs = [np.ascontiguousarray(x) for x in signals]
    if not xs:
        return [], []
    fmt = _fmt_of(xs[0])
    if any(_fmt_of(x) != fmt for x in xs):
        raise TypeError("all recordings of a batch must share one sample format")
    count = len(xs)
    outs = [np.empty(max(decode_len_bound(x.size, rate, settings), 1), dtype=np.float32) for x in xs]
    sig_ptrs = (C.c_void_p * count)(*[x.ctypes.data for x in xs])
    out_ptrs = (C.c_void_p * count)(*[o.ctypes.data for o in outs])
    lens = (C.c_uint64 * count)(*[x.size for x in xs])
    caps = (C.c_uint64 * count)(*[o.size for o in outs])
    nouts = (C.c_uint64 * count)()
    statuses = (C.c_int * count)(*([_lib.ERR_CUDA] * count))   # never "ok" unless the library says so
    devs = list(devices) if devices else [0]
    dev_arr = (C.c_int * len(devs))(*devs)
    rc = lib.apt_decode_batch(sig_ptrs, fmt, lens, count, rate, C.byref(s), int(bool(sync)), out_ptrs, caps, nouts,
                              statuses, dev_arr, len(devs), int(streams_per_device))
    if rc != _lib.OK and all(int(v) == rc for v in statuses):
        raise_for(rc)                      # nothing decoded at all (no device, bad settings ...): an error, not a result
    res = [outs[i][: nouts[i]] if statuses[i] == _lib.OK else None for i in range(count)]
    return res, [int(v) for v in statuses]
