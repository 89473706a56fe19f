"""The copy-out contract every image output path shares.  Whichever entry point a pass's image or PNG file leaves through,
a buffer one byte short is refused with APT_ERR_CAPACITY and the exact length it needs, a buffer of exactly that length
receives the bytes every other entry point gives, and the decoder or stream that refused can be used again."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RATE = 11_025
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


@pytest.fixture(scope="module")
def x(na):
    from noaa_apt_b200 import synth
    return synth.apt_pcm16(RATE, 12.0, seed=11)


def _kw(name):
    from noaa_apt_b200 import image
    if name == "grey":
        return dict(contrast=image.MINMAX)
    palette = np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]
    return dict(contrast=image.MINMAX, palette=palette, rgba=True)


def _decoder_wait(na, x, kw, cap):
    """apt_decoder_wait in PNG mode with a cap-byte buffer -> (status, nout, bytes); then the same decoder decodes again."""
    lib = na._lib.load()
    with na.Decoder(RATE, max_samples=x.size) as dec:
        dec.set_process_mode(**kw)
        dec.set_png_mode()
        out = np.empty(max(cap, 1), np.uint8)
        n = C.c_uint64(0)
        assert lib.apt_decoder_submit_host(dec._h, x.ctypes.data, na._lib.PCM16, x.size, 1, out.ctypes.data, cap) == 0
        st = lib.apt_decoder_wait(dec._h, C.byref(n))
        again = dec.decode(x)
    return st, n.value, out[: n.value].tobytes(), again


def _decode_png(na, x, kw, cap):
    from noaa_apt_b200 import image
    lib = na._lib.load()
    ps, _bpp, _keep = image.process_settings(**kw)
    png = image.png_settings()
    s = na.Settings().to_c()
    out = np.empty(max(cap, 1), np.uint8)
    n = C.c_uint64(0)
    st = lib.apt_decode_png(x.ctypes.data, na._lib.PCM16, x.size, RATE, C.byref(s), 1, C.byref(ps), C.byref(png),
                            out.ctypes.data, cap, C.byref(n), None, na._lib.STATUS_CB(0), None)
    return st, n.value, out[: n.value].tobytes()


def _recording(na, x, kw, cap):
    from noaa_apt_b200 import image
    lib = na._lib.load()
    ps, _bpp, _keep = image.process_settings(**kw)
    png = image.png_settings()
    with na.Recording(x, RATE) as rec:
        arr = (na._lib.CPass * 1)()
        arr[0].start, arr[0].end = 0, x.size
        out = np.empty(max(cap, 1), np.uint8)
        nouts = (C.c_uint64 * 1)()
        sts = (C.c_int * 1)()
        rc = lib.apt_recording_decode(rec._h, arr, 1, 1, C.byref(ps), C.byref(png), (C.c_void_p * 1)(out.ctypes.data),
                                      (C.c_uint64 * 1)(cap), nouts, None, sts)
    assert rc == sts[0]
    return rc, nouts[0], out[: nouts[0]].tobytes()


def _stream(na, x, kw, png, caps):
    """One stream finishing the same pass once per cap (reset in between) -> [(status, image_n, bytes)]."""
    from noaa_apt_b200 import image
    lib = na._lib.load()
    got = []
    with na.Stream(RATE, na.Settings(), max_push=RATE) as strm:
        strm.set_process_mode(max_rows=x.size // (RATE // 2) + 8, **kw)
        if png:
            strm.set_png_mode()
        for cap in caps:
            strm.reset()
            strm.push(x)
            rows_cap = C.c_uint64(0)
            assert lib.apt_stream_push_bound(strm._h, 0, C.byref(rows_cap)) == 0
            rows = np.empty(max(rows_cap.value, 2080), np.float32)
            img = np.empty(max(cap, 1), np.uint8)
            nout, image_n = C.c_uint64(0), C.c_uint64(0)
            ci = na._lib.CImageInfo()
            st = lib.apt_stream_finish_image(strm._h, rows.ctypes.data, rows.size, C.byref(nout), img.ctypes.data, cap,
                                             C.byref(image_n), C.byref(ci))
            got.append((st, image_n.value, img[: image_n.value].tobytes()))
        assert image._info(ci)["rows"] > 0
    return got


def _batch(na, x, kw, caps):
    """apt_decode_batch_image to PNG of x once per cap -> (statuses, nouts, outputs)."""
    from noaa_apt_b200 import image
    lib = na._lib.load()
    ps, _bpp, _keep = image.process_settings(**kw)
    png = image.png_settings()
    s = na.Settings().to_c()
    k = len(caps)
    outs = [np.empty(max(c, 1), np.uint8) for c in caps]
    nouts = (C.c_uint64 * k)()
    sts = (C.c_int * k)()
    dev = (C.c_int * 1)(0)
    lib.apt_decode_batch_image((C.c_void_p * k)(*[x.ctypes.data] * k), na._lib.PCM16, (C.c_uint64 * k)(*[x.size] * k), k, RATE,
                               C.byref(s), 1, C.byref(ps), C.byref(png), (C.c_void_p * k)(*[o.ctypes.data for o in outs]),
                               (C.c_uint64 * k)(*caps), nouts, None, sts, dev, 1, 2)
    return list(sts), list(nouts), [o[: nouts[i]].tobytes() if sts[i] == 0 else None for i, o in enumerate(outs)]


def _encode_batch(na, pixels, caps):
    """apt_png_encode_batch of the same image once per cap -> (status, nouts, outputs)."""
    from noaa_apt_b200 import image
    lib = na._lib.load()
    px = np.ascontiguousarray(pixels)
    ch = 1 if px.ndim == 2 else px.shape[2]
    png = image.png_settings()
    k = len(caps)
    outs = [np.empty(max(c, 1), np.uint8) for c in caps]
    nouts = (C.c_uint64 * k)()
    st = lib.apt_png_encode_batch((C.c_void_p * k)(*[px.ctypes.data] * k), (C.c_uint32 * k)(*[px.shape[0]] * k), k, px.shape[1], ch,
                                  C.byref(png), (C.c_void_p * k)(*[o.ctypes.data for o in outs]), (C.c_uint64 * k)(*caps), nouts)
    return st, list(nouts), [o[: nouts[i]].tobytes() for i, o in enumerate(outs)]


@pytest.mark.parametrize("name", ["grey", "rgba_palette"])
def test_one_copy_out_contract(na, x, name):
    from noaa_apt_b200 import image
    OK, CAP = na._lib.OK, na._lib.ERR_CAPACITY
    kw = _kw(name)
    want, _info = image.decode_png(None, None, x, RATE, **kw)
    pixels, _ = image.decode_image(None, None, x, RATE, **kw)
    L, P = len(want), pixels.nbytes
    assert L > 0 and P == pixels.shape[0] * 2080 * (4 if name != "grey" else 1)

    st, n, _, again = _decoder_wait(na, x, kw, L - 1)
    assert (st, n) == (CAP, L)
    assert again == want, "the decoder after a refused copy-out"
    st, n, got, _ = _decoder_wait(na, x, kw, L)
    assert (st, n, got) == (OK, L, want)

    assert _decode_png(na, x, kw, L - 1)[:2] == (CAP, L)
    assert _decode_png(na, x, kw, L) == (OK, L, want)

    assert _recording(na, x, kw, L - 1)[:2] == (CAP, L)
    assert _recording(na, x, kw, L) == (OK, L, want)

    short, exact = _stream(na, x, kw, True, [L - 1, L])
    assert short[:2] == (CAP, L)
    assert exact == (OK, L, want), "the stream after a refused copy-out"
    short, exact = _stream(na, x, kw, False, [P - 1, P])
    assert short[:2] == (CAP, P)
    assert exact == (OK, P, pixels.tobytes()), "the stream's pixels after a refused copy-out"

    assert _batch(na, x, kw, [L - 1, L]) == ([CAP, OK], [L, L], [None, want])

    st, nouts, outs = _encode_batch(na, pixels, [L - 1, L])
    assert (st, nouts, outs[1]) == (CAP, [L, L], want)
