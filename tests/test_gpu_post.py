"""The image stage's one owner (post.hpp): image mode is process mode with default settings, a sync redo ends in the same
image stage as any job, the stage vectorises only the buffers its kernels need aligned, and the stand-alone entry points
map device statuses as the decoder does."""
import ctypes as C

import numpy as np
import pytest
import torch

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth

pytestmark = pytest.mark.gpu

IMAGE_SLOTS = {image.MINMAX: ["post_stats", "post_bounds", "post_map_u8"],
               image.PERCENT: ["post_stats", "post_histogram", "post_bounds", "post_map_u8"],
               image.TELEMETRY: ["post_stats", "post_bounds", "post_map_u8"]}


@pytest.fixture(scope="module")
def recording():
    return synth.apt_signal(11025, 150, seed=12)    # 300 rows: enough for a telemetry frame (200 rows)


def _profiled_job(dec, x, sync):
    """(image bytes or the error, info, launches, slot names) of one job."""
    dec.set_profiling(True)
    c0 = dec.launch_count
    dec.submit(x, sync, out=np.empty(dec.out_bound(x.size), np.uint8))
    try:
        img = np.asarray(dec.wait()).ravel().copy()
    except na.err.Error as e:                                   # the same status from both modes
        img = (type(e), e.code, str(e))
    launches = dec.launch_count - c0
    slots = [k for k, _ in dec.kernel_times_ms()]
    dec.set_profiling(False)
    return img, dec.image_info(), launches, slots


@pytest.mark.parametrize("sync", [True, False])
@pytest.mark.parametrize("contrast", [image.MINMAX, image.PERCENT, image.TELEMETRY])
def test_image_mode_is_process_mode_with_default_settings(recording, contrast, sync):
    lib = na._lib.load()
    with na.Decoder(11025, na.Settings(), max_samples=recording.size) as dec:
        dec.decode(recording, sync)                                 # first job: lazy allocations
        assert lib.apt_decoder_set_image_mode(dec._h, contrast, 0.98) == 0
        img, info, launches, slots = _profiled_job(dec, recording, sync)
        dec.set_process_mode(contrast=contrast)
        img_p, info_p, launches_p, slots_p = _profiled_job(dec, recording, sync)
    assert (img == img_p) if isinstance(img, tuple) else np.array_equal(img, img_p)
    assert info["low"] == info_p["low"] and info["high"] == info_p["high"] and info["rows"] == info_p["rows"]
    assert info["telemetry_row"] == info_p["telemetry_row"]
    assert np.array_equal(info["wedges_a"], info_p["wedges_a"]) and np.array_equal(info["wedges_b"], info_p["wedges_b"])
    assert launches == launches_p
    assert slots == slots_p and slots[-len(IMAGE_SLOTS[contrast]):] == IMAGE_SLOTS[contrast]


@pytest.mark.parametrize("kw", [dict(contrast=image.MINMAX), dict(contrast=image.PERCENT, rgba=True),
                                dict(contrast=image.HISTOGRAM, rotate=True)])
def test_redo_job_image_is_process_of_its_own_rows(kw, monkeypatch):
    monkeypatch.setenv("APTB200_RECORD_POOL", "4096")               # read when the decoder is created
    x = synth.apt_signal(48000, 14, seed=42)
    x[x.size // 2:] = 0.0                                           # silence: every index a record, the pool overflows
    with na.Decoder(48000, na.Settings(), max_samples=x.size) as dec:
        rows = dec.decode(x, True)
        dec.set_process_mode(**kw)
        dec.set_profiling(True)
        img = dec.decode(x, True)
        slots = [k for k, _ in dec.kernel_times_ms()]
        info = dec.image_info()
    assert "lowpass_correlation" in slots                          # the Hbm kernels ran again after the overflow
    ref, ref_info = image.process(rows, **kw)
    assert np.array_equal(img, ref)
    assert (info["low"], info["high"], info["rows"]) == (ref_info["low"], ref_info["high"], ref_info["rows"])


def test_unaligned_device_output_without_a_finishing_pass(recording):
    with na.Decoder(11025, na.Settings(), max_samples=recording.size) as dec:
        dec.set_process_mode(contrast=image.MINMAX)
        want = dec.decode(recording, True)
        bound = dec.out_bound(recording.size)
        x = torch.from_numpy(recording).cuda()
        out = torch.zeros(bound + 16, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        dec.submit_device(x.data_ptr(), na._lib.F32, recording.size, True, out.data_ptr() + 1, bound)
        n = dec.wait()
        got = out[1:1 + n].cpu().numpy()
    assert np.array_equal(got, want.ravel())


def test_stand_alone_telemetry_too_short_is_too_short():
    rows = synth.apt_signal(11025, 60, seed=4)                      # 120 rows < 200
    rows = na.decode(na.Context(), na.Settings(), rows, 11025, True)
    lib = na._lib.load()
    ci = na._lib.CImageInfo()
    st = lib.apt_contrast_bounds(rows.ctypes.data, rows.size, image.TELEMETRY, C.c_float(0.98), C.byref(ci))
    assert st == na._lib.ERR_TOO_SHORT
    assert b"too short for telemetry" in lib.apt_last_error()
    with pytest.raises(na.err.Internal, match="too short for telemetry") as e:
        image.process(rows, image.TELEMETRY, rgba=True)
    assert e.value.code == na._lib.ERR_TOO_SHORT
