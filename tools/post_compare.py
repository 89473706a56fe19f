"""Before/after check of the image stage: every output of image mode, process mode and the stage entry points, with
apt_image_info, status codes and decoder launch counts, dumped by one library and compared with another's dump.
    APTB200_LIB=<lib A> python tools/post_compare.py dump a.npz
    APTB200_LIB=<lib B> python tools/post_compare.py dump b.npz
    python tools/post_compare.py compare a.npz b.npz        # exit status 1 on any difference"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def dump(path):
    import noaa_apt_b200 as na
    from noaa_apt_b200 import image, synth
    lib = na._lib.load()
    res = {}
    pal = np.load(os.path.join(ROOT, "tests", "golden", "palettes.npz"))["noaa-apt-daylight"]
    tune = (0.4, -0.3, -0.6, 0.8)
    modes = {f"image_c{c}": ("image", c) for c in (0, 1, 2)}
    modes.update({
        "minmax_grey": dict(contrast=image.MINMAX),
        "minmax_rgba": dict(contrast=image.MINMAX, rgba=True),
        "percent_grey": dict(contrast=image.PERCENT, percent=0.95),
        "histogram_grey_rotate": dict(contrast=image.HISTOGRAM, rotate=True),
        "histogram_rgba": dict(contrast=image.HISTOGRAM, rgba=True),
        "telemetry_palette_rotate_rgba": dict(contrast=image.TELEMETRY, rotate=True, palette=pal, tune=tune),
    })

    def info_vec(ci):
        return np.concatenate([np.array([ci.low, ci.high], np.float64), [float(ci.rows), float(ci.telemetry_row)],
                               np.array(ci.wedges_a[:], np.float64), np.array(ci.wedges_b[:], np.float64)])

    def put(key, st, data=None, ci=None, launches=None):
        res[key + "/status"] = np.array([st])
        if data is not None:
            res[key + "/data"] = np.asarray(data)
        if ci is not None:
            res[key + "/info"] = info_vec(ci)
        if launches is not None:
            res[key + "/launches"] = np.array([launches])

    def set_mode(dec, mode):
        if isinstance(mode, tuple):
            assert lib.apt_decoder_set_image_mode(dec._h, mode[1], C.c_float(0.98)) == 0
            return 1
        dec.set_process_mode(**mode)
        return 4 if mode.get("rgba") else 1

    recordings = {"11k_f32": (11025, synth.apt_signal(11025, 150, seed=12)),
                  "11k_pcm16": (11025, synth.apt_pcm16(11025, 150, seed=12)),
                  "48k_pcm16": (48000, synth.apt_pcm16(48000, 120, seed=3))}
    silent = synth.apt_signal(48000, 14, seed=42)
    silent[silent.size // 2:] = 0.0                                 # the record pool overflows: the sync redo runs
    recordings["48k_half_silent"] = (48000, silent)
    s = na.Settings().to_c()
    for rname, (rate, x) in recordings.items():
        if rname == "48k_half_silent":
            lib.apt_cache_clear()
            os.environ["APTB200_RECORD_POOL"] = "4096"              # read when a decoder is created
        fmt = na._lib.PCM16 if x.dtype == np.int16 else na._lib.F32
        for sync in (True, False):
            dec = na.Decoder(rate, na.Settings(), max_samples=x.size)
            bound = dec.out_bound(x.size)
            for mname, mode in modes.items():
                key = f"{rname}/sync{int(sync)}/{mname}"
                bpp = set_mode(dec, mode)
                # submit_host
                out = np.zeros(bound * bpp, np.uint8)
                c0 = dec.launch_count
                n = C.c_uint64(0)
                st = lib.apt_decoder_submit_host(dec._h, x.ctypes.data, fmt, x.size, int(sync), out.ctypes.data, out.size)
                if st == 0:
                    st = lib.apt_decoder_wait(dec._h, C.byref(n))
                ci = na._lib.CImageInfo()
                lib.apt_decoder_image_info(dec._h, C.byref(ci))
                put(key + "/host", st, out[: n.value], ci, dec.launch_count - c0)
                # submit_device
                import torch
                xd = torch.from_numpy(x).cuda()
                od = torch.zeros(bound * bpp + 16, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                c0 = dec.launch_count
                st = lib.apt_decoder_submit_device(dec._h, xd.data_ptr(), fmt, x.size, int(sync), od.data_ptr(), bound * bpp)
                if st == 0:
                    st = lib.apt_decoder_wait(dec._h, C.byref(n))
                lib.apt_decoder_image_info(dec._h, C.byref(ci))
                put(key + "/device", st, od[: n.value].cpu().numpy() if st == 0 else None, ci, dec.launch_count - c0)
                # one-shot forms
                ci = na._lib.CImageInfo()
                if isinstance(mode, tuple):
                    st = lib.apt_decode_image_u8(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(sync), mode[1], C.c_float(0.98),
                                                 out.ctypes.data, out.size, C.byref(n), C.byref(ci), na._lib.STATUS_CB(0), None)
                    put(key + "/decode_image_u8", st, out[: n.value] if st == 0 else None, ci)
                    ps, _, _keep = image.process_settings(mode[1])
                else:
                    ps, _, _keep = image.process_settings(**mode)
                st = lib.apt_decode_image(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(sync), C.byref(ps), out.ctypes.data,
                                          out.size, C.byref(n), C.byref(ci), na._lib.STATUS_CB(0), None)
                put(key + "/decode_image", st, out[: n.value] if st == 0 else None, ci)
                if rname.startswith("11k"):
                    png = image.png_settings()
                    pout = np.zeros(image.png_bound(2080, max(bound // 2080, 1), bpp) + 64, np.uint8)
                    st = lib.apt_decode_png(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(sync), C.byref(ps), C.byref(png),
                                            pout.ctypes.data, pout.size, C.byref(n), C.byref(ci), na._lib.STATUS_CB(0), None)
                    put(key + "/decode_png", st, pout[: n.value] if st == 0 else None, ci)
            dec.set_process_mode(None)
            dec.close()
        # the stage entry points on this recording's rows
        rows = na.decode(na.Context(), na.Settings(), x, rate, True)
        for mname, mode in modes.items():
            ps, bpp, _keep = image.process_settings(mode[1]) if isinstance(mode, tuple) else image.process_settings(**mode)
            out = np.zeros(rows.size * bpp, np.uint8)
            n = C.c_uint64(0)
            ci = na._lib.CImageInfo()
            st = lib.apt_process(rows.ctypes.data, rows.size, C.byref(ps), out.ctypes.data, out.size, C.byref(n), C.byref(ci))
            put(f"{rname}/process/{mname}", st, out[: n.value] if st == 0 else None, ci)
        for c in (0, 1, 2, 3):
            for sig_name, sig in (("rows", rows), ("partial", rows[: rows.size - 7])):
                ci = na._lib.CImageInfo()
                st = lib.apt_contrast_bounds(sig.ctypes.data, sig.size, c, C.c_float(0.98), C.byref(ci))
                put(f"{rname}/contrast_bounds/{sig_name}/c{c}", st, None, ci)
        a, b, v = (np.zeros(rows.size // 2080, np.float32) for _ in range(3))
        st = lib.apt_telemetry_rows(rows.ctypes.data, rows.size, a.ctypes.data, b.ctypes.data, v.ctypes.data)
        put(f"{rname}/telemetry_rows", st, np.concatenate([a, b, v]))
        m = np.zeros(rows.size, np.uint8)
        st = lib.apt_map_signal_u8(rows.ctypes.data, rows.size, C.c_float(float(rows.min())), C.c_float(float(rows.max()) * 0.9),
                                   m.ctypes.data)
        put(f"{rname}/map_signal_u8", st, m)
        q = np.zeros(rows.size, np.int16)
        st = lib.apt_quantize_i16(rows.ctypes.data, rows.size, q.ctypes.data)
        put(f"{rname}/quantize_i16", st, q)
    # the 12-value vector of the reference's test_map (noaa_apt.rs)
    v = np.array([-1.0, -0.5, 0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0, 1.5, 2.0, 0.3333], np.float32)
    m = np.zeros(v.size, np.uint8)
    put("test_map", lib.apt_map_signal_u8(v.ctypes.data, v.size, C.c_float(0.0), C.c_float(1.0), m.ctypes.data), m)
    np.savez(path, **res)
    print(f"{len(res)} arrays -> {path}")


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        if a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes():
            bad.append(k)
    statuses = sorted({int(a[k][0]) for k in a.files if k.endswith("/status")})
    print(f"{len(a.files)} / {len(b.files)} arrays; statuses seen {statuses}; {len(bad)} differ")
    for k in bad[:40]:
        print("DIFF", k)
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
