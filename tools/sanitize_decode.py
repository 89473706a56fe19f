"""Small decodes through every resampler path and a small PNG encode, for compute-sanitizer (tools/sanitize.sh)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import noaa_apt_b200 as na
from noaa_apt_b200 import synth
import oracle

cases = [(48000, "standard", 12), (96000, "standard", 12), (11025, "standard", 14), (48000, "fast", 12), (24960, "standard", 12)]
if len(sys.argv) > 1:
    cases = cases[: int(sys.argv[1])]
for rate, profile, seconds in cases:
    x = synth.apt_signal(rate, seconds, seed=3)
    s = na.Settings.profile(profile)
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        got = dec.decode(x)
        pos = dec.last_sync()
        got16 = dec.decode(synth.apt_pcm16(rate, seconds, seed=3))
    os_ = oracle.default_settings()
    os_.work_rate, os_.resample_atten = s.work_rate, s.resample_atten
    os_.resample_delta_freq, os_.resample_cutout, os_.demodulation_atten = s.resample_delta_freq, s.resample_cutout, s.demodulation_atten
    ref, st = oracle.decode_steps(x, rate, os_)
    ok = np.array_equal(pos, st["sync_pos"]) and got.size == ref.size and got16.size == ref.size
    print(rate, profile, "rows", got.size // 2080, "sync equal" if ok else "MISMATCH", flush=True)

# The PNG encoder (DESIGN.md §11): one small RGBA encode of several 4 KiB blocks with matches (look-back across block
# boundaries, words shared by blocks and warps), checked against the CPU restatement, and one decoder job in PNG mode.
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import _png_oracle as po                                            # noqa: E402
from noaa_apt_b200 import image                                     # noqa: E402

g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                         "argentina_excerpt.npz"))["grey"][:6, :700]
rgba = np.empty(g.shape + (4,), dtype=np.uint8)
rgba[..., :3] = g[..., None]
rgba[..., 3] = 255
png = image.encode_png(rgba, block_bytes=4096)
print("png encode", len(png), "bytes", "equal" if png == po.encode(rgba, block_bytes=4096) else "MISMATCH", flush=True)
x = synth.apt_signal(11025, 14, seed=3)
with na.Decoder(11025, na.Settings(), max_samples=x.size) as dec:
    dec.set_process_mode(image.MINMAX, rgba=True)
    img = dec.decode(x)
    dec.set_png_mode(block_bytes=4096)
    png = dec.decode(x)
print("png mode", len(png), "bytes", "equal" if png == image.encode_png(img, block_bytes=4096) else "MISMATCH", flush=True)

# The stream's image output (DESIGN.md §9): a small pass pushed in pieces with PNG output, the rows kept on the device,
# the image stage and the encoder at finish, against apt_decode_png of the whole recording.
with na.Stream(11025, na.Settings(), max_push=20000) as st:
    st.set_process_mode(image.PERCENT, rotate=True, rgba=True, max_rows=64)
    st.set_png_mode(block_bytes=4096)
    for at in range(0, x.size, 30011):
        st.push(x[at:at + 30011])
    _rows, spng, _info = st.finish_image()
want, _ = image.decode_png(None, na.Settings(), x, 11025, contrast=image.PERCENT, rotate=True, rgba=True, block_bytes=4096)
print("stream png", len(spng), "bytes", "equal" if spng == want else "MISMATCH", flush=True)

# Batch PNG output (DESIGN.md §11, "Batched encode"): three short recordings of different lengths, RGBA, 4 KiB blocks,
# decoded by two decoders and encoded in groups, each file against apt_decode_png of that recording alone.
xs = [synth.apt_signal(11025, sec, seed=4 + sec) for sec in (12, 15, 13)]
files, _infos, sts = image.decode_batch_png(xs, 11025, contrast=image.MINMAX, rgba=True, block_bytes=4096,
                                            streams_per_device=2)
same = sts == [0, 0, 0] and all(
    files[i] == image.decode_png(None, na.Settings(), x, 11025, contrast=image.MINMAX, rgba=True, block_bytes=4096)[0]
    for i, x in enumerate(xs))
print("batch png", [len(f or b"") for f in files], "bytes", "equal" if same else "MISMATCH", flush=True)

# The streamed first stage (FrontWindow, front.hpp) with the decimate kind, the only one with the scratch window d_r beside
# the envelope window: a 24 960 Hz stream and an audio watcher, each pushed in uneven pieces so that every window compacts,
# against apt_decode of the whole recording and the recording path (apt_recording_quality / _find_passes / _decode).
x = synth.apt_signal(24960, 14, seed=5)
pieces = [7001, 13, 30011, 1, 24960]
with na.Stream(24960, max_push=20000) as st:
    rows, at, i = [], 0, 0
    while at < x.size:
        rows.append(st.push(x[at:at + pieces[i % len(pieces)]]))
        at += pieces[i % len(pieces)]
        i += 1
    rows.append(st.finish())
got = np.concatenate(rows).ravel()
want = na.decode(None, na.Settings(), x, 24960, True)
print("stream 24960", got.size // 2080, "rows", "equal" if np.array_equal(got.view(np.uint32), want.view(np.uint32))
      else "MISMATCH", flush=True)

search = dict(max_gap_s=5.0, min_length_s=20.0)
x = synth.apt_passes(24960, [("noise", 6), ("pass", 40, 5), ("noise", 12)], seed=6)
with na.Watch(24960, search=search, max_push=12480) as w:
    qs, evs, at, i = [], [], 0, 0
    while at < x.size:
        q, e = w.push(x[at:at + pieces[i % len(pieces)]])
        qs.append(q)
        evs += e
        at += pieces[i % len(pieces)]
        i += 1
    q, e = w.finish()
    qs.append(q)
    evs += e
with na.Recording(x, 24960) as rec:
    q_ref = rec.quality()
    found = na.find_passes_quality(q_ref, x.size, 24960, **search)
    data, sts = rec.decode(found, True)
los = [e for e in evs if e.kind == "los"]
same = np.array_equal(np.concatenate(qs).view(np.uint32), q_ref.view(np.uint32)) and [e.pass_ for e in los] == found and \
    all(e.status == s and (s != 0 or np.array_equal(e.data.view(np.uint32), d.view(np.uint32)))
        for e, s, d in zip(los, sts, data))
print("watch 24960", len(found), "passes", "equal" if same and found else "MISMATCH", flush=True)
