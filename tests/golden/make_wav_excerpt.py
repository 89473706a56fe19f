"""Cuts two excerpts (60 s in total) out of the reference's own test recording
`test/test_11025hz.wav` (11025 Hz, 16-bit mono, 822 s; sha256 50160851becd5997...) and stores the
raw PCM16 samples in tests/golden/test_11025hz_excerpts.npz, so that the one real-world input the reference
ships (test/test.sh:45-46) reaches the CUDA kernels and the tests without the reference checkout.

    [0 s, 40 s)     the recording starts in noise: sync spacings from 1122 to 13454 work samples, the seed peak is
                    refined, several frames are skipped (decode.rs:241-253)
    [230 s, 250 s)  a noisy stretch in which the `while` at decode.rs:244 pushes the same position twice
                    (duplicate sync position -> duplicate image row) and the largest gap of the file (18708)

The file holds reference-owned DATA (a fixture), no reference code.  The sync positions the CPU oracle finds are
stored next to the samples as a drift guard; the GPU tests recompute them with the oracle on the box.

    python tests/golden/make_wav_excerpt.py <reference checkout>/test/test_11025hz.wav
"""
import hashlib
import os
import sys
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
EXCERPTS = {"start": (0, 40), "dup": (230, 250)}


def main(wav_path):
    import oracle
    with open(wav_path, "rb") as f:
        digest = hashlib.sha256(f.read()).hexdigest()
    with wave.open(wav_path) as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 11025)
        pcm = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2")
    out = {"rate": np.int64(11025), "sha256": np.array(digest)}
    for name, (t0, t1) in EXCERPTS.items():
        cut = pcm[t0 * 11025: t1 * 11025].copy()
        _, st = oracle.decode_steps(oracle.pcm16_to_f32(cut), 11025)
        out[f"pcm_{name}"] = cut
        out[f"sync_{name}"] = st["sync_pos"]
        print(name, cut.size, "samples,", st["sync_pos"].size, "sync positions, min spacing",
              int(np.diff(st["sync_pos"].astype(np.int64)).min()))
    np.savez_compressed(os.path.join(HERE, "test_11025hz_excerpts.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1])
