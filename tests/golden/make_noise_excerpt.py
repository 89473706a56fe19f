"""Stores the reference's receiver-noise recording `test/noise_48000hz.wav` (despite its name 11025 Hz, 16-bit mono,
30 s) as raw PCM16 samples in tests/golden/noise_11025hz.npz: real noise from a real receiver, for the test that the pass
search finds no pass in it.  The file holds reference-owned DATA (a fixture), no reference code.  The sha256 of the WAV
is stored next to the samples, and the sha256 of the samples themselves, so that the tests can tell the fixture is intact.

    python tests/golden/make_noise_excerpt.py <reference checkout>/test/noise_48000hz.wav
"""
import hashlib
import os
import sys
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def main(wav_path):
    with open(wav_path, "rb") as f:
        digest = hashlib.sha256(f.read()).hexdigest()
    with wave.open(wav_path) as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 11025)
        pcm = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.int16)
    np.savez(os.path.join(HERE, "noise_11025hz.npz"), pcm=pcm, rate=np.int64(11025), sha256=np.array(digest),
             pcm_sha256=np.array(hashlib.sha256(pcm.tobytes()).hexdigest()))
    print(pcm.size, "samples,", digest)


if __name__ == "__main__":
    main(sys.argv[1])
