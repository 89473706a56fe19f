"""Writes tests/golden/palettes.npz: two false-colour palettes of the reference (res/palettes/) as the (256, 256, 3) u8
RGB arrays processing::false_color reads after `into_rgb8` (alpha dropped).  noaa-apt-daylight.png is stored as RGBA,
WXtoImg-NO.png as RGB, so both conversions are covered.

    python tests/golden/make_palettes.py <noaa-apt source tree>

Needs Pillow.  The tests read only the .npz."""
import os
import sys

import numpy as np
from PIL import Image

NAMES = {"noaa-apt-daylight": "noaa-apt-daylight.png", "WXtoImg-NO": "WXtoImg-NO.png"}


def main(src):
    out = {}
    for key, fname in NAMES.items():
        with Image.open(os.path.join(src, "res", "palettes", fname)) as im:
            print(f"{fname}: mode {im.mode}, size {im.size}")
            rgb = np.asarray(im.convert("RGB"), dtype=np.uint8)
        assert rgb.shape == (256, 256, 3), rgb.shape
        out[key] = rgb
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "palettes.npz")
    np.savez_compressed(dst, **out)
    print(dst)


if __name__ == "__main__":
    main(sys.argv[1])
