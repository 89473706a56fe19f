"""Writes tests/golden/argentina_excerpt.npz: the first rows of the reference's decoded example image
(docs/examples/argentina.png, grey, 2080 px wide) as realistic APT content for the PNG encoder's tests.

    python tests/golden/make_png_excerpt.py <noaa-apt source tree>

Needs Pillow.  The tests read only the .npz."""
import os
import sys

import numpy as np
from PIL import Image

ROWS = 320


def main(src):
    with Image.open(os.path.join(src, "docs", "examples", "argentina.png")) as im:
        print(f"argentina.png: mode {im.mode}, size {im.size}")
        grey = np.asarray(im.convert("L"), dtype=np.uint8)
    assert grey.shape[1] == 2080, grey.shape
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "argentina_excerpt.npz")
    np.savez_compressed(dst, grey=np.ascontiguousarray(grey[:ROWS]))
    print(dst)


if __name__ == "__main__":
    main(sys.argv[1])
