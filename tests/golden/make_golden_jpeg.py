"""Writes tests/golden/jpeg.npz: a subset of the JPEG test matrix (tests/helpers/jpeg_cases.py) with the pixels the installed
Pillow decodes from it, and the Pillow / libjpeg-turbo versions.  The committed file was made with Pillow 12.2 on libjpeg-turbo
3.1; the CPU and GPU suites decode its files and compare against these pixels as well as against the live Pillow.

    python tests/golden/make_golden_jpeg.py
"""
import os
import sys

import numpy as np
import PIL
from PIL import features

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "helpers"))
import jpeg_cases as JC  # noqa: E402


def main():
    cases = [(n, b) for n, b in JC.matrix() if "640x480" not in n and "641x479" not in n][::4]
    files, pixels, shapes, names = [], [], [], []
    for name, data in cases:
        p = JC.pillow_rgb(data)
        files.append(np.frombuffer(data, np.uint8))
        pixels.append(p.reshape(-1))
        shapes.append(p.shape)
        names.append(name)
    np.savez_compressed(os.path.join(HERE, "jpeg.npz"), files=np.concatenate(files), file_ends=np.cumsum([len(f) for f in files]),
                        pixels=np.concatenate(pixels), pixel_ends=np.cumsum([len(p) for p in pixels]), shapes=np.array(shapes),
                        names=np.array(names), pillow=PIL.__version__, libjpeg_turbo=features.version("libjpeg_turbo"))
    print(len(cases), "files")


if __name__ == "__main__":
    main()
