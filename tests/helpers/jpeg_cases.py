"""Seeded JPEG test files for tests/test_jpeg_cpu.py, tests/test_gpu_jpeg.py and tests/golden/make_golden_jpeg.py.

The matrix crosses samplings (4:4:4, 4:2:2, 4:2:0 through Pillow's `subsampling`, 4:4:0 through OpenCV, grayscale), sizes
chosen to hit every residue of the 8- and 16-pixel MCU edges, qualities 1..100, Pillow's encoder options (optimised tables,
restart markers by blocks and by rows, extreme quantisation tables) and four kinds of content."""
import io

import cv2
import numpy as np
from PIL import Image

SAMPLINGS = ("444", "422", "420", "440", "gray")
SIZES = ((1, 1), (2, 3), (7, 9), (15, 17), (16, 16), (17, 33), (33, 65), (641, 479), (640, 480))   # (w, h)
QUALITIES = (1, 10, 50, 75, 95, 100)
OPTIONS = ("plain", "optimize", "rst_blocks1", "rst_blocks3", "rst_rows1", "qtables_extreme")
CONTENTS = ("noise", "scene", "flat", "checker")


def content(kind, w, h, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.broadcast_to(np.array([37, 201, 118], np.uint8), (h, w, 3)).copy()
    if kind == "checker":
        yy, xx = np.mgrid[0:h, 0:w]
        c = ((yy // 3 + xx // 3) % 2).astype(np.uint8) * 255
        return np.stack([c, 255 - c, c // 2], -1)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)          # smooth scene: gradients, a disc, mild noise
    r = 128 + 100 * np.sin(xx / 23.0) * np.cos(yy / 31.0)
    g = 255 * xx / max(w - 1, 1)
    b = 255 * yy / max(h - 1, 1)
    disc = (xx - w / 2) ** 2 + (yy - h / 2) ** 2 < (min(w, h) / 3) ** 2
    img = np.stack([r, g, b], -1)
    img[disc] = [250, 30, 60]
    img += rng.normal(0, 4, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def encode(img, sampling="420", quality=75, option="plain"):
    if sampling == "440":
        ok, buf = cv2.imencode(".jpg", img[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, quality,
                                                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])
        assert ok
        return buf.tobytes()
    kw = dict(quality=quality)
    if sampling == "gray":
        im = Image.fromarray(img[..., 1])
    else:
        im = Image.fromarray(img)
        kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[sampling]
    if option == "optimize":
        kw["optimize"] = True
    elif option == "rst_blocks1":
        kw["restart_marker_blocks"] = 1
    elif option == "rst_blocks3":
        kw["restart_marker_blocks"] = 3
    elif option == "rst_rows1":
        kw["restart_marker_rows"] = 1
    elif option == "qtables_extreme":
        kw.pop("quality")
        kw["qtables"] = [[1] * 64, [255] * 64] if sampling != "gray" else [[1] * 64]
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def pillow_rgb(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def matrix():
    """(name, bytes) of the test matrix: every sampling x size, every quality and option at chosen sizes, every content."""
    out = []
    for s in SAMPLINGS:
        for (w, h) in SIZES:
            out.append(("%s_%dx%d_q75_noise" % (s, w, h), encode(content("noise", w, h, w * 7 + h), s, 75)))
        for q in QUALITIES:
            for (w, h) in ((17, 33), (33, 65)):
                out.append(("%s_%dx%d_q%d_scene" % (s, w, h, q), encode(content("scene", w, h, q), s, q)))
        if s != "440":
            for o in OPTIONS[1:]:
                for (w, h) in ((33, 65), (641, 479)):
                    out.append(("%s_%dx%d_%s" % (s, w, h, o), encode(content("scene", w, h, 3), s, 90, o)))
        for c in CONTENTS:
            out.append(("%s_640x480_q95_%s" % (s, c), encode(content(c, 640, 480, 11), s, 95)))
    return out


def declined():
    """(name, bytes, expected decline reason substring) of files the GPU path must leave to Pillow."""
    img = content("scene", 40, 30, 1)
    out = []
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=80, progressive=True)
    out.append(("progressive", b.getvalue(), "progressive"))
    b = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(b, "JPEG", quality=80)
    out.append(("cmyk", b.getvalue(), "CMYK"))
    base = encode(img, "444", 80)
    app0_len = base[4] << 8 | base[5]
    assert base[2:4] == b"\xff\xe0"
    adobe = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"       # APP14, transform 0: RGB-coded
    out.append(("adobe_transform0", base[:2] + adobe + base[4 + app0_len:], "RGB-coded"))
    out.append(("cut_before_eoi", base[:len(base) - 40], "EOI"))
    return out
