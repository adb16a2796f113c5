"""GPU tests of the batched JPEG decoder (csrc/jpeg.cu, singleshotpose_b200/jpeg.py): byte-equal to Pillow and to the host build
of jpeg_core.h on the golden and the live matrix in mixed batches; batch- and launch-independence; the many-CTA case; the
Pillow fallback for declined files."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from singleshotpose_b200.jpeg import GpuJpegDecoder, decode_jpeg

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "tests", "helpers"))
import jpeg_cases as JC  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dec():
    return GpuJpegDecoder("cuda")


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("jpeghost") / "libjpeghost.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(REPO, "tests", "helpers", "jpeg_host.cpp")])
    lib = C.CDLL(so)
    lib.h_decode.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _mixed(blobs, seed):
    order = np.random.default_rng(seed).permutation(len(blobs))
    return [blobs[i] for i in order], order


def test_golden_in_mixed_batch(dec, golden_dir):
    g = np.load(os.path.join(golden_dir, "jpeg.npz"))
    files = [f.tobytes() for f in np.split(g["files"], g["file_ends"][:-1])]
    pix = [p.reshape(s) for p, s in zip(np.split(g["pixels"], g["pixel_ends"][:-1]), g["shapes"])]
    blobs, order = _mixed(files, 0)
    f0 = dec.fallbacks
    outs = dec(blobs)
    for o, i in zip(outs, order):
        assert np.array_equal(o.cpu().numpy(), pix[i])
    assert dec.fallbacks == f0


def test_matrix_in_mixed_batches_equals_pillow_and_host(dec, host):
    cases = JC.matrix()
    blobs, order = _mixed([b for _, b in cases], 1)
    f0 = dec.fallbacks
    for k in range(0, len(blobs), 48):
        chunk = blobs[k:k + 48]
        outs = dec(chunk)
        for o, b in zip(outs, chunk):
            want = JC.pillow_rgb(b)
            got = o.cpu().numpy()
            assert np.array_equal(got, want)
            h = np.zeros_like(want)
            assert host.h_decode(b, len(b), 1024, h.ctypes.data, np.zeros(2, np.int64).ctypes.data) == 0
            assert np.array_equal(got, h)
    assert dec.fallbacks == f0                  # every matrix file decoded on the GPU
    assert dec.launches > 0


def test_alone_equals_in_batch_of_192_and_across_launches(dec):
    cases = JC.matrix()
    probe = cases[len(cases) // 2][1]
    alone = dec([probe])[0].clone()
    others = [JC.encode(JC.content("scene", 160 + (i % 5) * 17, 120 + (i % 3) * 9, i), JC.SAMPLINGS[i % 5], 60 + i % 30) for i in range(191)]
    batch = others[:95] + [probe] + others[95:]
    a = dec(batch)
    b = dec(batch)
    assert torch.equal(a[95], alone) and torch.equal(b[95], alone)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_many_cta_batch_of_128_640x480(dec):
    blobs = [JC.encode(JC.content("scene", 640, 480, i), "420", 75 + i % 20) for i in range(128)]
    outs = dec(blobs)
    for i in (0, 37, 127):
        assert np.array_equal(outs[i].cpu().numpy(), JC.pillow_rgb(blobs[i]))
    assert all(o.shape == (480, 640, 3) for o in outs)


def test_declined_files_fall_back_to_pillow(dec):
    good = [JC.encode(JC.content("scene", 33, 65, i), "420", 80) for i in range(3)]
    bad = [b for _, b, r in JC.declined() if "EOI" not in r]
    blobs = [good[0], bad[0], good[1], bad[1], bad[2], good[2]]
    f0 = dec.fallbacks
    outs = dec(blobs)
    for o, b in zip(outs, blobs):
        assert np.array_equal(o.cpu().numpy(), JC.pillow_rgb(b))
    assert dec.fallbacks - f0 == len(bad)
    with pytest.raises(OSError):               # a truncated file raises, as Image.open(f).convert('RGB') does
        dec([good[0], JC.declined()[3][1]])


def test_decode_jpeg_one_file():
    b = JC.encode(JC.content("checker", 17, 33, 0), "422", 90)
    assert np.array_equal(decode_jpeg(b).cpu().numpy(), JC.pillow_rgb(b))


def test_batched_augmenter_device_resident_inputs_match_host_arrays():
    import random
    from singleshotpose_b200 import image, synth
    ims, mks, bgs = zip(*[synth.photo_sample(i, 160 + 8 * i, 120, 100 + 5 * i, 75) for i in range(5)])
    params = [image.draw_augmentation(im.shape[1], im.shape[0], 0.2, 0.1, 1.5, 1.5, random.Random(i)) for i, im in enumerate(ims)]
    aug = image.GpuAugmenter("cuda", keep_u8=True)
    x_host, _, u8_host = aug(list(ims), list(mks), list(bgs), (96, 64), params=params)
    dev = lambda arrs: [torch.from_numpy(a).cuda() for a in arrs]
    mixed_masks = [torch.from_numpy(m).cuda() if i % 2 else m for i, m in enumerate(mks)]   # device and host in one batch
    x_dev, _, u8_dev = aug(dev(ims), mixed_masks, dev(bgs), (96, 64), params=params)
    assert torch.equal(u8_dev, u8_host) and torch.equal(x_dev, x_host)
    assert aug.h2d_bytes < sum(a.nbytes for a in ims + bgs)            # device inputs are not staged


@pytest.mark.parametrize("shape", [(96, 96), (128, 96)])
@pytest.mark.parametrize("train", [True, False])
def test_listdataset_gpu_decode_equals_host_decode(tmp_path, shape, train):
    import random
    from singleshotpose_b200 import dataset, synth
    listfile, bgs = synth.write_linemod_like(str(tmp_path), n=6, ow=160, oh=120, fmt="jpg")
    out = {}
    for gd in (False, True):
        random.seed(3)
        ds = dataset.listDataset(listfile, shape=shape, shuffle=False, train=train, bg_file_names=bgs, batch_size=6,
                                 num_workers=1, gpu_decode=gd, cell_size=shape[0] // 13)   # the training schedule's size: 13 cells
        samples = [ds[i] for i in range(len(ds))]
        if gd:
            assert isinstance(samples[0]["img"], bytes)
        coll = dataset.GpuCollate("cuda")
        out[gd] = coll(samples)
        if gd:
            assert coll._jpeg.launches == 3 and coll._jpeg.fallbacks == 0         # one decoder call for the whole batch
    assert torch.equal(out[True][0], out[False][0]) and torch.equal(out[True][1], out[False][1])
