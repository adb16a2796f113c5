"""JPEG decoding on the GPU, byte-identical to what the reference's loader gets from Pillow:
`Image.open(path).convert('RGB')` (dataset.py, image.py) on a Pillow built on libjpeg-turbo.

  read_jpeg_size(data)   (w, h) from the frame header, pure Python: loader workers need the size for their random draws
                         without decoding and without loading CUDA.
  GpuJpegDecoder(device) decodes a list of file contents in one batch: one pinned staging fill, one host->device copy, three
                         launches (csrc/jpeg.cu) and one device->host copy of the per-image status words.  Files the GPU path
                         declines (progressive, arithmetic, CMYK, RGB-coded, 12-bit, other samplings, multi-scan, no EOI, ...)
                         or flags while decoding (corrupt entropy data, blocks where libjpeg-turbo's SIMD and C IDCT can
                         differ) are decoded by Pillow on the host and uploaded, so every result equals Pillow's; an exception
                         Pillow raises (a truncated file, say) propagates as it would in the reference.
  decode_jpeg(data)      one file.
"""
from __future__ import annotations

import collections
import ctypes as C
import io

import numpy as np
import torch
from PIL import Image

from ._lib import STRUCTS, SspError, call, load, stream_ptr

_SOF = {0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF}
STATUS_BITS = {1: "corrupt entropy-coded data", 2: "IDCT outside the SIMD/C agreement range", 4: "restart marker structure",
               8: "DC value outside int32"}


_Info, _Item = STRUCTS["ssp_jpeg_info"], STRUCTS["ssp_jpeg_item"]


def read_jpeg_size(data):
    """(width, height) of a JPEG from its first SOF marker, or None if `data` is not a JPEG or has no frame header."""
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return None
    p = 2
    while p < n:
        if data[p] != 0xFF:
            return None
        while p < n and data[p] == 0xFF:
            p += 1
        if p + 2 >= n:
            return None
        m = data[p]
        p += 1
        if m == 0x01 or 0xD0 <= m <= 0xD7:
            continue
        if m in (0xD9, 0xDA):
            return None
        if m in _SOF:
            return (data[p + 5] << 8 | data[p + 6], data[p + 3] << 8 | data[p + 4]) if p + 7 <= n else None
        p += data[p] << 8 | data[p + 1]
    return None


def _pillow_rgb(b):
    return np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


class GpuJpegDecoder:
    """Batched JPEG decoder.  Counters: `fallbacks` (images Pillow decoded), `fallback_reasons` (Counter of reason text),
    `h2d_bytes` (last call), `launches` (total), `serial_subsequences` (last call: 1024-bit subsequences whose decoder state no
    speculative candidate linked to, decoded serially -- the part of the entropy decode that did not run in parallel)."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self.fallbacks = 0
        self.fallback_reasons = collections.Counter()
        self.h2d_bytes = 0
        self.launches = 0
        self.serial_subsequences = 0
        self._stage = self._dev = self._work = self._status = self._status_h = None

    def _fallback(self, b, reason):
        self.fallbacks += 1
        self.fallback_reasons[reason] += 1
        a = _pillow_rgb(b)
        self.h2d_bytes += a.nbytes
        return torch.from_numpy(np.ascontiguousarray(a)).to(self.device)

    def __call__(self, blobs):
        with torch.cuda.device(self.device):        # buffers, launches and the wait all on the decoder's device
            return self._decode([bytes(b) for b in blobs])

    def _decode(self, blobs):
        lib = load()
        info = _Info()
        gpu, declined = [], []
        for i, b in enumerate(blobs):
            rc = lib.ssp_jpeg_parse(b, len(b), C.byref(info))
            if rc < 0:
                raise SspError("ssp_jpeg_parse failed (%d): %s" % (rc, lib.ssp_last_error().decode()))
            if rc == 0:
                gpu.append((i, info.height, info.width))
            else:
                declined.append((i, lib.ssp_jpeg_decline_reason(rc).decode()))
        outs = [None] * len(blobs)
        self.h2d_bytes = 0
        m = len(gpu)
        if m:
            total = sum(h * w * 3 for _, h, w in gpu)
            flat = torch.empty(total, dtype=torch.uint8, device=self.device)
            items = (_Item * m)()
            at = 0
            for k, (i, h, w) in enumerate(gpu):
                outs[i] = flat[at:at + h * w * 3].view(h, w, 3)
                items[k] = _Item(C.cast(C.c_char_p(blobs[i]), C.c_void_p), len(blobs[i]), outs[i].data_ptr())
                at += h * w * 3
            stage_bytes = int(lib.ssp_jpeg_stage_bytes(items, m))
            work_bytes = int(lib.ssp_jpeg_work_bytes(items, m))
            if stage_bytes < 0 or work_bytes < 0:
                raise SspError("ssp_jpeg sizes failed: %s" % lib.ssp_last_error().decode())
            if self._stage is None or self._stage.numel() < stage_bytes:
                self._stage = torch.empty(stage_bytes, dtype=torch.uint8).pin_memory()
                self._dev = torch.empty(stage_bytes, dtype=torch.uint8, device=self.device)
            if self._work is None or self._work.numel() < work_bytes:
                self._work = torch.empty(max(work_bytes, 16), dtype=torch.uint8, device=self.device)
            if self._status is None or self._status.numel() < 3 * m:
                self._status = torch.empty(3 * m, dtype=torch.int32, device=self.device)
                self._status_h = torch.empty(3 * m, dtype=torch.int32).pin_memory()
            dims = (C.c_longlong * 4)()
            call("ssp_jpeg_batch_plan", items, m, C.c_void_p(self._stage.data_ptr()), stage_bytes, dims)
            used = int(dims[3])
            self._dev[:used].copy_(self._stage[:used], non_blocking=True)
            self.h2d_bytes += used
            call("ssp_jpeg_batch_run", C.c_void_p(self._dev.data_ptr()), m, dims, C.c_void_p(self._work.data_ptr()),
                 self._work.numel(), C.c_void_p(self._status.data_ptr()), stream_ptr())
            self.launches += 3
            self._status_h[:3 * m].copy_(self._status[:3 * m], non_blocking=True)
        for i, reason in declined:                 # Pillow works while the device decodes
            outs[i] = self._fallback(blobs[i], reason)
        if m:
            torch.cuda.current_stream(self.device).synchronize()
            sh = self._status_h[:3 * m].tolist()
            st = [a | b for a, b in zip(sh[:m], sh[m:2 * m])]
            self.serial_subsequences = sum(sh[2 * m:])
            for (i, _, _), s in zip(gpu, st):
                if s:
                    reason = ", ".join(v for bit, v in STATUS_BITS.items() if s & bit)
                    outs[i] = self._fallback(blobs[i], reason)
        return outs


_default = {}


def decode_jpeg(data, device="cuda"):
    """One JPEG file's bytes -> (H, W, 3) uint8 CUDA tensor, equal to np.asarray(Image.open(f).convert('RGB'))."""
    dev = torch.device(device)
    if dev not in _default:
        _default[dev] = GpuJpegDecoder(dev)
    return _default[dev]([data])[0]
