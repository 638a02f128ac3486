"""Restatement of Pillow's `Image.resize(size, Image.BILINEAR)` on 8-bit RGB images (libImaging/Resample.c), in numpy,
and of the comparison grid the reference's scripts save (torchvision.utils.make_grid inside src/utils/util.py:87-104
save_videos_grid). It is what the scripts' `transforms.Resize((height, width))` does to every frame shown beside the
result, and what ap_resize_pil_bilinear_u8 and ap_video_grid_u8 are checked against.

Per axis, in -> out (box (0, 0, in_w, in_h)), in double:
  scale = in / out, fs = max(scale, 1), support = fs (the bilinear support is 1), ss = 1 / fs.
  Output index xx: center = (xx + 0.5) * scale, xmin = max((int)(center - support + 0.5), 0),
  n = min((int)(center + support + 0.5), in) - xmin taps; tap x has w = max(1 - |t|, 0), t = (x + xmin - center + 0.5) * ss;
  the weights are summed in tap order into ww and each divided by ww (when ww != 0); fixed point (int)(0.5 + w * 2^22).
Passes: horizontal first, over the source rows the vertical pass reads, each sum 2^21 + sum(p * k) >> 22 clamped to
0..255 and stored as uint8; then the vertical pass with the same rounding. A pass runs only if its axis changes size; a
same-size resize is a copy.
"""
from __future__ import annotations

import numpy as np

PRECISION_BITS = 22


def coeffs(n_in: int, n_out: int):
    """(xmin int64 [n_out], taps int64 [n_out], k int64 [n_out, ksize]) of Pillow's precompute_coeffs +
    normalize_coeffs_8bpc for the bilinear filter; k is zero beyond each index's taps."""
    scale = float(n_in) / n_out
    fs = max(scale, 1.0)
    support = fs
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    xmin = np.zeros(n_out, np.int64)
    taps = np.zeros(n_out, np.int64)
    k = np.zeros((n_out, ksize), np.int64)
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), n_in) - lo
        w = []
        ww = 0.0
        for x in range(n):
            t = abs((x + lo - center + 0.5) * ss)
            v = 1.0 - t if t < 1.0 else 0.0
            w.append(v)
            ww += v
        for x in range(n):
            v = w[x] / ww if ww != 0.0 else w[x]
            k[xx, x] = int(0.5 + v * (1 << PRECISION_BITS))
        xmin[xx], taps[xx] = lo, n
    return xmin, taps, k


def _pass(rows, n_out, axis_coeffs):
    """One 8-bit pass along axis 1 of int64 [R, n_in, 3] -> uint8 [R, n_out, 3]."""
    xmin, taps, k = axis_coeffs
    acc = np.full((rows.shape[0], n_out, 3), 1 << (PRECISION_BITS - 1), np.int64)
    for j in range(k.shape[1]):
        idx = np.minimum(xmin + j, rows.shape[1] - 1)
        kj = np.where(j < taps, k[:, j], 0)
        acc += rows[:, idx, :] * kj[None, :, None]
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize(img, size):
    """Image.fromarray(img).resize(size, Image.BILINEAR) for uint8 img [h, w, 3] and size = (W, H) -> uint8 [H, W, 3]."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3, (img.dtype, img.shape)
    h, w = img.shape[:2]
    W, H = int(size[0]), int(size[1])
    ymin, ytaps, ky = coeffs(h, H)
    first, last = int(ymin[0]), int(ymin[-1] + ytaps[-1])
    out = img
    if W != w:                                   # only the source rows [first, last) the vertical pass reads
        out = _pass(img[first:last].astype(np.int64), W, coeffs(w, W))
        ymin = ymin - first
    else:
        out = img[first:last] if H != h else img
        ymin = ymin - first
    if H != h:
        t = np.ascontiguousarray(out.astype(np.int64).transpose(1, 0, 2))      # rows <-> columns
        out = _pass(t, H, (ymin, ytaps, ky)).transpose(1, 0, 2)
    return np.ascontiguousarray(out)


def resize_frames(frames, size):
    """[L, h, w, 3] -> [L, H, W, 3], frame by frame."""
    return np.stack([resize(f, size) for f in frames], 0)


def to_tensor_bytes(u8):
    """The bytes save_videos_grid writes for a uint8 frame that went through ToTensor: trunc(fl(fl(v / 255) * 255))
    in fp32 — which is v again for every byte value (pinned by tests/test_pil_resize_cpu.py)."""
    x = np.asarray(u8).astype(np.float32) / np.float32(255)
    return (x * np.float32(255)).astype(np.uint8)


def video_bytes(x):
    """(x * 255).astype(uint8) of save_videos_grid on fp32 values in [0, 1]: trunc(fl(x * 255))."""
    return (np.asarray(x, dtype=np.float32) * np.float32(255)).astype(np.uint8)


def grid_geometry(B: int, n_rows: int, H: int, W: int):
    """(xmaps, ymaps, GH, GW) of torchvision.utils.make_grid(padding=2) for B tiles of H x W; B = 1 is the tile itself."""
    if B == 1:
        return 1, 1, H, W
    xmaps = min(n_rows, B)
    ymaps = -(-B // xmaps)
    return xmaps, ymaps, ymaps * (H + 2) + 2, xmaps * (W + 2) + 2


def compose_grid(tiles, n_rows: int):
    """uint8 [T, GH, GW, 3] grid frames of uint8 tiles [T, H, W, 3] (already the bytes of each tile), padding 0."""
    B = len(tiles)
    T, H, W, _ = tiles[0].shape
    xmaps, _, GH, GW = grid_geometry(B, n_rows, H, W)
    if B == 1:
        return np.array(tiles[0], dtype=np.uint8)
    out = np.zeros((T, GH, GW, 3), np.uint8)
    for i, t in enumerate(tiles):
        y, x = 2 + (i // xmaps) * (H + 2), 2 + (i % xmaps) * (W + 2)
        out[:, y:y + H, x:x + W] = t
    return out
