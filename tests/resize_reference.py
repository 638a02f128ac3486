"""Integer restatement of OpenCV's `cv2.resize(img, (W, H))` with the default INTER_LINEAR on 8-bit, 3-channel images,
in numpy: the fixed-point coefficient tables, the horizontal pass into int32 and the vertical pass as cv2's vectorised
kernel rounds it. It is what the reference's FaceMeshVisualizer.draw_landmarks (src/utils/draw_util.py:146) and the
scripts (scripts/vid2vid.py:199-200) apply to the 512 x 512 landmark canvas, and what ap_resize_linear_u8 is checked
against.

  - scale = 1 / (dst / src) in double; per destination index d, f = (float)((d + 0.5) * scale - 0.5), s = floor(f),
    f -= s in float; coefficients rint((1 - f) * 2048) and rint(f * 2048) (round half to even).
  - Columns: s < 0 gives s = 0, f = 0 and s >= src - 1 gives s = src - 1, f = 0; the second tap is min(s + 1, src - 1).
  - Rows: f is not clamped; only the two row indices s and s + 1 are clipped to [0, src - 1].
  - Horizontal: H = p[s] * c0 + p[s1] * c1 (int32). Vertical: ((((H0 >> 4) * b0) >> 16) + (((H1 >> 4) * b1) >> 16) + 2)
    >> 2, saturated to uint8.

cv2 copies a same-size image and takes its INTER_AREA path for an exact 2x downscale on both axes; the formula above
gives the same bytes in both cases (the identity, and (a + b + c + d + 2) >> 2), so neither needs its own branch.
"""
from __future__ import annotations

import numpy as np

COEF_BITS = 11
COEF_SCALE = 1 << COEF_BITS


def axis_taps(src: int, dst: int, clamp_f: bool):
    """(i0, i1, c0, c1) int64 arrays [dst]: the two source indices and fixed-point weights of every destination index."""
    scale = 1.0 / (float(dst) / float(src))
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_f:
        lo = s < 0
        s[lo], f[lo] = 0, 0
        hi = s >= src - 1
        s[hi], f[hi] = src - 1, 0
    one = np.float32(1.0)
    c0 = np.rint((one - f) * np.float32(COEF_SCALE)).astype(np.int64)
    c1 = np.rint(f * np.float32(COEF_SCALE)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), c0, c1


def resize(img, size):
    """cv2.resize(img, size) for uint8 img [h, w, 3] and size = (W, H) -> uint8 [H, W, 3]."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3, (img.dtype, img.shape)
    h, w = img.shape[:2]
    W, H = int(size[0]), int(size[1])
    x0, x1, a0, a1 = axis_taps(w, W, clamp_f=True)
    y0, y1, b0, b1 = axis_taps(h, H, clamp_f=False)
    p = img.astype(np.int64)

    def horizontal(rows):                  # [H, W, 3] int32 values of the horizontal pass on the given source rows
        r = p[rows]
        return r[:, x0] * a0[None, :, None] + r[:, x1] * a1[None, :, None]

    v = ((((horizontal(y0) >> 4) * b0[:, None, None]) >> 16)
         + (((horizontal(y1) >> 4) * b1[:, None, None]) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def resize_frames(frames, size):
    """[L, h, w, 3] -> [L, H, W, 3], frame by frame."""
    return np.stack([resize(f, size) for f in frames], 0)
