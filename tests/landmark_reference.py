"""Integer restatement of the landmark rasteriser (mediapipe `drawing_utils.draw_landmarks` with connections only, on
OpenCV's `cv2.line(img, p0, p1, color, 2)` in LINE_8 mode) and of the landmark conversion in front of it, in plain Python
integers and numpy. It walks the scanlines and Bresenham steps the way OpenCV's drawing code does (ThickLine ->
FillConvexPoly in 16.16 fixed point, the polygon outline with Line2, radius-1 filled end caps), so that the device kernel's
closed-form row expressions are checked against an independent formulation.

Only segments whose two endpoints lie on the canvas are restated: `draw_landmarks` drops every landmark outside [0, 1]
before it draws, so cv2 never receives any other kind.
"""
from __future__ import annotations

import math
import sys

import numpy as np

CANVAS = 512
XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
HALF = XY_ONE >> 1
# the radius-1 filled circle cv2 draws at each end of a thick line (what it draws for a zero-length segment)
CAP = ((0, -1), (-1, 0), (0, 0), (1, 0), (0, 1))


def _put(img, x, y, c):
    H, W = img.shape[:2]
    if 0 <= x < W and 0 <= y < H:
        img[y, x] = c


def _div_trunc(a, b):
    """C integer division (rounds toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def _clip_line(W, H, p1, p2):
    """Cohen-Sutherland clip of a 16.16 segment to the (W x H) << 16 rectangle, with the intercepts rounded as a double
    quotient truncated toward zero (Python's int / int is the correctly rounded double quotient)."""
    right, bottom = W - 1, H - 1
    (x1, y1), (x2, y2) = p1, p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int((a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int((a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int((a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int((a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, (x1, y1), (x2, y2)


def line2(img, p1, p2, c):
    """One-pixel line between 16.16 points (OpenCV's Line2)."""
    H, W = img.shape[:2]
    ok, (x1, y1), (x2, y2) = _clip_line(W << XY_SHIFT, H << XY_SHIFT, p1, p2)
    if not ok:
        return
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            dy = -dy
            x1, x2, y1, y2 = x2, x1, y2, y1
        x_step, y_step = XY_ONE, _div_trunc(dy << XY_SHIFT, ax | 1)
        ecount = (x2 - x1) >> XY_SHIFT
    else:
        if dy < 0:
            dx = -dx
            x1, x2, y1, y2 = x2, x1, y2, y1
        x_step, y_step = _div_trunc(dx << XY_SHIFT, ay | 1), XY_ONE
        ecount = (y2 - y1) >> XY_SHIFT
    x1 += HALF
    y1 += HALF
    _put(img, (x2 + HALF) >> XY_SHIFT, (y2 + HALF) >> XY_SHIFT, c)
    for _ in range(ecount + 1):
        _put(img, x1 >> XY_SHIFT, y1 >> XY_SHIFT, c)
        x1 += x_step
        y1 += y_step


def fill_convex(img, v, c):
    """Scanline fill of a convex polygon of 16.16 vertices plus its outline (OpenCV's FillConvexPoly, LINE_8)."""
    H, W = img.shape[:2]
    npts = len(v)
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    imin = 0
    p0 = v[-1]
    for k, p in enumerate(v):
        if p[1] < ymin:
            ymin, imin = p[1], k
        ymax = max(ymax, p[1])
        xmax = max(xmax, p[0])
        xmin = min(xmin, p[0])
        line2(img, p0, p, c)
        p0 = p
    xmin, xmax = (xmin + HALF) >> XY_SHIFT, (xmax + HALF) >> XY_SHIFT
    ymin, ymax = (ymin + HALF) >> XY_SHIFT, (ymax + HALF) >> XY_SHIFT
    if npts < 3 or xmax < 0 or ymax < 0 or xmin >= W or ymin >= H:
        return
    ymax = min(ymax, H - 1)
    edge = [dict(idx=imin, ye=ymin, di=1, x=-XY_ONE, dx=0), dict(idx=imin, ye=ymin, di=npts - 1, x=-XY_ONE, dx=0)]
    y = ymin
    edges = npts
    while True:
        for e in edge:
            if y >= e["ye"]:
                idx0 = e["idx"]
                idx = (idx0 + e["di"]) % npts
                while True:
                    edges -= 1
                    if edges < 0:
                        break
                    ty = (v[idx][1] + HALF) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        e["ye"] = ty
                        e["dx"] = _div_trunc((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        e["x"] = xs
                        e["idx"] = idx
                        break
                    idx0 = idx
                    idx = (idx + e["di"]) % npts
        if edges < 0:
            break
        if y >= 0:
            lo, hi = sorted((edge[0]["x"], edge[1]["x"]))
            xx1, xx2 = (lo + HALF) >> XY_SHIFT, (hi + HALF) >> XY_SHIFT
            if xx2 >= 0 and xx1 < W:
                img[y, max(xx1, 0):min(xx2, W - 1) + 1] = c
        edge[0]["x"] += edge[0]["dx"]
        edge[1]["x"] += edge[1]["dx"]
        y += 1
        if y > ymax:
            break


def thick_line2(img, p0, p1, c):
    """cv2.line(img, p0, p1, c, thickness=2) for integer pixel endpoints on the canvas."""
    p0 = (p0[0] << XY_SHIFT, p0[1] << XY_SHIFT)
    p1 = (p1[0] << XY_SHIFT, p1[1] << XY_SHIFT)
    dx = (p0[0] - p1[0]) / XY_ONE
    dy = (p1[1] - p0[1]) / XY_ONE
    r = dx * dx + dy * dy
    if abs(r) > sys.float_info.epsilon:
        r = XY_ONE / math.sqrt(r)          # thickness 2 << (XY_SHIFT - 1)
        dpx, dpy = int(np.rint(dy * r)), int(np.rint(dx * r))   # cvRound: round half to even
        fill_convex(img, [(p0[0] + dpx, p0[1] + dpy), (p0[0] - dpx, p0[1] - dpy),
                          (p1[0] - dpx, p1[1] - dpy), (p1[0] + dpx, p1[1] + dpy)], c)
    for p in (p0, p1):
        cx, cy = p[0] >> XY_SHIFT, p[1] >> XY_SHIFT
        for ox, oy in CAP:
            _put(img, cx + ox, cy + oy, c)


def landmark_pixels(keypoints, image_size, normed):
    """keypoints [N, C >= 2] -> (int pixel coordinates [N, 2], kept [N]) as draw_landmarks derives them: the protobuf float32
    x / y (divided by image_size in float64 first unless normed), kept iff both lie in [0, 1] (NaN is dropped), pixel
    min(floor(v * 512), 511)."""
    kp = np.asarray(keypoints, dtype=np.float64)[:, :2]     # draw_util.py reads columns 0 and 1 only
    if normed:
        xy = kp.astype(np.float32)
    else:
        with np.errstate(over="ignore", invalid="ignore"):
            xy = np.stack([kp[:, 0] / image_size[0], kp[:, 1] / image_size[1]], 1).astype(np.float32)
    xy = xy.astype(np.float64)
    with np.errstate(invalid="ignore"):
        kept = np.all((xy >= 0.0) & (xy <= 1.0), axis=1)
    px = np.zeros(kp.shape, dtype=np.int64)
    px[kept] = np.minimum(np.floor(xy[kept] * CANVAS), CANVAS - 1).astype(np.int64)
    return px, kept


def draw_frame(keypoints, edges, colors, image_size=(CANVAS, CANVAS), normed=False):
    """One frame of FaceMeshVisualizer.draw_landmarks: uint8 [512, 512, 3], edges drawn in table order (later edges
    overwrite earlier ones), colour bytes in channel order."""
    edges = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    colors = np.asarray(colors, dtype=np.uint8).reshape(-1, 3)
    n = len(keypoints)
    if ((edges < 0) | (edges >= n)).any():
        raise ValueError("landmark index out of range")
    px, kept = landmark_pixels(keypoints, image_size, normed)
    img = np.zeros((CANVAS, CANVAS, 3), dtype=np.uint8)
    for (a, b), c in zip(edges, colors):
        if kept[a] and kept[b]:
            thick_line2(img, (int(px[a, 0]), int(px[a, 1])), (int(px[b, 0]), int(px[b, 1])), c)
    return img


def draw_frames(keypoints, edges, colors, image_size=(CANVAS, CANVAS), normed=False):
    """keypoints [L, N, 2] -> uint8 [L, 512, 512, 3]."""
    return np.stack([draw_frame(k, edges, colors, image_size, normed) for k in keypoints], 0)


def project_points(points_3d, matrices, proj, image_shape):
    """Per-point part of pose_util.project_points(_with_trans): (X_h . M^T) . P left to right with every dot product
    summed k = 0..3 in float64, then divide by w and map [-1, 1] to pixels. points_3d [L, N, 3] float64, matrices
    [L, 4, 4], proj the float32-built 4x4 P promoted to float64; image_shape (H, W)."""
    pts = np.asarray(points_3d, dtype=np.float64)
    L, N, _ = pts.shape
    xh = np.concatenate([pts, np.ones((L, N, 1))], axis=2)
    out = np.zeros((L, N, 2))
    for i in range(L):
        m = np.asarray(matrices[i], dtype=np.float64)
        t = [((xh[i, :, 0] * m[j, 0] + xh[i, :, 1] * m[j, 1]) + xh[i, :, 2] * m[j, 2]) + xh[i, :, 3] * m[j, 3]
             for j in range(4)]
        u = [((t[0] * proj[0, j] + t[1] * proj[1, j]) + t[2] * proj[2, j]) + t[3] * proj[3, j] for j in range(4)]
        out[i, :, 0] = (u[0] / u[3] + 1) * 0.5 * image_shape[1]
        out[i, :, 1] = (u[1] / u[3] + 1) * 0.5 * image_shape[0]
    return out
