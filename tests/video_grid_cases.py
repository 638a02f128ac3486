"""Seeded inputs shaped like the tail of each reference script (the frames beside the result, the reference image and the
decoded video, in the scripts' tile order), shared by oracle/make_golden_video_grid.py, which runs the unmodified
save_videos_grid on them, and the tests, which rebuild the same inputs from the seeds.

A case is (n_rows, (height, width), tiles); a tile is
  ("frames", uint8 [T', h, w, 3], bgr)  frames at their own size that go through the script's pose_transform
                                        (transforms.Resize((height, width)) + ToTensor); bgr: cv2.cvtColor(BGR2RGB) first
  ("video", fp32 [1, 3, T, height, width], False)  the pipeline's video (fp16 values widened) or the frame
                                        interpolator's fp32 output
The reference image is a one-frame "frames" tile, repeated over T as the scripts repeat it.
"""
from __future__ import annotations

import hashlib

import numpy as np


def _frames(rng, n, h, w):
    return rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def _video(rng, T, h, w, fp16=True):
    v = rng.random((1, 3, T, h, w), dtype=np.float32)
    return v.astype(np.float16).astype(np.float32) if fp16 else v


def cases():
    """name -> (n_rows, (height, width), tiles), rebuilt from fixed seeds."""
    out = {}
    r = np.random.default_rng(1001)
    # audio2vid (audio2vid.py:207-260): the BGR pose frames are drawn at the output size; one more frame than the video
    out["audio2vid_40x56"] = (3, (40, 56), [("frames", _frames(r, 1, 77, 53), False),
                                            ("frames", _frames(r, 4, 40, 56), True), ("video", _video(r, 3, 40, 56), False)])
    r = np.random.default_rng(1002)
    out["audio2vid_512"] = (3, (512, 512), [("frames", _frames(r, 1, 640, 480), False),
                                            ("frames", _frames(r, 2, 512, 512), True), ("video", _video(r, 2, 512, 512), False)])
    r = np.random.default_rng(1003)
    out["audio2vid_768"] = (3, (768, 768), [("frames", _frames(r, 1, 512, 512), False),
                                            ("frames", _frames(r, 2, 768, 768), True), ("video", _video(r, 2, 768, 768), False)])
    # vid2vid (vid2vid.py:147-162, 228-243): a 60 fps source is read with step 2; tiles [ref, video, source]
    r = np.random.default_rng(1004)
    src = _frames(r, 4, 1920, 1080)[::2]
    out["vid2vid_1080x1920_step2"] = (3, (512, 512), [("frames", _frames(r, 1, 700, 500), False),
                                                      ("video", _video(r, 2, 512, 512), False), ("frames", src, False)])
    r = np.random.default_rng(1005)
    out["vid2vid_1920x1080"] = (3, (512, 512), [("frames", _frames(r, 1, 512, 512), False),
                                                ("video", _video(r, 2, 512, 512), False),
                                                ("frames", _frames(r, 2, 1080, 1920), False)])
    # pose2vid (pose2vid.py:146-151, 181-196): a pose video at another size
    r = np.random.default_rng(1006)
    out["pose2vid_48x64"] = (3, (48, 64), [("frames", _frames(r, 1, 33, 47), False),
                                           ("frames", _frames(r, 3, 90, 70), False), ("video", _video(r, 3, 48, 64), False)])
    # app.py:258-262: n_rows=1 and the video alone (make_grid returns the frame itself, no padding)
    r = np.random.default_rng(1007)
    out["app_40x56"] = (1, (40, 56), [("video", _video(r, 3, 40, 56), False)])
    # -acc: the frame interpolator's fp32 output is shorter than the pose frames
    r = np.random.default_rng(1008)
    out["acc_40x56"] = (3, (40, 56), [("frames", _frames(r, 1, 40, 56), False),
                                      ("frames", _frames(r, 5, 40, 56), True), ("video", _video(r, 3, 40, 56, fp16=False), False)])
    return out


def input_digest(tiles):
    """SHA-256 of every tile's bytes: pins the generator the goldens were made from."""
    h = hashlib.sha256()
    for tile in tiles:
        h.update(np.ascontiguousarray(tile[1]).tobytes())
    return h.hexdigest()


def frames_digest(frames):
    return hashlib.sha256(np.ascontiguousarray(frames).tobytes()).hexdigest()


def restated_grid(case):
    """The grid frames of a case from the numpy restatements alone: Pillow's resize (pil_resize_reference), the ToTensor
    round trip, the channel swap of cvtColor(BGR2RGB), the repeat / cut to T and make_grid."""
    import pil_resize_reference as PR
    n_rows, (height, width), tiles = case
    T = next(t[1].shape[2] for t in tiles if t[0] == "video")
    parts = []
    for kind, data, bgr in tiles:
        if kind == "video":
            parts.append(PR.video_bytes(data[0]).transpose(1, 2, 3, 0))
            continue
        frames = PR.resize_frames(data[:T], (width, height))
        frames = PR.to_tensor_bytes(frames[..., ::-1] if bgr else frames)
        parts.append(np.repeat(frames, T, 0) if len(frames) == 1 else frames)
    return PR.compose_grid(parts, n_rows)
