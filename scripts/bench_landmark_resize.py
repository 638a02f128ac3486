"""Pose frames at sizes other than 512 x 512: the reference's host path against the device path, at L = 150 and 300 frames
(5 and 10 s at 30 fps), median of --calls calls after one warm-up, for the two script arms that resize the canvas.

  vid2vid   a 1080 x 1920 (W x H) source video: keypoints projected at the source size, drawn at it and resized to
            512 x 512 (scripts/vid2vid.py:194-200).
  audio2vid -W 768 -H 768: keypoints projected at 768 x 768 and drawn at it (scripts/audio2vid.py:199-218).

  host    per frame: the mediapipe drawing loop (oracle/mediapipe_shim, on cv2.line) + the cv2.resize calls of the script,
          then the pipeline's pose intake (_pose_maps_to_tensor: pinned staging, copy, 2x - 1). Skipped when cv2 does
          not import.
  device  projection (project_points_with_trans from the host meshes, or project_points from the fp32 mesh offsets
          already on the device) + vis.draw_pose_frames + the pipeline's intake of the CUDA uint8 frames.

The host projection is not timed (the numpy projection is not part of the product). `identical` compares the two arms'
intake tensors. Edge table and mesh: the forehead_edge=False spec and the seeded mesh of
tests/golden/landmark_frames_reference.npz.

    python scripts/bench_landmark_resize.py [--calls 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types
from collections import namedtuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aniportrait_b200.pipelines import landmarks as LM  # noqa: E402
from aniportrait_b200.pipelines.pipeline_pose2vid_long import Pose2VideoPipeline  # noqa: E402

Spec = namedtuple("Spec", "color thickness circle_radius")


def median_ms(fn, calls):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = np.load(os.path.join(ROOT, "tests", "golden", "landmark_frames_reference.npz"))
    spec = {tuple(int(v) for v in e): Spec(tuple(int(v) for v in c), 2, 1)
            for e, c in zip(g["spec0_edges"], g["spec0_colors"])}
    vis = LM.enable_kernels(types.SimpleNamespace(face_connection_spec=spec))
    holder = types.SimpleNamespace(cond_image_processor=None)
    try:
        sys.path.insert(0, os.path.join(ROOT, "oracle", "mediapipe_shim"))
        import cv2
        from mediapipe.solutions import drawing_utils
        from mediapipe.framework.formats import landmark_pb2
    except ImportError:
        cv2 = None
    gpu = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"

    def host_draw(verts, size):
        """FaceMeshVisualizer.draw_landmarks(size, verts): the 512 x 512 canvas, then cv2.resize to size."""
        image = np.zeros((512, 512, 3), dtype=np.uint8)
        lms = landmark_pb2.NormalizedLandmarkList()
        for i in range(verts.shape[0]):
            lm = lms.landmark.add()
            lm.x = verts[i, 0] / size[0]
            lm.y = verts[i, 1] / size[1]
            lm.z = 1.0
        drawing_utils.draw_landmarks(image=image, landmark_list=lms, connections=spec.keys(),
                                     landmark_drawing_spec=None, connection_drawing_spec=spec)
        return cv2.resize(image, size)

    rng = np.random.default_rng(0)
    for L in (150, 300):
        # vid2vid: per-frame meshes and matrices from the host, 1080 x 1920 source, 512 x 512 output
        src_w, src_h = 1080, 1920
        pick = rng.integers(0, len(g["vid_verts"]), L)
        verts = g["vid_verts"][pick] + rng.standard_normal((L, 468, 3)) * 0.2
        mats = g["vid_mats"][pick]
        kp_vid = LM.project_points_with_trans(verts, mats, [src_h, src_w]).cpu().numpy()
        # audio2vid at 768 x 768: fp32 offsets on the device
        side = 768
        offs = (rng.standard_normal((L, 468, 3)) * 0.2).astype(np.float32)
        poses = g["pose_seq"][rng.integers(0, len(g["pose_seq"]), L)]
        kp_a2v = LM.project_points(offs, g["trans_mat"], poses, [side, side], base=g["mesh_base"]).cpu().numpy()
        offs_dev = torch.from_numpy(offs).to(dev)

        def device_vid2vid():
            kp = LM.project_points_with_trans(verts, mats, [src_h, src_w])
            frames = vis.draw_pose_frames((src_w, src_h), kp, out_size=(512, 512))
            return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, 512, 512, dev)

        def device_audio2vid():
            kp = LM.project_points(offs_dev, g["trans_mat"], poses, [side, side], base=g["mesh_base"])
            frames = vis.draw_pose_frames((side, side), kp)
            return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, side, side, dev)

        def host_vid2vid():
            frames = [cv2.resize(host_draw(v, (src_w, src_h)), (512, 512)) for v in kp_vid]
            return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, 512, 512, dev)

        def host_audio2vid():
            frames = [cv2.resize(host_draw(v, (side, side)), (side, side)) for v in kp_a2v]
            return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, side, side, dev)

        arms = [("vid2vid", f"{src_w}x{src_h}->512x512", device_vid2vid, host_vid2vid),
                ("audio2vid", f"{side}x{side}", device_audio2vid, host_audio2vid)]
        for arm, sizes, device_arm, host_arm in arms:
            res = {"arm": arm, "sizes": sizes, "L": L, "gpu": gpu, "power_limit": power}
            res["device_ms"] = median_ms(device_arm, args.calls)
            if cv2 is not None:
                res["host_ms"] = median_ms(host_arm, args.calls)
                res["identical"] = bool(torch.equal(host_arm(), device_arm()))
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
