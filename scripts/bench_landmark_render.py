"""Pose-frame rendering time: the reference's host path against the device path, at L = 150 and 300 frames (5 and 10 s of
audio at 30 fps), median of --calls calls after one warm-up.

  host    per frame: the mediapipe drawing loop (oracle/mediapipe_shim, on cv2.line) + cv2.resize, then the pipeline's
          pose intake (_pose_maps_to_tensor: pinned staging, copy, 2x - 1). Skipped when cv2 does not import.
  device  project_points (fp32 mesh offsets already on the device) + draw_landmarks_batch (one launch) + the pipeline's
          intake of the CUDA uint8 frames.

The projection of the host arm is not timed (the numpy projection is not part of the product). Edge table and mesh: the
forehead_edge=False spec and the seeded mesh of tests/golden/landmark_frames_reference.npz.

    python scripts/bench_landmark_render.py [--calls 5]
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
    rng = np.random.default_rng(0)
    for L in (150, 300):
        offs = (rng.standard_normal((L, 468, 3)) * 0.2).astype(np.float32)
        poses = g["pose_seq"][rng.integers(0, len(g["pose_seq"]), L)]
        kp_host = LM.project_points(offs, g["trans_mat"], poses, [512, 512], base=g["mesh_base"]).cpu().numpy()
        offs_dev = torch.from_numpy(offs).to(dev)
        res = {"L": L, "gpu": gpu, "power_limit": power}

        def device_arm():
            kp = LM.project_points(offs_dev, g["trans_mat"], poses, [512, 512], base=g["mesh_base"])
            frames = vis.draw_landmarks_batch((512, 512), kp)
            return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, 512, 512, dev)
        res["device_ms"] = median_ms(device_arm, args.calls)
        if cv2 is not None:
            def host_arm():
                frames = []
                for verts in kp_host:
                    image = np.zeros((512, 512, 3), dtype=np.uint8)
                    lms = landmark_pb2.NormalizedLandmarkList()
                    for i in range(verts.shape[0]):
                        lm = lms.landmark.add()
                        lm.x = verts[i, 0] / 512
                        lm.y = verts[i, 1] / 512
                        lm.z = 1.0
                    drawing_utils.draw_landmarks(image=image, landmark_list=lms, connections=spec.keys(),
                                                 landmark_drawing_spec=None, connection_drawing_spec=spec)
                    frames.append(cv2.resize(image, (512, 512)))
                return Pose2VideoPipeline._pose_maps_to_tensor(holder, frames, 512, 512, dev)
            res["host_ms"] = median_ms(host_arm, args.calls)
            same = torch.equal(host_arm(), device_arm())
            res["identical"] = bool(same)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
