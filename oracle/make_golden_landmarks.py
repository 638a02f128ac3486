"""TEST INFRASTRUCTURE — generates tests/golden/landmark_frames_reference.npz by running the UNMODIFIED reference
FaceMeshVisualizer.draw_landmarks (src/utils/draw_util.py, on oracle/mediapipe_shim and real cv2) and
pose_util.project_points / project_points_with_trans / smooth_pose_seq (src/utils/pose_util.py, numpy + scipy) on seeded
meshes and poses.

    ANIPORTRAIT_REFERENCE=<checkout> python oracle/make_golden_landmarks.py

Stored: both connection specs (forehead_edge False / True) in draw order, the reference's head-pose template
configs/inference/head_pose_temp/pose_temp.npy, the seeded meshes, offsets, poses and matrices with the reference's
projections of them, smoothed pose sequences, and drawn frames for a list of cases (normed reference pose, projected
frames, landmarks exactly at 0 and 1, just outside [0, 1] and NaN, coincident endpoints, overlapping edges of different
colours, a mesh partly off the canvas, the [478, 3] landmarks of the face landmarker as the scripts pass them), with the
cv2 version used. Compressed, under 1 MB.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "landmark_frames_reference.npz")
N = 468


def main():
    ref = os.environ.get("ANIPORTRAIT_REFERENCE", "")
    if not os.path.isdir(os.path.join(ref, "src", "utils")):
        raise SystemExit("set ANIPORTRAIT_REFERENCE to an AniPortrait checkout")
    sys.path.insert(0, os.path.join(ROOT, "oracle", "mediapipe_shim"))
    sys.path.insert(0, ref)
    import cv2
    from src.utils.draw_util import FaceMeshVisualizer
    from src.utils import pose_util

    vis = [FaceMeshVisualizer(forehead_edge=False), FaceMeshVisualizer(forehead_edge=True)]
    g = {"cv2_version": np.array(cv2.__version__)}
    for s, v in enumerate(vis):
        g[f"spec{s}_edges"] = np.array(list(v.face_connection_spec.keys()), dtype=np.int32)
        g[f"spec{s}_colors"] = np.array([d.color for d in v.face_connection_spec.values()], dtype=np.uint8)
        g[f"spec{s}_thickness"] = np.array([d.thickness for d in v.face_connection_spec.values()], dtype=np.int32)
    pose_temp = np.load(os.path.join(ref, "configs", "inference", "head_pose_temp", "pose_temp.npy"))
    g["pose_temp"] = pose_temp

    rng = np.random.default_rng(20261017)
    # a face-sized cloud in the reference's canonical-mesh units, 40 units in front of the camera
    base = rng.uniform([-7.0, -9.0, -3.0], [7.0, 9.0, 3.0], size=(N, 3))
    trans = np.eye(4)
    trans[:3, 3] = [0.3, -0.5, -40.0]
    L = 8
    offsets = (rng.standard_normal((L, N, 3)) * 0.2).astype(np.float32)
    mirrored = np.concatenate((pose_temp, pose_temp[-2:0:-1]), axis=0)      # audio2vid.py:167-169
    pose_seq = np.tile(mirrored, (L // len(mirrored) + 1, 1))[:L]
    g.update(mesh_base=base, trans_mat=trans, offsets=offsets, pose_seq=pose_seq)
    g["proj_a"] = pose_util.project_points(offsets + base, trans, pose_seq, [512, 512])
    g["smooth_7"] = pose_util.smooth_pose_seq(pose_temp, 7)
    g["smooth_3"] = pose_util.smooth_pose_seq(pose_temp[:40], 3)
    euler = rng.uniform(-40, 40, size=(16, 3))
    g["euler"] = euler
    g["euler_mats"] = np.stack([pose_util.euler_and_translation_to_matrix(e, [1.0, 2.0, 3.0]) for e in euler])
    # vid2vid path: per-frame meshes and smoothed matrices
    L2 = 4
    verts = base[None] + rng.standard_normal((L2, N, 3)) * 0.3
    parr = np.concatenate([rng.uniform(-15, 15, (L2, 3)), rng.uniform(-1, 1, (L2, 3)) + trans[:3, 3]], 1)
    parr = pose_util.smooth_pose_seq(parr, window_size=3)
    mats = np.stack([pose_util.euler_and_translation_to_matrix(p[:3], p[3:6]) for p in parr])
    g.update(vid_verts=verts, vid_mats=mats)
    g["proj_b"] = pose_util.project_points_with_trans(verts, mats, [512, 512])

    cases = []   # (name, spec, normed, keypoints [N, 2] float64)
    cases.append(("normed_ref_pose_s0", 0, True, (g["proj_a"][0] / 512).astype(np.float32).astype(np.float64)))
    cases.append(("normed_ref_pose_s1", 1, True, (g["proj_a"][1] / 512).astype(np.float32).astype(np.float64)))
    for i in range(0, L, 2):
        cases.append((f"projected_a{i}_s{i // 2 % 2}", i // 2 % 2, False, g["proj_a"][i]))
    cases.append(("projected_b0_s0", 0, False, g["proj_b"][0]))
    kp = rng.uniform(0, 1, (N, 2))
    edges0 = g["spec0_edges"]
    ends = np.unique(edges0.reshape(-1))
    kp[ends[0::4]] = rng.choice([0.0, 1.0], size=(len(ends[0::4]), 2))
    kp[ends[1::4], 0] = 1.0
    kp[ends[2::4], 1] = 0.0
    cases.append(("exact_0_and_1", 0, True, kp))
    kp = g["proj_a"][2].copy()
    sel = ends[0::3]
    kp[sel[0::4], 0] = -1e-7
    kp[sel[1::4], 1] = 512 * (1 + 1e-7)
    kp[sel[2::4], 0] = 512 * (1 + 1e-10)      # rounds to 1.0f: kept, pixel 511
    kp[sel[3::4], 1] = np.nan
    cases.append(("just_outside_and_nan", 0, False, kp))
    kp = g["proj_a"][3].copy()
    for a, b in edges0[::3]:
        kp[b] = kp[a]
    cases.append(("coincident_endpoints", 0, False, kp))
    kp = g["proj_a"][4].copy()
    centre = kp[ends].mean(0)
    kp[ends] = centre + (kp[ends] - centre) * 0.25     # crowd every edge into the middle: colours overlap
    cases.append(("overlapping_colours", 1, False, kp))
    cases.append(("partly_off_canvas", 0, False, g["proj_a"][5] + [190.0, -150.0]))
    frames = []
    for name, s, normed, kp in cases:
        frames.append(vis[s].draw_landmarks((512, 512), kp, normed=normed))
    g.update(case_names=np.array([c[0] for c in cases]), case_spec=np.array([c[1] for c in cases], dtype=np.int32),
             case_normed=np.array([c[2] for c in cases]), case_keypoints=np.stack([c[3] for c in cases]),
             case_frames=np.stack(frames))
    # the reference pose as audio2vid.py:153-155 / vid2vid.py:139-140 draw it: LMKExtractor's float32 [478, 3] (x, y, z)
    # landmarks (468 mesh points + 10 iris points), normed; draw_util.py reads columns 0 and 1 only
    rng = np.random.default_rng(478)
    xy = np.concatenate([g["proj_a"][6] / 512, rng.uniform(0.35, 0.65, (10, 2))])
    g["lmks478"] = np.concatenate([xy, rng.normal(0.0, 0.05, (478, 1))], 1).astype(np.float32)
    g["lmks478_frames"] = np.stack([v.draw_landmarks((512, 512), g["lmks478"], normed=True) for v in vis])
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1e6:.2f} MB, {len(cases)} frames, cv2 {cv2.__version__}")
    for (name, *_), f in zip(cases, frames):
        print(f"  {name}: {int((f.any(axis=2)).sum())} drawn pixels")


if __name__ == "__main__":
    main()
