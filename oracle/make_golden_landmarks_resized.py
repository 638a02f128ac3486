"""TEST INFRASTRUCTURE — generates tests/golden/landmark_frames_resized_reference.npz by running the UNMODIFIED reference
FaceMeshVisualizer.draw_landmarks (src/utils/draw_util.py, on oracle/mediapipe_shim and real cv2) at image sizes other
than 512 x 512, where it ends in cv2.resize, and the vid2vid chain (scripts/vid2vid.py:197-200: draw at the source
video's size, then cv2.resize to 512 x 512), on the seeded meshes and cases of tests/golden/landmark_frames_reference.npz.

    ANIPORTRAIT_REFERENCE=<checkout> python oracle/make_golden_landmarks_resized.py

Stored, with the cv2 version used and the forehead_edge=False connection spec both scripts draw with:
  one_*   audio2vid at -W/-H other than 512 (audio2vid.py:199-205): pose_util.project_points at [H, W], drawn at (W, H).
          Frames up to 768 x 768 as arrays, larger ones as SHA-256 digests of their bytes.
  chain_* vid2vid: keypoints at the source size (projected frames, the normed reference pose, a mesh partly off the
          canvas), drawn at the source size and resized to 512 x 512. The 512 x 512 frames as arrays, the frames at the
          source size as SHA-256 digests.
Compressed, under 1 MB.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "golden", "landmark_frames_reference.npz")
OUT = os.path.join(ROOT, "tests", "golden", "landmark_frames_resized_reference.npz")
ONE_SIZES = [(768, 768), (512, 768), (768, 512), (1080, 1920), (1920, 1080), (720, 1280), (1024, 1024)]   # (W, H)
CHAIN_SOURCES = [(1080, 1920), (1920, 1080), (720, 1280), (1024, 1024)]                                  # (W, H)
ARRAY_MAX = 768


def digest(frame):
    return hashlib.sha256(np.ascontiguousarray(frame).tobytes()).hexdigest()


def main():
    ref = os.environ.get("ANIPORTRAIT_REFERENCE", "")
    if not os.path.isdir(os.path.join(ref, "src", "utils")):
        raise SystemExit("set ANIPORTRAIT_REFERENCE to an AniPortrait checkout")
    sys.path.insert(0, os.path.join(ROOT, "oracle", "mediapipe_shim"))
    sys.path.insert(0, ref)
    import cv2
    from src.utils.draw_util import FaceMeshVisualizer
    from src.utils import pose_util

    src = dict(np.load(SRC))
    vis = FaceMeshVisualizer(forehead_edge=False)
    g = {"cv2_version": np.array(cv2.__version__),
         "edges": np.array(list(vis.face_connection_spec.keys()), dtype=np.int32),
         "colors": np.array([d.color for d in vis.face_connection_spec.values()], dtype=np.uint8)}
    assert np.array_equal(g["edges"], src["spec0_edges"]) and np.array_equal(g["colors"], src["spec0_colors"])
    pts = src["offsets"] + src["mesh_base"]           # audio2vid.py:183: pred + face_result['lmks3d']
    names = {"one": [], "chain": []}

    def add(kind, name, size, normed, kp, frame, extra=None):
        names[kind].append(name)
        g[f"{kind}_{name}_size"] = np.array(size, dtype=np.int32)
        g[f"{kind}_{name}_normed"] = np.array(normed)
        g[f"{kind}_{name}_keypoints"] = kp
        if kind == "chain" or max(frame.shape[:2]) <= ARRAY_MAX:
            g[f"{kind}_{name}_frame"] = frame
        else:
            g[f"{kind}_{name}_sha256"] = np.array(digest(frame))
        for k, v in (extra or {}).items():
            g[f"{kind}_{name}_{k}"] = v

    # audio2vid at another size: one resize of the canvas
    for W, H in ONE_SIZES:
        proj = pose_util.project_points(pts[:4], src["trans_mat"], src["pose_seq"][:4], [H, W])
        for i in (0, 3):
            add("one", f"{W}x{H}_a{i}", (W, H), False, proj[i], vis.draw_landmarks((W, H), proj[i], normed=False))
    # the reference pose, normed, drawn at a non-square -W/-H (audio2vid.py:155)
    kp = src["case_keypoints"][list(src["case_names"]).index("normed_ref_pose_s0")]
    add("one", "512x768_ref_pose", (512, 768), True, kp, vis.draw_landmarks((512, 768), kp, normed=True))

    # vid2vid: draw at the source video's size, then cv2.resize(lmk_img, (512, 512))
    for W, H in CHAIN_SOURCES:
        proj = pose_util.project_points_with_trans(src["vid_verts"][:2], src["vid_mats"][:2], [H, W])
        cases = [(f"{W}x{H}_b0", False, proj[0]), (f"{W}x{H}_ref_pose", True, kp),
                 (f"{W}x{H}_off_canvas", False, proj[1] + [0.4 * W, -0.3 * H])]
        for name, normed, k in cases:
            lmk = vis.draw_landmarks((W, H), k, normed=normed)
            assert lmk.shape == (H, W, 3)
            add("chain", name, (W, H), normed, k, cv2.resize(lmk, (512, 512)), {"source_sha256": np.array(digest(lmk))})
    g["one_names"] = np.array(names["one"])
    g["chain_names"] = np.array(names["chain"])
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1e6:.2f} MB, {len(names['one'])} one-resize and "
          f"{len(names['chain'])} vid2vid frames, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
