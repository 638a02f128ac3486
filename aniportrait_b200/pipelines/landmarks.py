"""Face-mesh projection and landmark pose frames on the device — the stage of the reference's scripts that turns the
predicted mesh into the pose images the pipeline is conditioned on (scripts/audio2vid.py:199-222, scripts/vid2vid.py:194-203):
pose_util.project_points / project_points_with_trans (src/utils/pose_util.py:30-59) and FaceMeshVisualizer.draw_landmarks
(src/utils/draw_util.py:124-148, mediapipe drawing_utils.draw_landmarks on cv2.line).

    from aniportrait_b200.pipelines import landmarks
    vis = landmarks.enable_kernels(FaceMeshVisualizer(forehead_edge=False))
    kp = landmarks.project_points(pred, face_result["trans_mat"], pose_seq, [height, width], base=face_result["lmks3d"])
    pose_frames = vis.draw_pose_frames((width, height), kp)           # CUDA uint8 [L, height, width, 3]
    video = pipe(ref_image_pil, pose_frames, ref_pose, width, height, len(pose_frames), steps, cfg).videos

vid2vid draws at the source video's size and resizes once more (scripts/vid2vid.py:197-200):
    pose_frames = vis.draw_pose_frames((frame_width, frame_height), kp, out_size=(width, height))

The drawn bytes equal the reference's frame for frame, cv2.resize included. The host only builds the per-frame 4x4
matrices (the Euler angles to rotation restated in numpy, no scipy) and reads the edge table and colours from the
caller's own visualizer; there is no CPU fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops

CANVAS = ops.LMK_CANVAS   # draw_util.py:125 ini_size


def _device(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("aniportrait_b200.pipelines.landmarks runs on CUDA (sm_90a) only: no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _to_device(x, dtype, device):
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))
    return t.to(device=device, dtype=dtype).contiguous()


# ------------------------------------------------------------------------------------------------------ projection
def perspective_matrix(aspect_ratio) -> np.ndarray:
    """P of pose_util.py:7-27 and :31 (create_perspective_matrix(...).reshape(4, 4).T): built in float32 as the reference
    builds it, returned promoted to float64 (as numpy promotes it in the float64 matmul)."""
    pm = np.zeros(16, dtype=np.float32)
    f = 1.0 / np.tan(np.pi / 180. * 63 / 2.)
    near, far = 1, 10000
    denom = 1.0 / (near - far)
    pm[0] = f / aspect_ratio
    pm[5] = f
    pm[10] = (near + far) * denom
    pm[11] = -1.
    pm[14] = 1. * far * near * denom
    pm[5] *= -1.
    return pm.reshape(4, 4).T.astype(np.float64)


def euler_and_translation_to_matrix(euler_angles, translation_vector) -> np.ndarray:
    """pose_util.py:62-70: 4x4 of the extrinsic x-y-z rotation by `euler_angles` degrees (Rz @ Ry @ Rx, as
    scipy's Rotation.from_euler('xyz', ..., degrees=True)) and the translation."""
    a, b, c = np.deg2rad(np.asarray(euler_angles, dtype=np.float64))
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    m = np.eye(4)
    m[:3, :3] = [[cb * cc, sa * sb * cc - ca * sc, ca * sb * cc + sa * sc],
                 [cb * sc, sa * sb * sc + ca * cc, ca * sb * sc - sa * cc],
                 [-sb, sa * cb, ca * cb]]
    m[:3, 3] = translation_vector
    return m


def smooth_pose_seq(pose_seq, window_size=5):
    """pose_util.py:81-89: centred moving mean, the window clipped at both ends."""
    smoothed_pose_seq = np.zeros_like(pose_seq)
    for i in range(len(pose_seq)):
        start = max(0, i - window_size // 2)
        end = min(len(pose_seq), i + window_size // 2 + 1)
        smoothed_pose_seq[i] = np.mean(pose_seq[start:end], axis=0)
    return smoothed_pose_seq


def _project(points_3d, matrices, image_shape, base):
    mats = np.ascontiguousarray(matrices, dtype=np.float64)
    L = mats.shape[0]
    if base is not None and getattr(points_3d, "dtype", None) not in (np.float32, torch.float32):
        raise TypeError(f"with `base`, points_3d is the fp32 per-frame offset (got "
                        f"{getattr(points_3d, 'dtype', type(points_3d))}); pass an fp64 mesh without `base` instead")
    device = _device(points_3d, base)
    if base is None:
        pts, offs = _to_device(points_3d, torch.float64, device), None
    else:
        pts = _to_device(base, torch.float64, device)
        offs = _to_device(points_3d, torch.float32, device).reshape(L, pts.shape[-2], 3)
    if pts.dim() != 2 and pts.shape[0] != L:
        raise ValueError(f"{pts.shape[0]} frames of points for {L} matrices")
    proj = perspective_matrix(image_shape[1] / image_shape[0])
    return ops.project_points(pts, _to_device(mats, torch.float64, device), proj.reshape(-1),
                              float(image_shape[1]), float(image_shape[0]), offsets=offs)


def project_points(points_3d, transformation_matrix, pose_vectors, image_shape, base=None) -> torch.Tensor:
    """pose_util.project_points on the device -> CUDA fp64 [L, N, 2]. points_3d [L, N, 3] (numpy or tensor) is the mesh
    per frame; with `base` ([N, 3] fp64, face_result['lmks3d']) it is instead the fp32 per-frame offset (the Audio2Mesh
    output [L, N * 3] straight from the device), added to `base` in fp64 as numpy's `pred + lmks3d` does; any other dtype
    raises TypeError rather than being rounded to fp32."""
    pose_vectors = np.asarray(pose_vectors, dtype=np.float64)
    trans = np.asarray(transformation_matrix, dtype=np.float64)
    mats = np.stack([trans @ euler_and_translation_to_matrix(p[:3], p[3:]) for p in pose_vectors])
    return _project(points_3d, mats, image_shape, base)


def project_points_with_trans(points_3d, transformation_matrices, image_shape, base=None) -> torch.Tensor:
    """pose_util.project_points_with_trans on the device -> CUDA fp64 [L, N, 2] (`base` as for project_points)."""
    return _project(points_3d, np.asarray(transformation_matrices, dtype=np.float64), image_shape, base)


# ------------------------------------------------------------------------------------------------------ drawing
def edge_table(face_connection_spec):
    """(edges int32 [E, 2], colours uint8 [E, 3]) in draw order from a {(start, end): DrawingSpec} mapping: its iteration
    order (a key inserted twice keeps its first position and its last spec)."""
    edges, colors = [], []
    for (a, b), spec in face_connection_spec.items():
        if spec.thickness != 2:
            raise NotImplementedError(f"landmark edges of thickness {spec.thickness}: only thickness 2 is implemented")
        edges.append((int(a), int(b)))
        colors.append(tuple(int(c) for c in spec.color))
    if len(edges) > ops.LMK_MAX_EDGES:
        raise NotImplementedError(f"{len(edges)} landmark edges: at most {ops.LMK_MAX_EDGES} are implemented")
    return np.array(edges, dtype=np.int32).reshape(-1, 2), np.array(colors, dtype=np.uint8).reshape(-1, 3)


def _check_size(image_size):
    if tuple(int(v) for v in image_size) != (CANVAS, CANVAS):
        raise NotImplementedError(f"draw_landmarks to image_size {tuple(image_size)}: draw_landmarks and "
                                  f"draw_landmarks_batch draw the {CANVAS}x{CANVAS} canvas only; draw_pose_frames "
                                  "draws at any size")


def _frame_size(size, what):
    """(W, H) as ints, each side in [1, ops.RESIZE_MAX_SIDE] (ValueError otherwise)."""
    wh = tuple(int(v) for v in size)
    if len(wh) != 2 or not all(1 <= v <= ops.RESIZE_MAX_SIDE for v in wh):
        raise ValueError(f"{what} {tuple(size)}: expected (width, height), each in [1, {ops.RESIZE_MAX_SIDE}]")
    return wh


def resize_frames(frames, size) -> torch.Tensor:
    """cv2.resize(frame, size) with the default INTER_LINEAR for every frame of CUDA uint8 frames [L, h, w, 3] ->
    CUDA uint8 [L, H, W, 3] for size = (W, H), byte for byte, in one launch. Every side lies in [1, 8192]."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dtype == torch.uint8):
        raise TypeError("resize_frames takes a CUDA uint8 tensor [L, h, w, 3]")
    if frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError(f"frames must be [L, h, w, 3], got {tuple(frames.shape)}")
    return ops.resize_linear_u8(frames.contiguous(), _frame_size(size, "size"))


# frames drawn per launch by draw_pose_frames when it resizes: the 512 x 512 canvas scratch stays under 101 MB
POSE_CHUNK = 128


def _pose_stages(image_size, out_size):
    """The sizes the canvas is resized to, in order: image_size (draw_landmarks' own cv2.resize), then out_size. A size
    equal to the one before it is dropped: cv2.resize to the same size is a copy."""
    sizes = [_frame_size(image_size, "image_size")]
    if out_size is not None:
        sizes.append(_frame_size(out_size, "out_size"))
    stages, prev = [], (CANVAS, CANVAS)
    for size in sizes:
        if size != prev:
            stages.append(size)
        prev = size
    return stages


def enable_kernels(vis):
    """Bind a FaceMeshVisualizer (reference src/utils/draw_util.py) to the device kernels. Its face_connection_spec is read
    once; afterwards
      vis.draw_landmarks(image_size, keypoints, normed=False)        -> numpy uint8 [H, W, 3], the reference's bytes
      vis.draw_landmarks_batch(image_size, keypoints, normed=False) -> CUDA uint8 [L, H, W, 3] for keypoints [L, N, C],
                                                                       one kernel launch, 1 <= L <= 67108863
      vis.draw_pose_frames(image_size, keypoints, normed=False, out_size=None)
          -> CUDA uint8 [L, H', W', 3]: per frame, cv2.resize(reference draw_landmarks(image_size, kp), out_size), or the
             reference's draw_landmarks frame alone when out_size is None, at any sizes in [1, 8192]. Frames are drawn
             in chunks of POSE_CHUNK, each one draw launch plus at most one resize launch (none when every resize is to
             the size before it); no frame at image_size is stored when out_size differs from it.
    As in the reference, keypoints may carry more than two columns (LMKExtractor's [478, 3] x, y, z landmarks); only
    columns 0 and 1 are read. draw_landmarks and draw_landmarks_batch implement image_size (512, 512) only
    (NotImplementedError otherwise). Returns vis."""
    edges, colors = edge_table(vis.face_connection_spec)

    def device_keypoints(keypoints):
        if keypoints.ndim != 3 or keypoints.shape[2] < 2:
            raise ValueError(f"keypoints must be [L, N, C >= 2], got {tuple(keypoints.shape)}")
        n = keypoints.shape[1]
        bad = (edges < 0) | (edges >= n)
        if bad.any():
            a, b = edges[np.nonzero(bad.any(axis=1))[0][0]]
            raise ValueError(f"Landmark index is out of range. Invalid connection from landmark #{a} to landmark #{b}.")
        return _to_device(keypoints[:, :, :2], torch.float64, _device(keypoints))

    def draw_landmarks_batch(image_size, keypoints, normed=False):
        _check_size(image_size)
        kp = device_keypoints(keypoints)
        return ops.draw_landmarks(kp, float(image_size[0]), float(image_size[1]), bool(normed), edges, colors)

    def draw_pose_frames(image_size, keypoints, normed=False, out_size=None):
        stages = _pose_stages(image_size, out_size)
        kp = device_keypoints(keypoints)
        size_x, size_y = float(image_size[0]), float(image_size[1])
        if not stages:
            return ops.draw_landmarks(kp, size_x, size_y, bool(normed), edges, colors)
        W, H = stages[-1]
        mid = stages[0] if len(stages) == 2 else None
        out = torch.empty(kp.shape[0], H, W, 3, dtype=torch.uint8, device=kp.device)
        for i in range(0, kp.shape[0], POSE_CHUNK):
            canvas = ops.draw_landmarks(kp[i:i + POSE_CHUNK], size_x, size_y, bool(normed), edges, colors)
            ops.resize_linear_u8(canvas, (W, H), mid=mid, out=out[i:i + POSE_CHUNK])
        return out

    def draw_landmarks(image_size, keypoints, normed=False):
        if keypoints.ndim != 2:
            raise ValueError(f"keypoints must be [N, C >= 2], got {tuple(keypoints.shape)}")
        return draw_landmarks_batch(image_size, keypoints[None], normed)[0].cpu().numpy()

    vis.draw_landmarks = draw_landmarks
    vis.draw_landmarks_batch = draw_landmarks_batch
    vis.draw_pose_frames = draw_pose_frames
    return vis
