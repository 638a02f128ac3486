"""The side-by-side comparison video of the reference's scripts, on the device: every frame shown beside the result goes
through `transforms.Compose([transforms.Resize((height, width)), transforms.ToTensor()])` (Pillow's bilinear resize),
the tiles are concatenated with torch.cat, and save_videos_grid (src/utils/util.py:87-104) lays each frame out with
torchvision.utils.make_grid and writes `(x * 255).numpy().astype(np.uint8)`. Here the frames stay uint8 (ToTensor
followed by `* 255` and the uint8 cast gives every byte back), the resize is ap_resize_pil_bilinear_u8 and the grid is
one ap_video_grid_u8 launch, byte for byte the frames save_videos_grid hands to its encoder.

audio2vid (scripts/audio2vid.py:207-260), with the pose frames of landmarks.enable_kernels(vis).draw_pose_frames, which
are BGR like the reference's:
    video = pipe(ref_image_pil, pose_frames, ref_pose, width, height, L, steps, cfg, output_type="cuda").videos
    ref = video_grid.pose_transform_frames([ref_image_pil], (height, width))
    pose = video_grid.pose_transform_frames(pose_frames, (height, width))          # same size: no launch
    frames = video_grid.grid_frames([ref, pose, video], n_rows=3, bgr=[False, True, False])
    save_videos_from_pil([Image.fromarray(f) for f in frames.cpu().numpy()], save_path, fps)

vid2vid (scripts/vid2vid.py:147-162, 228-243): the source frames, sliced with the script's step, resized on upload:
    src = video_grid.pose_transform_frames(source_images[:args_L:step], (height, width))
    frames = video_grid.grid_frames([ref, video, src], n_rows=3)

pose2vid (scripts/pose2vid.py:146-151, 181-196):
    pose = video_grid.pose_transform_frames(pose_images[:args_L], (height, width))
    frames = video_grid.grid_frames([ref, pose, video], n_rows=3)

app.py (scripts/app.py:258-262): video_grid.grid_frames([video], n_rows=1) is the video's own frames.

With -acc, the frame interpolator's fp32 host output can be passed after `.to("cuda")`; a pose tile longer than the video
contributes its first T frames, as the scripts' `[:, :, :video.shape[2]]` does. There is no CPU fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops

# host frames are uploaded through a pinned buffer of at most this many bytes, one resize launch per chunk: the device
# scratch does not grow with the number of frames
UPLOAD_CHUNK_BYTES = 64 << 20


def _size(size):
    hw = tuple(int(v) for v in size)
    if len(hw) != 2 or not all(1 <= v <= ops.RESIZE_MAX_SIDE for v in hw):
        raise ValueError(f"size {tuple(size)}: expected (height, width), each in [1, {ops.RESIZE_MAX_SIDE}]")
    return hw


def _host_shape(f):
    """(h, w) of an RGB PIL image or an HxWx3 uint8 array, without reading its pixels."""
    if hasattr(f, "mode") and hasattr(f, "size"):
        if f.mode != "RGB":
            raise ValueError(f"PIL image of mode {f.mode}: only RGB frames are implemented")
        return f.size[1], f.size[0]
    if not (isinstance(f, np.ndarray) and f.dtype == np.uint8 and f.ndim == 3 and f.shape[2] == 3):
        raise TypeError(f"frames must be RGB PIL images or HxWx3 uint8 arrays, got "
                        f"{getattr(f, 'dtype', type(f))} {getattr(f, 'shape', '')}")
    return f.shape[:2]


def pose_transform_frames(frames, size) -> torch.Tensor:
    """The scripts' `pose_transform` (transforms.Resize(size) + ToTensor) read back as `* 255` bytes: CUDA uint8
    [L, height, width, 3] for size = (height, width), the order of transforms.Resize.
    frames: a list of same-size RGB PIL images or HxWx3 uint8 arrays, a uint8 array [L, h, w, 3], or a CUDA uint8 tensor
    [L, h, w, 3]. A CUDA tensor is resized in one launch, or returned as it is when its size already matches. Host frames
    are uploaded in chunks of at most UPLOAD_CHUNK_BYTES through a pinned buffer, one resize launch per chunk (none when
    the size matches)."""
    H, W = _size(size)
    if isinstance(frames, torch.Tensor):
        if not (frames.is_cuda and frames.dtype == torch.uint8):
            raise TypeError("pose_transform_frames takes a CUDA uint8 tensor, host frames or a uint8 array")
        if frames.dim() != 4 or frames.shape[3] != 3:
            raise ValueError(f"frames must be [L, h, w, 3], got {tuple(frames.shape)}")
        if tuple(frames.shape[1:3]) == (H, W):
            return frames
        return ops.resize_pil_bilinear_u8(frames.contiguous(), (W, H))
    host = list(frames)                                # pixels are read chunk by chunk, straight into the pinned buffer
    if not host:
        raise ValueError("pose_transform_frames: no frames")
    h, w = _host_shape(host[0])
    if any(_host_shape(f) != (h, w) for f in host):
        raise ValueError("pose_transform_frames: the frames differ in size")
    if not (1 <= h <= ops.RESIZE_MAX_SIDE and 1 <= w <= ops.RESIZE_MAX_SIDE):
        raise ValueError(f"frames of {w}x{h}: every side must lie in [1, {ops.RESIZE_MAX_SIDE}]")
    if w > ops.RESIZE_PIL_MAX_SCALE * W or h > ops.RESIZE_PIL_MAX_SCALE * H:
        raise ValueError(f"{(w, h)} -> {(W, H)} shrinks an axis by more than {ops.RESIZE_PIL_MAX_SCALE}x")
    if not torch.cuda.is_available():
        raise RuntimeError("aniportrait_b200.pipelines.video_grid runs on CUDA (sm_90a) only: no CPU fallback")
    device = torch.device("cuda", torch.cuda.current_device())
    L = len(host)
    same = (h, w) == (H, W)
    chunk = max(1, min(L, UPLOAD_CHUNK_BYTES // (h * w * 3)))
    out = torch.empty(L, H, W, 3, dtype=torch.uint8, device=device)
    stream = torch.cuda.current_stream(device)
    # two pinned buffers: the host fills one while the other's upload is in flight
    pins = [torch.empty(chunk, h, w, 3, dtype=torch.uint8, pin_memory=True) for _ in range(min(2, -(-L // chunk)))]
    done = [None] * len(pins)
    scratch = None if same else torch.empty(chunk, h, w, 3, dtype=torch.uint8, device=device)
    for j, i in enumerate(range(0, L, chunk)):
        n = min(chunk, L - i)
        b = j % len(pins)
        if done[b] is not None:
            done[b].synchronize()
        pin = pins[b].numpy()
        for k in range(n):
            pin[k] = np.asarray(host[i + k])
        dst = out[i:i + n] if same else scratch[:n]
        dst.copy_(pins[b][:n], non_blocking=True)
        done[b] = torch.cuda.Event()
        done[b].record(stream)
        if not same:
            ops.resize_pil_bilinear_u8(scratch[:n], (W, H), out=out[i:i + n])
    return out


def grid_frames(tiles, n_rows: int, bgr=None, frames=None, out=None) -> torch.Tensor:
    """save_videos_grid's frames of torch.cat(tiles, dim=0) with make_grid(nrow=n_rows), as CUDA uint8 [T, GH, GW, 3] in
    one launch: each equals `(make_grid(x, nrow=n_rows) * 255).numpy().astype(np.uint8)` transposed to HWC.
    tiles: CUDA uint8 frames [T' >= T or 1, H, W, 3] (pose_transform_frames' output; one frame is repeated over T, as the
    scripts repeat the reference image; bgr[i] swaps the channels of tile i, for BGR pose frames), or CUDA fp16 / fp32
    videos [1, 3, T' >= T, H, W] in [0, 1] of any strides (output_type="cuda" of the pipeline). T is the video tiles'
    frame count unless `frames` is given. out: a contiguous uint8 [T, GH, GW, 3] buffer to reuse.
    Mismatched tile sizes, a uint8 tile with 1 < T' < T, host tensors and other dtypes raise before any launch."""
    tiles = list(tiles)
    for i, t in enumerate(tiles):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise TypeError(f"grid_frames: tile {i} is not a CUDA tensor (no CPU fallback)")
    if frames is None:
        lengths = {int(t.shape[2]) for t in tiles if t.dtype != torch.uint8 and t.dim() == 5}
        if len(lengths) != 1:
            raise ValueError(f"grid_frames: the video tiles have frame counts {sorted(lengths)}; pass frames=T")
        frames = lengths.pop()
    return ops.video_grid_u8(tiles, int(n_rows), int(frames), bgr=bgr, out=out)
