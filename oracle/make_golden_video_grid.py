"""TEST INFRASTRUCTURE — generates tests/golden/video_grid_reference.npz by running the UNMODIFIED reference
src/utils/util.py:save_videos_grid on the seeded cases of tests/video_grid_cases.py, each built into the tensor the
scripts build: every frame beside the result through transforms.Compose([Resize((height, width)), ToTensor()]) (BGR pose
frames through cv2.cvtColor(BGR2RGB) and Image.fromarray first), the reference image repeated over T, torch.cat along the
batch dim with the pose tensor cut to the video's length.

    ANIPORTRAIT_REFERENCE=<checkout> python oracle/make_golden_video_grid.py

util imports `av` at module scope; a stub module stands in for it, and util.save_videos_from_pil is replaced by a
function that keeps the PIL frames, so the stub is never called. Stored per case: n_rows, the frames as uint8 arrays when
the grid is at most 200 pixels wide, else as one SHA-256 digest of all frames, and the digest of the inputs. The Pillow,
torchvision and torch versions are recorded. Compressed, under 1 MB.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "video_grid_reference.npz")
ARRAY_MAX_WIDTH = 200


def script_tail(case, transforms, Image, cv2, torch):
    """The tensor the scripts hand to save_videos_grid, and n_rows."""
    n_rows, (height, width), tiles = case
    pose_transform = transforms.Compose([transforms.Resize((height, width)), transforms.ToTensor()])
    T = next(t[1].shape[2] for t in tiles if t[0] == "video")
    parts = []
    for kind, data, bgr in tiles:
        if kind == "video":
            parts.append(torch.from_numpy(data))
            continue
        frames = [Image.fromarray(cv2.cvtColor(f, cv2.COLOR_BGR2RGB) if bgr else f) for f in data]
        if len(frames) == 1:                                          # the reference image, repeated over the video
            t = pose_transform(frames[0]).unsqueeze(1).unsqueeze(0)
            parts.append(t.repeat(1, 1, T, 1, 1))
        else:
            t = torch.stack([pose_transform(f) for f in frames], dim=0).transpose(0, 1).unsqueeze(0)
            parts.append(t[:, :, :T])
    return torch.cat(parts, dim=0), n_rows


def main():
    ref = os.environ.get("ANIPORTRAIT_REFERENCE", "")
    if not os.path.isdir(os.path.join(ref, "src", "utils")):
        raise SystemExit("set ANIPORTRAIT_REFERENCE to an AniPortrait checkout")
    sys.modules.setdefault("av", types.ModuleType("av"))
    sys.path.insert(0, ref)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import cv2
    import PIL
    import torch
    import torchvision
    from PIL import Image
    from torchvision import transforms
    from src.utils import util
    import video_grid_cases as VC

    captured = []
    util.save_videos_from_pil = lambda pil_images, path, fps=8: captured.append(pil_images)
    g = {"pillow_version": np.array(PIL.__version__), "torchvision_version": np.array(torchvision.__version__),
         "torch_version": np.array(torch.__version__)}
    names = []
    scratch = tempfile.mkdtemp()           # save_videos_grid makes the directory of its path; nothing is written there
    for name, case in VC.cases().items():
        video, n_rows = script_tail(case, transforms, Image, cv2, torch)
        captured.clear()
        util.save_videos_grid(video, os.path.join(scratch, f"{name}.mp4"), n_rows=n_rows)
        frames = np.stack([np.asarray(im) for im in captured[0]], 0)
        assert frames.dtype == np.uint8 and frames.ndim == 4 and frames.shape[3] == 3, frames.shape
        names.append(name)
        g[f"{name}_n_rows"] = np.array(n_rows)
        g[f"{name}_shape"] = np.array(frames.shape, dtype=np.int64)
        g[f"{name}_input_sha256"] = np.array(VC.input_digest(case[2]))
        if frames.shape[2] <= ARRAY_MAX_WIDTH:
            g[f"{name}_frames"] = frames
        else:
            g[f"{name}_sha256"] = np.array(VC.frames_digest(frames))
    os.rmdir(scratch)
    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1e6:.3f} MB, {len(names)} cases, Pillow {PIL.__version__}, "
          f"torchvision {torchvision.__version__}")


if __name__ == "__main__":
    main()
