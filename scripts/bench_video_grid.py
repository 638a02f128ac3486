"""The scripts' comparison-video tail: the reference's host path against the device path, at L = 150 and 300 frames (5 and
10 s at 30 fps).

  vid2vid          1080 x 1920 (W x H) source frames beside a 512 x 512 result; tiles [reference, video, source]
                   (scripts/vid2vid.py:147-162, 228-243)
  audio2vid 512    BGR pose frames at 512 x 512; tiles [reference, pose, video] (scripts/audio2vid.py:207-260)
  audio2vid 768    the same at -W 768 -H 768

  host    the scripts' tail from the PIL / numpy frames and the pipeline's fp32 host video: pose_transform (Resize +
          ToTensor) per frame, cv2.cvtColor(BGR2RGB) first for the pose frames, the reference image repeated, torch.cat,
          then save_videos_grid's per-frame loop up to the PIL images (make_grid, * 255, astype(uint8), Image.fromarray);
          the encoder is not run. Timed once (it takes seconds).
  device  pose_transform_frames of the host frames (audio2vid: the CUDA pose frames of draw_pose_frames, already at the
          size), then grid_frames on the pipeline's fp16 video (output_type="cuda"): CUDA uint8 grid frames. device_ms
          ends there; device_d2h_ms also copies the frames to host memory, where an encoder would read them. Median of
          --calls calls after one warm-up.

`identical` compares the device frames with the host arm's PIL frames byte for byte; `peak_device_mb` is the device
memory the device arm allocated at its peak, its output included. The source frames cycle through 8 seeded images.

    python scripts/bench_video_grid.py [--calls 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aniportrait_b200.pipelines import video_grid as VG  # noqa: E402


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
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    import torchvision
    from einops import rearrange
    from PIL import Image
    dev = torch.device("cuda:0")
    gpu = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    import cv2
    from torchvision import transforms
    rng = np.random.default_rng(0)

    def save_videos_grid_frames(videos, n_rows):
        """src/utils/util.py:87-100, the loop of save_videos_grid up to its PIL frames."""
        videos = rearrange(videos, "b c t h w -> t b c h w")
        outputs = []
        for x in videos:
            x = torchvision.utils.make_grid(x, nrow=n_rows)
            x = x.transpose(0, 1).transpose(1, 2).squeeze(-1)
            x = (x * 255).numpy().astype(np.uint8)
            outputs.append(Image.fromarray(x))
        return outputs

    for L in (150, 300):
        for arm, side, src_wh in (("vid2vid", 512, (1080, 1920)), ("audio2vid", 512, None), ("audio2vid", 768, None)):
            size = (side, side)
            ref_pil = Image.fromarray(rng.integers(0, 256, (700, 500, 3), dtype=np.uint8))
            video16 = torch.from_numpy(rng.random((1, 3, L, side, side), dtype=np.float32)).half().to(dev)
            if arm == "vid2vid":
                distinct = [Image.fromarray(rng.integers(0, 256, (src_wh[1], src_wh[0], 3), dtype=np.uint8))
                            for _ in range(8)]
                frames = [distinct[i % 8] for i in range(L)]
                bgr = False
            else:
                distinct = [rng.integers(0, 256, (side, side, 3), dtype=np.uint8) for _ in range(8)]
                frames = [distinct[i % 8] for i in range(L)]
                pose_dev = torch.from_numpy(np.stack(frames)).to(dev)       # draw_pose_frames' CUDA output
                bgr = True

            def device_arm(copy=False):
                ref = VG.pose_transform_frames([ref_pil], size)
                if arm == "vid2vid":
                    out = VG.grid_frames([ref, video16, VG.pose_transform_frames(frames, size)], n_rows=3)
                else:
                    out = VG.grid_frames([ref, VG.pose_transform_frames(pose_dev, size), video16], n_rows=3,
                                         bgr=[False, True, False])
                return out.cpu() if copy else out

            def host_arm():
                pose_transform = transforms.Compose([transforms.Resize(size), transforms.ToTensor()])
                video = video16.float().cpu()                              # output_type="tensor"
                ref = pose_transform(ref_pil).unsqueeze(1).unsqueeze(0).repeat(1, 1, L, 1, 1)
                pil = [Image.fromarray(cv2.cvtColor(f, cv2.COLOR_BGR2RGB)) if bgr else f for f in frames]
                other = torch.stack([pose_transform(p) for p in pil], dim=0).transpose(0, 1).unsqueeze(0)
                tiles = [ref, video, other[:, :, :L]] if arm == "vid2vid" else [ref, other[:, :, :L], video]
                return save_videos_grid_frames(torch.cat(tiles, dim=0), 3)

            res = {"arm": arm, "sizes": (f"{src_wh[0]}x{src_wh[1]}->" if src_wh else "") + f"{side}x{side}", "L": L,
                   "gpu": gpu, "power_limit": power}
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            res["device_ms"] = median_ms(device_arm, args.calls)
            res["peak_device_mb"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
            res["device_d2h_ms"] = median_ms(lambda: device_arm(copy=True), args.calls)
            t0 = time.perf_counter()
            host = host_arm()
            res["host_ms"] = (time.perf_counter() - t0) * 1e3
            got = device_arm(copy=True).numpy()
            res["identical"] = bool(len(host) == len(got) and all(np.array_equal(np.asarray(h), g)
                                                                  for h, g in zip(host, got)))
            del host, got
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
