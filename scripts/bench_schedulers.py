"""Times one video of the benchmarked geometry (512x512, L = 16, CFG 3.5; seeded full-size weights, bench.py's
build_product_pipeline) under each sampler the pipeline runs:

  ddim_25     DDIMScheduler, 25 steps (bench.py's workload)
  dpmpp_2m_N  DPMSolverMultistepScheduler.from_config(ddim.config), dpmsolver++ 2M midpoint, N = 10, 15, 20 steps
  euler_25    EulerDiscreteScheduler.from_config(ddim.config), 25 steps

Per arm: run_device with CUDA graphs after one warm-up video (capture), CUDA events around each of --reps videos (median,
min, max) -> device ms per video and per step; and the arm's update kernel alone (ap_cfg_ddim_step_f16 or
ap_cfg_multistep_step_f16 with second-order coefficients) timed with events over --launches launches on the loop's
tensors. The card's name and power limit are read in the same run. The trained weights are absent: nothing here says
anything about output quality at fewer steps.

    python scripts/bench_schedulers.py [--reps 5] [--launches 2000]

Prints JSON lines. Fails without a CUDA device (there is no CPU measurement).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_schedulers.py needs a CUDA device (no CPU measurement)")
    import bench
    from aniportrait_b200 import _lib, ops
    from aniportrait_b200.pipelines.scheduler import (DPMSolverMultistepScheduler, EulerDiscreteScheduler,
                                                      multistep_coefficients)
    from aniportrait_b200.pipelines.sharding import step_weights
    dev = torch.device("cuda", 0)
    _lib.init(0)
    name, power = card()
    print(json.dumps(dict(gpu=name, power_limit=power)), flush=True)
    pipe = bench.build_product_pipeline(dev)
    ddim = pipe.scheduler
    ref_image, poses, _ = bench.synthetic_inputs(1000, bench.L)
    H, W, L = bench.H, bench.W, bench.L
    clip_px = pipe.clip_image_processor.preprocess(ref_image.resize((224, 224)), return_tensors="pt").pixel_values
    clip_px = clip_px.to(dev, torch.float16)
    ref_t = pipe.ref_image_processor.preprocess(ref_image, height=H, width=W).to(dev, torch.float16)
    pose_t = torch.cat([pipe.cond_image_processor.preprocess(p, height=H, width=W) for p in poses], 0).to(dev, torch.float16)
    lat0 = torch.randn((1, 4, L, H // 8, W // 8), generator=torch.Generator().manual_seed(42),
                       dtype=torch.float16).to(dev)
    arms = [("ddim_25", ddim, 25)]
    arms += [(f"dpmpp_2m_{n}", DPMSolverMultistepScheduler.from_config(ddim.config), n) for n in (10, 15, 20)]
    arms.append(("euler_25", EulerDiscreteScheduler.from_config(ddim.config), 25))

    # the update kernel alone on the loop's tensors: acc [2, L, 64, 64, 4] fp32, latents fp16, history fp32
    acc = torch.zeros(2, L, H // 8, W // 8, 4, dtype=torch.float32, device=dev)
    lat = torch.randn(L, H // 8, W // 8, 4, generator=torch.Generator().manual_seed(1)).to(dev, torch.float16)
    hist = torch.zeros(L, H // 8, W // 8, 4, dtype=torch.float32, device=dev)
    inv = step_weights(torch.ones(L), True).to(dev, torch.float32)

    def kernel_us(fn):
        for _ in range(50):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.launches

    for arm, sched, steps in arms:
        pipe.scheduler = sched
        pipe.run_device(clip_px, ref_t, pose_t, lat0, steps, bench.GUIDANCE, decode=True)     # builds + captures
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pipe.run_device(clip_px, ref_t, pose_t, lat0, steps, bench.GUIDANCE, decode=True)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        t = pipe.collect_timings()
        if arm.startswith("ddim"):
            a_t, a_p = pipe._alpha_pair(int(sched.timesteps[5]))
            kern = "ap_cfg_ddim_step_f16"
            us = kernel_us(lambda: ops.cfg_ddim_step(acc, inv, bench.GUIDANCE, a_t, a_p, lat, "v_prediction", 0.0))
        else:
            table = multistep_coefficients(sched)
            co = max(table, key=lambda c: abs(c.k_1))          # a step that reads and writes the history
            kern = "ap_cfg_multistep_step_f16"
            us = kernel_us(lambda: ops.cfg_multistep_step(acc, inv, bench.GUIDANCE, co, lat, hist))
        med = statistics.median(ms)
        print(json.dumps(dict(arm=arm, steps=steps, device_ms_per_video=round(med, 2), min_ms=round(min(ms), 2),
                              max_ms=round(max(ms), 2), device_ms_per_step=round(med / steps, 2),
                              denoise_ms=round(t["denoise_ms"], 2), decode_ms=round(t["decode_ms"], 2),
                              update_kernel=kern, update_kernel_us=round(us, 2), reps=args.reps,
                              launches=args.launches, gpu=name, power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
