"""Times the CLIP ViT-L/14 image encoder at batch 1 on one GPU, with seeded weights (tests/helpers.full_clip_encoder), four
ways:

  hf_eager        the transformers CLIPVisionModelWithProjection in fp16, as the pipelines run it without kernels
  hf_graph        the same module captured once into a CUDA graph and replayed
  kernels_eager   clip_vision.enable_kernels(module): the library's sm_90a kernels
  kernels_graph   the kernel path captured once into a CUDA graph and replayed

Each: warm-up, CUDA events around every call, the median of --iters calls. Also the rel-L2 of both fp16 paths' image_embeds
against the fp32 module, the GFLOP of one call computed from the shapes, and the card's name and power limit read in the
same run.

    python scripts/bench_clip_encoder.py --out DIR [--iters 100] [--warmup 10]

Writes DIR/bench_clip_encoder.json and prints it. Fails without a CUDA device (there is no CPU measurement).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gflop(B: int = 1, C: int = 1024, T: int = 257, F: int = 4096, layers: int = 24, kpatch: int = 588,
          proj: int = 768) -> float:
    """Multiply-adds x 2 of one call: patch embedding, per layer q|k|v, QK^T, PV, out, fc1, fc2, and the projection."""
    M = B * T
    f = M * kpatch * C
    f += layers * (M * C * 3 * C + 2 * B * T * T * C + M * C * C + 2 * M * C * F)
    f += B * C * proj
    return 2.0 * f / 1e9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return name, power


def time_calls(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times), max(times)


def captured(fn):
    """fn() captured once into a CUDA graph (after an eager warm-up on the capture stream); returns (replay, outputs)."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g.replay, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_encoder: no CUDA device (this script only measures on the GPU)")
    torch.backends.cuda.matmul.allow_tf32 = False      # the fp32 module is the accuracy yardstick
    torch.backends.cudnn.allow_tf32 = False
    from clip_helpers import c1_params, clip_pixels, full_clip_encoder, rel_l2
    from aniportrait_b200.models.clip_vision import enable_kernels
    dev = torch.device("cuda:0")
    name, power = card()
    m32 = full_clip_encoder(c1_params()["seeds"]["clip"]).to(dev)
    hf = copy.deepcopy(m32).half()
    kern = enable_kernels(copy.deepcopy(m32).half())
    px = clip_pixels(1).to(dev, torch.float16)
    res = {}
    with torch.no_grad():
        want = m32(px.float()).image_embeds
        for label, mod in (("hf", hf), ("kernels", kern)):
            fn = lambda mod=mod: mod(px).image_embeds  # noqa: E731
            eager = time_calls(fn, args.iters, args.warmup)
            r = dict(eager_ms_median=round(eager[0], 4), eager_ms_min=round(eager[1], 4),
                     eager_ms_max=round(eager[2], 4), image_embeds_rel_l2_vs_fp32=rel_l2(fn(), want))
            try:
                replay, out = captured(fn)
                replay()
                torch.cuda.synchronize()
                graph = time_calls(replay, args.iters, args.warmup)
                r.update(graph_ms_median=round(graph[0], 4), graph_ms_min=round(graph[1], 4),
                         graph_ms_max=round(graph[2], 4), graph_equals_eager=bool(torch.equal(out, fn())))
            except Exception as e:   # a module that cannot be captured: report it, keep the eager numbers
                torch.cuda.synchronize()
                r["graph_error"] = f"{type(e).__name__}: {e}"
            res[label] = r
    gf = gflop()
    for r in res.values():
        r["eager_tflops"] = round(gf / r["eager_ms_median"], 1)
        if "graph_ms_median" in r:
            r["graph_tflops"] = round(gf / r["graph_ms_median"], 1)
    name2, power2 = card()
    out = dict(metric="CLIP ViT-L/14 image encoder, batch 1, fp16", gpu=name, power_limit=power,
               power_limit_after=power2, iters=args.iters, warmup=args.warmup, gflop=round(gf, 1),
               torch=torch.__version__, **res)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_clip_encoder.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
