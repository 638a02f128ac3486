"""Times the Audio2Pose head-pose decoder alone (the encoder features are given) two ways on one GPU, with the seeded
full-size a2p weights (8 layers, E = 512; seeded, not the trained checkpoint):

  torch    kv_cached_infer: the incremental decoder in fp32 torch ops (TF32 off), one step captured in a CUDA graph and
           replayed per frame (audio_models/pose_infer.py)
  kernels  PoseDecoder.decode: the folded cross-attention GEMM and the one-launch decoder kernel (ap_pose_decoder_f16)

for T = 150 (a 5 s chunk) and T = 299 (the longest merged last chunk): warm-up, CUDA events around each call, the median,
min and max of --iters calls; µs per frame; the rel-L2 between the two outputs; the card's name and power limit read in
the same run.

    python scripts/bench_pose_decoder.py --out DIR [--iters 20] [--warmup 3]

Writes DIR/bench_pose_decoder.json and prints it. Fails without a CUDA device (there is no CPU measurement).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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


class _FeaturesIn:
    """The model with its audio encoder replaced by given features (kv_cached_infer then runs the decoder alone)."""

    def __init__(self, model, feats):
        self._m = model
        self.audio_encoder = lambda *a, **k: types.SimpleNamespace(last_hidden_state=feats, hidden_states=[feats])

    def __getattr__(self, name):
        return getattr(self._m, name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_pose_decoder: no CUDA device (this script only measures on the GPU)")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from audio_helpers import rel_l2
    from pose_decoder_helpers import build_a2p_full, features
    from aniportrait_b200 import ops
    from aniportrait_b200.audio_models import kv_cached_infer
    from aniportrait_b200.audio_models.pose_decoder import PoseDecoder
    from oracle import audio as OA
    dev = torch.device("cuda:0")
    name, power = card()
    model = build_a2p_full().to(dev)
    dec = PoseDecoder(model)
    id_seed = torch.tensor([OA.ID_SEED], device=dev)
    results = []
    with torch.no_grad():
        for T in (150, 299):
            feats = features(T, seed=T).to(dev)
            f16 = feats.half()
            ref_model = _FeaturesIn(model, feats)
            t_ms = time_calls(lambda: kv_cached_infer(ref_model, None, T, id_seed=id_seed), args.iters, args.warmup)
            k_ms = time_calls(lambda: dec.decode(f16, T, id_seed), args.iters, args.warmup)
            err = rel_l2(dec.decode(f16, T, id_seed), kv_cached_infer(ref_model, None, T, id_seed=id_seed))
            results.append(dict(T=T, torch_graph_ms_median=round(t_ms[0], 3), torch_graph_ms_min=round(t_ms[1], 3),
                                torch_graph_ms_max=round(t_ms[2], 3), kernels_ms_median=round(k_ms[0], 3),
                                kernels_ms_min=round(k_ms[1], 3), kernels_ms_max=round(k_ms[2], 3),
                                torch_graph_us_per_frame=round(1e3 * t_ms[0] / T, 1),
                                kernels_us_per_frame=round(1e3 * k_ms[0] / T, 1),
                                speedup=round(t_ms[0] / k_ms[0], 2), rel_l2=err))
    name2, power2 = card()
    out = dict(metric="Audio2Pose decoder alone (seeded full-size weights), one chunk per call", gpu=name,
               power_limit=power, power_limit_after=power2, cluster_ctas=ops.pose_decoder_ctas(0), iters=args.iters,
               warmup=args.warmup, torch=torch.__version__, results=results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_pose_decoder.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
