"""Times the wav2vec2-base audio encoder + Audio2Mesh head two ways on one GPU, with seeded base-size weights:

  hf      the transformers module in fp32, as scripts/audio2vid.py runs it (oracle/audio.py's call order)
  kernels enable_kernels(model).infer: the library's sm_90a kernels

for a 5 s and a 10 s clip: warm-up, CUDA events, the median of --iters calls each; the rel-L2 between the two Audio2Mesh
outputs; the GFLOP of one call computed from the shapes; the card's name and power limit read in the same run.

    python scripts/bench_audio_encoder.py --out DIR [--iters 20] [--warmup 3]

Writes DIR/bench_audio_encoder.json and prints it. Fails without a CUDA device (there is no CPU measurement).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gflop(samples: int, seq_len: int) -> float:
    """Multiply-adds x 2 of one encoder + Audio2Mesh call (convolutions, projection, positional conv, 12 layers, head)."""
    from aniportrait_b200.audio_models.wav2vec2 import conv_frames
    fr = conv_frames(samples)
    ks = (10, 3, 3, 3, 3, 2, 2)
    f = fr[0] * 512 * 10
    f += sum(fr[i] * 512 * 512 * ks[i] for i in range(1, 7))
    T = seq_len
    f += T * 512 * 768                          # feature projection
    f += T * 768 * 48 * 128                     # grouped positional convolution
    per_layer = T * 768 * 2304 + 2 * T * T * 768 + T * 768 * 768 + 2 * T * 768 * 3072
    f += 12 * per_layer
    f += T * 768 * 512 + T * 512 * 1404         # in_fn, out_fn
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_audio_encoder: no CUDA device (this script only measures on the GPU)")
    torch.backends.cuda.matmul.allow_tf32 = False     # audio2vid runs the module in plain fp32
    torch.backends.cudnn.allow_tf32 = False
    from audio_helpers import build_a2m, rel_l2
    from aniportrait_b200.audio_models import enable_kernels
    from oracle import audio as OA
    dev = torch.device("cuda:0")
    name, power = card()
    hf_model = build_a2m().to(dev)
    k_model = enable_kernels(build_a2m().to(dev))
    results = []
    with torch.no_grad():
        for secs in (5, 10):
            S = 16000 * secs
            T = OA.seq_len_of(S)
            x = OA.waveform(S).to(dev)
            hf_ms = time_calls(lambda: OA.mesh_infer(hf_model, x, T), args.iters, args.warmup)
            k_ms = time_calls(lambda: k_model.infer(x, T), args.iters, args.warmup)
            err = rel_l2(k_model.infer(x, T), OA.mesh_infer(hf_model, x, T))
            gf = gflop(S, T)
            results.append(dict(clip_s=secs, samples=S, seq_len=T, gflop=round(gf, 2),
                                hf_fp32_ms_median=round(hf_ms[0], 3), hf_fp32_ms_min=round(hf_ms[1], 3),
                                hf_fp32_ms_max=round(hf_ms[2], 3), kernels_ms_median=round(k_ms[0], 3),
                                kernels_ms_min=round(k_ms[1], 3), kernels_ms_max=round(k_ms[2], 3),
                                speedup=round(hf_ms[0] / k_ms[0], 2), kernels_tflops=round(gf / k_ms[0], 1),
                                a2m_rel_l2=err))
    name2, power2 = card()
    out = dict(metric="wav2vec2-base + Audio2Mesh, one clip per call", gpu=name, power_limit=power,
               power_limit_after=power2, iters=args.iters, warmup=args.warmup, torch=torch.__version__,
               results=results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_audio_encoder.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
