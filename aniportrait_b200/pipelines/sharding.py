"""Host-side work partitioning of the denoising loop (SURVEY.md §8e). Pure Python / CPU torch: unit-testable with gloo.

Within one DDIM step every context window is an independent UNet call (reference pipeline_pose2vid_long.py:519-548);
their predictions are summed per frame; under CFG the sums are divided by the per-frame window count and CFG-combined,
without CFG the reference steps on the sums themselves (:551-559). Sharding the windows over ranks therefore needs
exactly one sum-all-reduce of the fp32 accumulator per step."""
from __future__ import annotations

from typing import List

import torch

from .context import get_context_scheduler


def plan_windows(num_frames: int, num_inference_steps: int, context_schedule="uniform", context_frames=16,
                 context_stride=1, context_overlap=4):
    """Window list (frame indices, wrap-around) and per-frame 1/count, as the reference computes them every step with
    step=0 (so they are step-invariant)."""
    windows = list(get_context_scheduler(context_schedule)(0, num_inference_steps, num_frames, context_frames,
                                                           context_stride, context_overlap))
    counts = torch.zeros(num_frames)
    for wd in windows:
        for f in set(wd):     # a frame repeated inside one window counts once (reference :546-548: counter[:, :, c] += 1)
            counts[f] += 1
    if (counts == 0).any():
        raise ValueError("context schedule leaves frames uncovered")
    return windows, 1.0 / counts


def windows_of_rank(windows: List[List[int]], rank: int, world: int, shard: bool) -> List[List[int]]:
    """Static round-robin assignment (every rank must derive the same plan without communication)."""
    if not shard or world == 1:
        return list(windows)
    return [wd for i, wd in enumerate(windows) if i % world == rank]


def plan_units(n_windows: int, cfg: bool, world: int, cond_cost: float = 1.2) -> List[List[tuple]]:
    """(window, CFG branch) work units of one denoising step, statically assigned to ranks (SURVEY.md §8e: window-only
    granularity caps an 8-GPU run of 11 windows at 5.5x). Longest-processing-time-first over the unit costs (the
    conditional branch attends to twice the keys: ~1.2x), ties broken by index, so every rank derives the same plan.
    Returns per rank a list of (window_index, branch) with branch in {"both", "uncond", "cond"}; the two branches of a
    window that land on the same rank are fused into one "both" call."""
    if not cfg:
        per = [[] for _ in range(world)]
        for k in range(n_windows):
            per[k % world].append((k, "both"))
        return per
    units = [(cond_cost, k, "cond") for k in range(n_windows)] + [(1.0, k, "uncond") for k in range(n_windows)]
    units.sort(key=lambda u: (-u[0], u[1]))
    load = [0.0] * world
    per = [[] for _ in range(world)]
    for cost, k, br in units:
        r = min(range(world), key=lambda i: (load[i], i))
        load[r] += cost
        per[r].append((k, br))
    out = []
    for lst in per:
        wins = {}
        for k, br in lst:
            wins.setdefault(k, set()).add(br)
        out.append(sorted((k, "both" if len(b) == 2 else next(iter(b))) for k, b in wins.items()))
    return out


def accumulate(acc: torch.Tensor, pred: torch.Tensor, window: List[int]):
    """CPU reference of ap_scatter_accumulate_f16: acc[b, window[f]] += pred[b, f] (acc fp32 [B, L, ...])."""
    last = {f: j for j, f in enumerate(window)}     # repeated frame: its last occurrence wins, counted once
    for f, j in last.items():
        acc[:, f] += pred[:, j].to(acc.dtype)
    return acc


def step_weights(inv_count: torch.Tensor, cfg: bool) -> torch.Tensor:
    """Per-frame weights of the accumulated predictions that ap_cfg_ddim_step_f16 takes as its inv_count. The reference
    divides by the window count only under CFG (:551-552: `noise_pred / counter` sits inside `if
    do_classifier_free_guidance`); without CFG it steps on the sum of the overlapping windows' predictions."""
    return inv_count if cfg else torch.ones_like(inv_count)


def combine(acc: torch.Tensor, inv_count: torch.Tensor, guidance: float):
    """The prediction the reference steps on (:551-557). acc [B, L, ...] -> [L, ...]: B == 2 (CFG) is the overlap average
    then classifier-free guidance, B == 1 the plain sum over the windows."""
    shape = [1, -1] + [1] * (acc.dim() - 2)
    avg = acc * step_weights(inv_count, acc.shape[0] == 2).view(*shape)
    if acc.shape[0] == 2:
        return avg[0] + guidance * (avg[1] - avg[0])
    return avg[0]
