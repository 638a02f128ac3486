"""Full-size Audio2Pose inputs for the pose decoder tests and scripts/bench_pose_decoder.py: the causal + ALiBi mask and
the positional table at the reference's 600 positions (the goldens store only their first seq_len rows), the seeded a2p
model built on them, and synthetic encoder features."""
import torch

from audio_helpers import build_a2p
from aniportrait_b200.synthetic import _sinusoid_pe

MAX_LEN = 600    # PositionalEncoding(max_len=600) and init_biased_mask(max_seq_len=600) of the reference


def alibi_causal_mask(heads: int = 8, n: int = MAX_LEN) -> torch.Tensor:
    """[heads, n, n] fp32: -slope_h * (i - j) for key j <= query i, -inf above the diagonal, with the ALiBi slopes
    2^(-8 (h + 1) / heads) (Press et al., period 1)."""
    slopes = torch.tensor([2.0 ** (-8.0 * (h + 1) / heads) for h in range(heads)], dtype=torch.float32)
    i = torch.arange(n).unsqueeze(1)
    j = torch.arange(n).unsqueeze(0)
    dist = (i - j).float()
    mask = -slopes.view(heads, 1, 1) * dist
    return mask.masked_fill((j > i).unsqueeze(0), float("-inf"))


def build_a2p_full(only_last: bool = True):
    """The seeded a2p stand-in of audio_helpers with the full 600-position mask and positional table."""
    m = build_a2p({"pe": _sinusoid_pe(MAX_LEN, 512), "biased_mask": alibi_causal_mask()})
    m._only_last_features = only_last
    return m


def features(frames: int, seed: int = 0) -> torch.Tensor:
    """Synthetic encoder features [1, frames, 768], fp16-representable (the encoder hands the decoder fp16)."""
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.randn(1, frames, 768, generator=g).half().float()
