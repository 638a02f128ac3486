"""Shared pieces of the CLIP image-encoder tests: the seeded encoders of tests/helpers.py and the C1 golden's CLIP input."""
import os

import torch

from helpers import full_clip_encoder, pipeline_inputs, rel_l2, small_clip_encoder  # noqa: F401

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMALL_SEED = 31


def c1_params() -> dict:
    return torch.load(os.path.join(GOLDEN, "pipeline_c1_full.pt"))["params"]


def f16_exact(m):
    """The module with every parameter rounded to fp16 and kept in fp32: the fp16 packing of such a module is lossless, so
    the packed layout can be compared with the module itself at fp32 precision."""
    return m.half().float().eval()


def clip_pixels(B: int = 1) -> torch.Tensor:
    """[B, 3, 224, 224] fp32: image 0 is what the long pipeline feeds CLIP for the C1 golden (the reference image squashed to
    224 x 224, CLIPImageProcessor); image i > 0 is the reference image of input seed + i, prepared the same way."""
    from transformers import CLIPImageProcessor
    P = c1_params()
    proc = CLIPImageProcessor()
    imgs = []
    for i in range(B):
        ref_image, _, _ = pipeline_inputs(P["size"], 1, P["seeds"]["inputs"] + i)
        imgs.append(proc.preprocess(ref_image.resize((224, 224)), return_tensors="pt").pixel_values)
    return torch.cat(imgs)
