"""fp32 torch restatement of aniportrait_b200.models.clip_vision.run() on the same packed dict: the patchify layout with
its CLS column, the tiled position residual, the padded heads and the strided CLS-row projection. It runs on any device;
tests/test_clip_encoder_cpu.py pins it to the transformers CLIPVisionModelWithProjection it was packed from, so the packing
logic is checked without a GPU."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def patchify(pixels: torch.Tensor, patch: int, kpad: int) -> torch.Tensor:
    """[B, 3, H, W] -> [B (1 + Gh Gw), kpad] in the pixels' dtype: per image a CLS row (1.0 in column 3 P^2), then the
    patches in flatten(2) order with columns (c, ky, kx) (F.unfold's order), zero padded."""
    B = pixels.shape[0]
    cols = F.unfold(pixels, kernel_size=patch, stride=patch).transpose(1, 2)          # [B, G^2, 3 P^2]
    kdata = cols.shape[-1]
    out = torch.zeros(B, 1 + cols.shape[1], kpad, dtype=pixels.dtype, device=pixels.device)
    out[:, 0, kdata] = 1
    out[:, 1:, :kdata] = cols
    return out.reshape(-1, kpad)


def _ln(x, norm):
    g, b, eps = norm
    return F.layer_norm(x, (x.shape[-1],), g.float(), b.float(), eps)


@torch.no_grad()
def run(pk: dict, pixels: torch.Tensor):
    """-> (image_embeds [B, projection_dim], last_hidden_state [B, 1 + G^2, C]) in fp32 on the pixels' device."""
    dev = pixels.device
    f = lambda t: t.to(dev, torch.float32)  # noqa: E731
    B = pixels.shape[0]
    T, C, heads, d, dpad = pk["tokens"], pk["width"], pk["heads"], pk["head_dim"], pk["dpad"]
    hp = heads * dpad
    a = patchify(pixels.float(), pk["patch"], pk["patch_w"].shape[1])
    h = a @ f(pk["patch_w"]).t() + f(pk["pos"]).repeat(B, 1)
    h = _ln(h, pk["pre_ln"])
    for L in pk["layers"]:
        y = _ln(h, L["ln1"])
        qkv = y @ f(L["qkv_w"]).t() + f(L["qkv_b"])
        q, k, v = (qkv[:, i * hp:(i + 1) * hp].reshape(B, T, heads, dpad).transpose(1, 2) for i in range(3))
        p = torch.softmax((q @ k.transpose(-1, -2)) * d ** -0.5, dim=-1)                # zero pad columns add nothing
        att = (p @ v)[..., :d].transpose(1, 2).reshape(B * T, heads * d)
        h = h + att @ f(L["out_w"]).t() + f(L["out_b"])
        y = _ln(h, L["ln2"])
        z = y @ f(L["fc1_w"]).t() + f(L["fc1_b"])
        z = z * torch.sigmoid(1.702 * z) if pk["quick_gelu"] else F.gelu(z)
        h = h + z @ f(L["fc2_w"]).t() + f(L["fc2_b"])
    post = _ln(h, pk["post_ln"])
    cls = post.as_strided((B, C), (T * C, 1))
    return cls @ f(pk["proj_w"]).t(), h.view(B, T, C)
