"""The CLIP image encoder (transformers CLIPVisionModelWithProjection, ViT-L/14 in AniPortrait) on the library's sm_90a
kernels.

The pipelines call `image_encoder(clip_pixels).image_embeds` once per video (the reference's pipeline_pose2vid_long.py:
375-381). Here the module's parameters are packed once to fp16 GEMM operands and the forward pass is:

  pixels [B, 3, 224, 224] (fp16 or fp32) -> ap_patchify_nchw_f16                  -> [B (1 + G^2), Kpad]
  -> ap_gemm_f16 (patch weight with class_embedding in column 3 P^2, position table tiled to B images as the residual)
  -> ap_layernorm_f16 (pre_layrnorm)
  -> L x [LayerNorm, q|k|v GEMM, ap_attention_f16 (one frame per image), out GEMM + residual, LayerNorm,
          GEMM + quick-GELU (AP_GEMM_QUICK_GELU; or erf-GELU), GEMM + residual]                    (pre-LN layers)
  -> ap_layernorm_f16 (post_layernorm) -> ap_gemm_f16 over the CLS rows (a strided A view, lda = (1 + G^2) C, no gather)

`enable_kernels(image_encoder)` rebinds `forward` on the instance; parameters, state dict and module tree are untouched.
There is no fallback: inputs or configurations the kernels do not cover raise.
"""
from __future__ import annotations

import types

import torch

from .. import _lib, ops
from .modeling import PackedCache, f16, f32

ACTIVATIONS = ("quick_gelu", "gelu")     # config.hidden_act values the fc1 epilogue implements
MAX_HEAD_DIM = 192                       # the attention kernel's widest padded head
KERNELS_ATTR = "_aniportrait_kernels"    # set on an encoder whose forward runs on the kernels (part of a session key)


def check_config(cfg) -> None:
    """Raises NotImplementedError naming the first field of a CLIPVisionConfig the kernels do not implement."""
    def refuse(field, why):
        raise NotImplementedError(f"CLIP kernels: config.{field} = {getattr(cfg, field, None)!r} is not supported ({why})")
    if cfg.hidden_act not in ACTIVATIONS:
        refuse("hidden_act", f"only {' / '.join(ACTIVATIONS)}")
    if cfg.num_channels != 3:
        refuse("num_channels", "RGB input only")
    if cfg.image_size % cfg.patch_size:
        refuse("patch_size", f"must divide image_size {cfg.image_size}")
    if cfg.hidden_size % 64 or cfg.hidden_size > 2048:
        refuse("hidden_size", "a multiple of 64, at most 2048")
    if cfg.hidden_size % cfg.num_attention_heads:
        refuse("num_attention_heads", f"must divide hidden_size {cfg.hidden_size}")
    d = cfg.hidden_size // cfg.num_attention_heads
    if d % 8 or d > MAX_HEAD_DIM:
        refuse("num_attention_heads", f"head dim {d} must be a multiple of 8 and at most {MAX_HEAD_DIM}")
    if cfg.intermediate_size % 32:
        refuse("intermediate_size", "a multiple of 32")
    if cfg.projection_dim % 32:
        refuse("projection_dim", "a multiple of 32")


def kernels_enabled(image_encoder) -> bool:
    """True once enable_kernels() has rebound this encoder's forward."""
    return bool(getattr(image_encoder, KERNELS_ATTR, False))


def _pad_heads(w: torch.Tensor, heads: int, dpad: int) -> torch.Tensor:
    """q / k / v weight [heads d, K] or bias [heads d] -> zero rows after each head's d rows (heads dpad rows)."""
    w = w.detach().float()
    if w.dim() == 1:
        return ops.pad_head_rows(w.unsqueeze(1), heads, dpad).squeeze(1)
    return ops.pad_head_rows(w, heads, dpad)


def _ln(norm) -> tuple:
    return f32(norm.weight), f32(norm.bias), float(norm.eps)


def pack_encoder(model) -> dict:
    """fp16 GEMM operands and fp32 biases / norm affines of a CLIPVisionModelWithProjection, in the layout run() reads."""
    cfg = model.config
    check_config(cfg)
    vm = model.vision_model
    emb = vm.embeddings
    C, heads, P = cfg.hidden_size, cfg.num_attention_heads, cfg.patch_size
    d = C // heads
    dpad = ops.head_pad(d)
    kdata, kpad = 3 * P * P, ops.patch_kpad(P)
    pw = torch.zeros(C, kpad, dtype=torch.float32, device=emb.patch_embedding.weight.device)
    pw[:, :kdata] = emb.patch_embedding.weight.detach().float().reshape(C, kdata)
    pw[:, kdata] = emb.class_embedding.detach().float()
    layers = []
    for l in vm.encoder.layers:
        a, mlp = l.self_attn, l.mlp
        layers.append(dict(
            ln1=_ln(l.layer_norm1),
            qkv_w=f16(torch.cat([_pad_heads(p.weight, heads, dpad) for p in (a.q_proj, a.k_proj, a.v_proj)])),
            qkv_b=f32(torch.cat([_pad_heads(p.bias, heads, dpad) for p in (a.q_proj, a.k_proj, a.v_proj)])),
            out_w=f16(a.out_proj.weight), out_b=f32(a.out_proj.bias),
            ln2=_ln(l.layer_norm2),
            fc1_w=f16(mlp.fc1.weight), fc1_b=f32(mlp.fc1.bias),
            fc2_w=f16(mlp.fc2.weight), fc2_b=f32(mlp.fc2.bias)))
    G = cfg.image_size // P
    return dict(patch=P, image_size=cfg.image_size, tokens=1 + G * G, width=C, heads=heads, head_dim=d, dpad=dpad,
                quick_gelu=cfg.hidden_act == "quick_gelu", patch_w=f16(pw), pos=f16(emb.position_embedding.weight),
                pre_ln=_ln(vm.pre_layrnorm), layers=layers, post_ln=_ln(vm.post_layernorm),
                proj_w=f16(model.visual_projection.weight), pos_tiled={})


def _tiled_positions(pk: dict, B: int) -> torch.Tensor:
    """The position table repeated for B images ([B (1 + G^2), C] fp16): the residual of the patch-embedding GEMM. Built
    once per batch size (the first call at a size, before any graph capture of it) and kept with the packed weights."""
    t = pk["pos_tiled"].get(B)
    if t is None:
        t = pk["pos"].repeat(B, 1).contiguous()
        pk["pos_tiled"][B] = t
    return t


def run(pk: dict, pixels: torch.Tensor):
    """The encoder on the library's kernels. pixels: contiguous [B, 3, S, S] fp16 or fp32 on the device, S = image_size.
    Returns (image_embeds fp16 [B, projection_dim], last_hidden_state fp16 [B, 1 + G^2, C])."""
    B = pixels.shape[0]
    T, C, heads, d, dpad = pk["tokens"], pk["width"], pk["heads"], pk["head_dim"], pk["dpad"]
    hp = heads * dpad
    a = ops.patchify(pixels, pk["patch"])
    x = ops.gemm(a, pk["patch_w"], residual=_tiled_positions(pk, B))
    h = ops.layer_norm(x, *pk["pre_ln"])
    quick = pk["quick_gelu"]
    for L in pk["layers"]:
        y = ops.layer_norm(h, *L["ln1"])
        qkv = ops.gemm(y, L["qkv_w"], bias=L["qkv_b"])
        att = ops.attention(qkv[:, :hp], qkv[:, hp:2 * hp], qkv[:, 2 * hp:], n_frames=B, tokens=T, heads=heads,
                            head_dim=d, dpad=dpad)
        h = ops.gemm(att, L["out_w"], bias=L["out_b"], residual=h)
        y = ops.layer_norm(h, *L["ln2"])
        f = ops.gemm(y, L["fc1_w"], bias=L["fc1_b"], quick_gelu=quick, gelu=not quick)
        h = ops.gemm(f, L["fc2_w"], bias=L["fc2_b"], residual=h)
    post = ops.layer_norm(h, *pk["post_ln"])
    cls = post.as_strided((B, C), (T * C, 1))            # row 0 of every image: the pooled output
    return ops.gemm(cls, pk["proj_w"]), h.view(B, T, C)


def _check_call(cfg, pixel_values, interpolate_pos_encoding, kwargs) -> torch.Tensor:
    """Refusals in the order: unsupported options, shape, device. Returns the contiguous fp16 / fp32 pixels."""
    if interpolate_pos_encoding:
        raise NotImplementedError("CLIP kernels: interpolate_pos_encoding=True is not supported")
    for name in ("output_attentions", "output_hidden_states"):
        if kwargs.pop(name, None) or getattr(cfg, name, False):
            raise NotImplementedError(f"CLIP kernels: {name}=True is not supported (only the last hidden state and the "
                                      "image embeddings are computed)")
    if kwargs:
        raise NotImplementedError(f"CLIP kernels: keyword arguments {sorted(kwargs)} are not supported")
    if not isinstance(pixel_values, torch.Tensor):
        raise ValueError("You have to specify pixel_values")
    if pixel_values.dim() != 4 or pixel_values.shape[1] != cfg.num_channels:
        raise ValueError(f"CLIP: pixel_values must be [batch, {cfg.num_channels}, H, W], got {tuple(pixel_values.shape)}")
    h, w = pixel_values.shape[-2:]
    if h != cfg.image_size or w != cfg.image_size:
        raise ValueError(f"Input image size ({h}*{w}) doesn't match model ({cfg.image_size}*{cfg.image_size}).")
    if pixel_values.shape[0] < 1:
        raise ValueError("CLIP: empty batch")
    if not pixel_values.is_cuda:
        raise _lib.ApError("CLIP kernels need the pixels as a CUDA tensor (no CPU fallback)")
    if pixel_values.dtype not in (torch.float16, torch.float32):
        pixel_values = pixel_values.float()
    return pixel_values.contiguous()


def _forward(model, cache: PackedCache, pixel_values=None, interpolate_pos_encoding=False, **kwargs):
    """CLIPVisionModelWithProjection.forward's call shape and result, computed by run()."""
    from transformers.models.clip.modeling_clip import CLIPVisionModelOutput
    return_dict = kwargs.pop("return_dict", None)
    px = _check_call(model.config, pixel_values, interpolate_pos_encoding, kwargs)
    pk = cache.get(model, lambda: pack_encoder(model))
    with torch.no_grad():
        embeds, last = run(pk, px)
    dtype = model.dtype
    if dtype != torch.float16:
        embeds, last = embeds.to(dtype), last.to(dtype)
    out = CLIPVisionModelOutput(image_embeds=embeds, last_hidden_state=last)
    return out.to_tuple() if return_dict is False else out


def enable_kernels(image_encoder):
    """Run a transformers CLIPVisionModelWithProjection instance on the library's kernels: only its bound `forward`
    changes (HF's call shape `forward(pixel_values, interpolate_pos_encoding=False, **kwargs)`, a CLIPVisionModelOutput with
    image_embeds and last_hidden_state in the module's dtype). Batches of any size are supported. Returns the encoder."""
    if not (hasattr(image_encoder, "vision_model") and hasattr(image_encoder, "visual_projection")
            and hasattr(image_encoder, "config")):
        raise TypeError(f"enable_kernels: {type(image_encoder).__name__} is not a CLIPVisionModelWithProjection")
    check_config(image_encoder.config)
    cache = PackedCache()

    def forward(self, pixel_values=None, interpolate_pos_encoding=False, **kwargs):
        return _forward(self, cache, pixel_values, interpolate_pos_encoding, **kwargs)
    image_encoder.forward = types.MethodType(forward, image_encoder)
    setattr(image_encoder, KERNELS_ATTR, True)
    return image_encoder
