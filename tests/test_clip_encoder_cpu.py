"""CPU checks of the CLIP image encoder on the library's kernels (aniportrait_b200/models/clip_vision.py): the fp32
restatement oracle/clip.py on pack_encoder()'s layout against the transformers module, the patch / CLS / position operands
against the module's embeddings, the configurations and calls enable_kernels refuses, and the module state it leaves
alone."""
import copy

import pytest
import torch

from clip_helpers import SMALL_SEED, c1_params, clip_pixels, f16_exact, full_clip_encoder, rel_l2, small_clip_encoder
from oracle import clip as OC


def _module_outputs(m, px):
    with torch.no_grad():
        out = m(px)
    return out.image_embeds, out.last_hidden_state


@pytest.mark.parametrize("B", [1, 2])
def test_oracle_matches_module_small(B):
    from aniportrait_b200.models.clip_vision import pack_encoder
    m = f16_exact(small_clip_encoder(SMALL_SEED))
    px = clip_pixels(B)
    emb, last = OC.run(pack_encoder(m), px)
    want_emb, want_last = _module_outputs(m, px)
    assert emb.shape == want_emb.shape and last.shape == want_last.shape == (B, 50, 64)
    assert rel_l2(emb, want_emb) < 1e-5 and rel_l2(last, want_last) < 1e-5


def test_oracle_matches_module_vit_l_14():
    from aniportrait_b200.models.clip_vision import pack_encoder
    m = f16_exact(full_clip_encoder(c1_params()["seeds"]["clip"]))
    px = clip_pixels(1)
    pk = pack_encoder(m)
    assert pk["tokens"] == 257 and pk["patch_w"].shape == (1024, 640) and pk["layers"][0]["qkv_w"].shape == (3072, 1024)
    emb, last = OC.run(pk, px)
    want_emb, want_last = _module_outputs(m, px)
    e1, e2 = rel_l2(emb, want_emb), rel_l2(last, want_last)
    print(f"ViT-L/14 oracle vs fp32 module: image_embeds {e1:.2e}, last_hidden_state {e2:.2e}")
    assert e1 < 1e-5 and e2 < 1e-5


@pytest.mark.parametrize("B", [1, 3])
def test_patch_operands_reproduce_embeddings(B):
    """patchify + CLS column + tiled position residual == vision_model.embeddings(pixels) (both sides in float64, so the
    comparison sees the layout and not the summation order)."""
    from aniportrait_b200 import ops
    from aniportrait_b200.models.clip_vision import pack_encoder
    for m, P in ((f16_exact(small_clip_encoder(SMALL_SEED)), 32), (f16_exact(full_clip_encoder(405)), 14)):
        pk = pack_encoder(m)
        px = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(B), dtype=torch.float64)
        a = OC.patchify(px, P, ops.patch_kpad(P))
        got = a @ pk["patch_w"].double().t() + pk["pos"].double().repeat(B, 1)
        with torch.no_grad():
            want = m.vision_model.embeddings.double()(px)
        assert rel_l2(got, want.reshape(got.shape)) < 1e-6


def test_small_config_head_padding():
    """The small stand-in's 16-wide heads are padded to 64 rows each in q|k|v (zero rows and zero bias)."""
    from aniportrait_b200.models.clip_vision import pack_encoder
    m = small_clip_encoder(SMALL_SEED)
    pk = pack_encoder(m)
    assert (pk["head_dim"], pk["dpad"], pk["heads"]) == (16, 64, 4)
    w, b = pk["layers"][0]["qkv_w"].float(), pk["layers"][0]["qkv_b"]
    assert w.shape == (3 * 4 * 64, 64) and b.shape == (3 * 4 * 64,)
    rows = w.view(3, 4, 64, 64)
    assert rows[:, :, 16:].abs().sum() == 0 and b.view(3, 4, 64)[:, :, 16:].abs().sum() == 0
    q = m.vision_model.encoder.layers[0].self_attn.q_proj.weight.detach().half().float()
    assert torch.equal(rows[0, :, :16].reshape(64, 64), q)


@pytest.mark.parametrize("field,value", [("hidden_act", "relu"), ("num_channels", 4), ("num_attention_heads", 16),
                                         ("num_attention_heads", 2), ("patch_size", 15), ("hidden_size", 96),
                                         ("intermediate_size", 100), ("projection_dim", 20)])
def test_check_config_refuses(field, value):
    from transformers import CLIPVisionConfig
    from aniportrait_b200.models.clip_vision import check_config
    kw = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=4, image_size=224,
              patch_size=32, projection_dim=768)
    kw[field] = value
    if field == "num_attention_heads" and value == 2:
        kw["hidden_size"] = 512            # head dim 256 > 192
    with pytest.raises(NotImplementedError, match=field):
        check_config(CLIPVisionConfig(**kw))


def test_check_config_accepts_test_configs_and_gelu():
    from aniportrait_b200.models.clip_vision import check_config
    check_config(small_clip_encoder(SMALL_SEED).config)
    cfg = copy.deepcopy(small_clip_encoder(SMALL_SEED).config)
    cfg.hidden_act = "gelu"
    check_config(cfg)
    from transformers import CLIPVisionConfig
    check_config(CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                                  image_size=224, patch_size=14, projection_dim=768))


def test_enable_kernels_refuses_unsupported_calls():
    from aniportrait_b200 import _lib
    from aniportrait_b200.models.clip_vision import enable_kernels
    m = enable_kernels(small_clip_encoder(SMALL_SEED))
    px = torch.randn(1, 3, 224, 224)
    with pytest.raises(_lib.ApError):                                      # CPU pixels: no fallback
        m(px)
    with pytest.raises(ValueError, match="doesn't match"):
        m(torch.randn(1, 3, 192, 192))
    with pytest.raises(NotImplementedError, match="interpolate_pos_encoding"):
        m(px, interpolate_pos_encoding=True)
    with pytest.raises(NotImplementedError, match="output_attentions"):
        m(px, output_attentions=True)
    with pytest.raises(NotImplementedError, match="output_hidden_states"):
        m(px, output_hidden_states=True)
    with pytest.raises(TypeError):
        enable_kernels(torch.nn.Linear(2, 2))
    bad = small_clip_encoder(SMALL_SEED)
    bad.config.hidden_act = "relu"
    with pytest.raises(NotImplementedError, match="hidden_act"):
        enable_kernels(bad)


def test_enable_kernels_leaves_module_state_alone():
    from aniportrait_b200.models.clip_vision import enable_kernels, kernels_enabled
    m = small_clip_encoder(SMALL_SEED)
    sd0 = copy.deepcopy(m.state_dict())
    names0 = [n for n, _ in m.named_parameters()]
    mods0 = [n for n, _ in m.named_modules()]
    assert not kernels_enabled(m)
    enable_kernels(m)
    assert kernels_enabled(m) and "forward" in vars(m)
    assert list(m.state_dict()) == list(sd0) and all(torch.equal(m.state_dict()[k], v) for k, v in sd0.items())
    assert [n for n, _ in m.named_parameters()] == names0 and [n for n, _ in m.named_modules()] == mods0
