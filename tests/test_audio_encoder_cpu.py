"""CPU checks of the wav2vec2 encoder on the library's kernels (aniportrait_b200/audio_models/wav2vec2.py): the fp32 oracle
against the stored reference outputs, the weight repacks against torch's convolutions, the configurations and inputs
enable_kernels refuses, and the module state it leaves alone."""
import copy

import pytest
import torch
import torch.nn.functional as F

from audio_helpers import build_a2m, build_a2p, golden, rel_l2, wav2vec2_base
from oracle import audio as OA


def test_oracle_matches_reference_golden():
    """oracle/audio.py (transformers submodules in the reference wrapper's order) reproduces the unmodified reference's
    last_hidden_state and Audio2Mesh output for the short clip; the re-created weights match the stored checksums."""
    gold = golden(OA.SAMPLES[0])
    m = build_a2m()
    assert OA.state_checksums(m.state_dict()) == gold["a2m_checksums"]
    a2p = build_a2p(gold)
    assert OA.state_checksums({k: v for k, v in a2p.state_dict().items() if k != "PPE.pe"}) == gold["a2p_checksums"]
    x = OA.waveform(gold["samples"])
    assert float(x.double().sum()) == gold["waveform_sum"] and float(x.double().square().sum()) == gold["waveform_sq"]
    last, states = OA.encoder_forward(m.audio_encoder, x, gold["seq_len"])
    assert len(states) == 13 and last.shape == (1, gold["seq_len"], 768)
    assert rel_l2(last, gold["last_hidden_state"]) < 1e-5
    assert rel_l2(OA.mesh_infer(m, x, gold["seq_len"]), gold["mesh"]) < 1e-5


@pytest.mark.parametrize("k,T", [(3, 79), (3, 80), (2, 9), (2, 10)])
def test_strided_conv_repack_matches_conv1d(k, T):
    """The [Cout, k*C] tap-major repack over frame pairs (A row m = frames 2m, 2m+1 with row stride 2C, plus frame 2m+2
    for k = 3) is F.conv1d(stride=2)."""
    from aniportrait_b200 import ops
    g = torch.Generator().manual_seed(k * 100 + T)
    C = 64
    x = torch.randn(T, C, generator=g)
    w = torch.randn(48, C, k, generator=g)
    want = F.conv1d(x.t().unsqueeze(0), w, stride=2)[0].t()
    to = (T - k) // 2 + 1
    wp = ops.pack_conv1d_weight(w).float()
    a = x.as_strided((to, 2 * C), (2 * C, 1))
    if k == 3:
        a = torch.cat([a, x[2:].as_strided((to, C), (2 * C, 1))], 1)
    assert rel_l2(a @ wp.t(), want) < 2e-3            # fp16 weights


def test_positional_conv_repack_matches_module():
    """Weight norm folded in fp32 + [C, K, C/groups] repack, evaluated as a per-group im2col matmul, reproduces the module's
    pos_conv_embed (conv, SamePad, GELU)."""
    from aniportrait_b200 import ops
    from aniportrait_b200.audio_models.wav2vec2 import fold_weight_norm
    m = build_a2m()
    pce = m.audio_encoder.encoder.pos_conv_embed
    conv = pce.conv
    T, C, G, K = 42, 768, conv.groups, conv.kernel_size[0]
    x = torch.randn(1, T, C, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = pce(x)[0]
    wp = ops.pack_pos_conv_weight(fold_weight_norm(conv)).float()          # [C, K, C/G]
    xp = F.pad(x[0], (0, 0, K // 2, K // 2))                             # [T + K, C]
    cols = xp.unfold(0, K, 1)[:T]                                        # [T, C, K]
    cpg = C // G
    out = torch.empty(T, C)
    for gi in range(G):
        a = cols[:, gi * cpg:(gi + 1) * cpg].permute(0, 2, 1).reshape(T, K * cpg)
        out[:, gi * cpg:(gi + 1) * cpg] = a @ wp[gi * cpg:(gi + 1) * cpg].reshape(cpg, K * cpg).t()
    got = F.gelu(out + conv.bias.detach())
    assert rel_l2(got, want) < 2e-3


@pytest.mark.parametrize("field,value", [("feat_extract_norm", "layer"), ("do_stable_layer_norm", True),
                                         ("conv_dim", (256,) * 7), ("conv_kernel", (10, 3, 3, 3, 3, 3, 2)),
                                         ("conv_stride", (5, 2, 2, 2, 2, 2, 1)), ("hidden_act", "relu"),
                                         ("feat_extract_activation", "relu"), ("num_attention_heads", 8)])
def test_enable_kernels_rejects_other_configs(field, value):
    from aniportrait_b200.audio_models import enable_kernels
    from aniportrait_b200.audio_models.wav2vec2 import check_config
    from audio_helpers import Audio2MeshStandIn
    from transformers import Wav2Vec2Config
    cfg = Wav2Vec2Config(**{field: value})
    name = "num_attention_heads" if field == "num_attention_heads" else field
    with pytest.raises(NotImplementedError, match=name):
        check_config(cfg)
    if field in ("hidden_act", "num_attention_heads", "feat_extract_norm"):      # a few through the public entry point
        m = Audio2MeshStandIn(wav2vec2_base(num_hidden_layers=1, **{field: value}))
        with pytest.raises(NotImplementedError, match=name):
            enable_kernels(m)


def test_enable_kernels_rejects_unsupported_inputs():
    from aniportrait_b200 import _lib
    from aniportrait_b200.audio_models import enable_kernels
    m = enable_kernels(build_a2m())
    enc = m.audio_encoder
    x = OA.waveform(4000)
    with pytest.raises(_lib.ApError):                                    # CPU input: no fallback
        enc(x, seq_len=8)
    with pytest.raises(_lib.ApError):
        m.infer(x, 8)
    with pytest.raises(NotImplementedError, match="batch"):
        enc(x.repeat(2, 1), seq_len=8)
    with pytest.raises(NotImplementedError, match="attention_mask"):
        enc(x, seq_len=8, attention_mask=torch.ones(1, 4000, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="mask_time_indices"):
        enc(x, seq_len=8, mask_time_indices=torch.zeros(1, 8, dtype=torch.bool))
    with pytest.raises(NotImplementedError, match="output_attentions"):
        enc(x, seq_len=8, output_attentions=True)
    with pytest.raises(ValueError, match="400"):
        enc(x[:, :399], seq_len=1)
    with pytest.raises(TypeError):
        enable_kernels(torch.nn.Linear(2, 2))


def test_enable_kernels_leaves_module_state_alone():
    """Only bound methods change: the state dict (keys and values), named_parameters() and the module tree are the same."""
    from aniportrait_b200.audio_models import enable_kernels, enable_kv_cache
    m = build_a2m()
    sd0 = copy.deepcopy(m.state_dict())
    names0 = [n for n, _ in m.named_parameters()]
    mods0 = [n for n, _ in m.named_modules()]
    enable_kernels(m)
    assert list(m.state_dict()) == list(sd0) and all(torch.equal(m.state_dict()[k], v) for k, v in sd0.items())
    assert [n for n, _ in m.named_parameters()] == names0 and [n for n, _ in m.named_modules()] == mods0
    assert "forward" in vars(m.audio_encoder) and "infer" in vars(m)
    p = build_a2p(golden(OA.SAMPLES[0]))
    keys = list(p.state_dict())
    enable_kv_cache(enable_kernels(p))
    assert list(p.state_dict()) == keys and "infer" in vars(p)
