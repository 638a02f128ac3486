"""The Audio2Pose decoder on the kernels, without a GPU: the folded cross-attention, the weight packing, the refused
configurations and inputs, and the untouched module state."""
import copy

import pytest
import torch
import torch.nn.functional as F

from audio_helpers import build_a2p, golden, rel_l2
from oracle import audio as OA
from pose_decoder_helpers import alibi_causal_mask, build_a2p_full, features


def test_full_size_mask_and_table_extend_the_reference_ones():
    """The 600-position mask and positional table the GPU tests use start with the rows the unmodified reference made."""
    from aniportrait_b200.synthetic import _sinusoid_pe
    gold = golden(OA.SAMPLES[0])
    T = gold["seq_len"]
    assert torch.equal(alibi_causal_mask()[:, :T, :T], gold["biased_mask"])
    assert torch.equal(_sinusoid_pe(600, 512)[:, :T], gold["pe"])


@pytest.mark.parametrize("only_last", [True, False])
def test_folded_cross_matches_per_layer_chain(only_last):
    """W f + b of the fold reproduces out_proj(v_proj(in_fn(.))) of every layer, as kv_cached_infer evaluates it, on the
    last hidden state or (only_last=False) on the mean of 13 states when f is their sum."""
    from aniportrait_b200.audio_models.pose_decoder import E, fold_cross
    m = build_a2p_full(only_last)
    states = [features(37, seed=s)[0] for s in range(13 if not only_last else 1)]
    f = sum(states)
    mem = m.in_fn(f / len(states))
    w, b = fold_cross(m, only_last, len(states))
    assert w.dtype == torch.float32 and w.shape == (8 * E, 768) and b.shape == (8 * E,)
    got = f @ w.t() + b
    with torch.no_grad():
        for li, l in enumerate(m.transformer_decoder.layers):
            ca = l.multihead_attn
            want = ca.out_proj(F.linear(mem, ca.in_proj_weight[2 * E:], ca.in_proj_bias[2 * E:]))
            assert rel_l2(got[:, li * E:(li + 1) * E], want) <= 1e-6, li


def test_packed_parameters_unpack_to_the_module():
    from aniportrait_b200 import ops
    from aniportrait_b200.audio_models.pose_decoder import pack_decoder
    m = build_a2p_full()
    pk = pack_decoder(m, True, 1)
    L = pk["layers"]
    off = dict(b_qkv=(0, 1536), b_out=(1536, 2048), b_ff1=(2048, 3072), b_ff2=(3072, 3584), ln1_g=(3584, 4096),
               ln1_b=(4096, 4608), ln2_g=(4608, 5120), ln2_b=(5120, 5632), ln3_g=(5632, 6144), ln3_b=(6144, 6656))
    assert L["vec"].shape == (8, ops.POSE_VEC) and L["vec"].dtype == torch.float32
    for i, l in enumerate(m.transformer_decoder.layers):
        sa = l.self_attn
        for key, p in (("w_qkv", sa.in_proj_weight), ("w_out", sa.out_proj.weight), ("w_ff1", l.linear1.weight),
                       ("w_ff2", l.linear2.weight)):
            assert L[key].dtype == torch.float16 and torch.equal(L[key][i], p.detach().half()), (i, key)
        want = dict(b_qkv=sa.in_proj_bias, b_out=sa.out_proj.bias, b_ff1=l.linear1.bias, b_ff2=l.linear2.bias,
                    ln1_g=l.norm1.weight, ln1_b=l.norm1.bias, ln2_g=l.norm2.weight, ln2_b=l.norm2.bias,
                    ln3_g=l.norm3.weight, ln3_b=l.norm3.bias)
        for key, (a, b) in off.items():
            assert torch.equal(L["vec"][i, a:b], want[key].detach()), (i, key)
    assert pk["eps"] == m.transformer_decoder.layers[0].norm1.eps
    for key, p in (("pose_map_w", m.pose_map.weight), ("pose_map_b", m.pose_map.bias),
                   ("pose_map_r_w", m.pose_map_r.weight), ("pose_map_r_b", m.pose_map_r.bias),
                   ("id_w", m.id_embed.weight)):
        assert pk[key].dtype == torch.float32 and torch.equal(pk[key], p.detach()), key
    assert pk["cross_w"].dtype == torch.float16 and pk["cross_b"].dtype == torch.float32


def _pose_kernels(model):
    from aniportrait_b200.audio_models import enable_kernels
    return enable_kernels(model)


def _refuses(model, exc, match, T=8, id_seed=torch.tensor([OA.ID_SEED]), x=None):
    x = OA.waveform(4000) if x is None else x
    with pytest.raises(exc, match=match):
        model.infer(x, T, id_seed=id_seed)


def test_refused_configurations():
    import torch.nn as nn

    def fresh():
        return _pose_kernels(build_a2p_full())

    m = fresh()
    m.transformer_decoder.layers[3].norm_first = True
    _refuses(m, NotImplementedError, "norm_first")
    m = fresh()
    m.transformer_decoder.norm = nn.LayerNorm(512)
    _refuses(m, NotImplementedError, "final decoder norm")
    m = fresh()
    m.transformer_decoder.layers[0].activation = F.gelu
    _refuses(m, NotImplementedError, "not ReLU")
    for E, heads, ffn in ((256, 8, 1024), (512, 4, 1024), (512, 8, 2048)):
        m = build_a2p_full()
        layer = nn.TransformerDecoderLayer(d_model=E, nhead=heads, dim_feedforward=ffn, batch_first=True)
        m.transformer_decoder = nn.TransformerDecoder(layer, num_layers=2)
        _refuses(_pose_kernels(m), NotImplementedError, "only E = 512")


def test_refused_inputs():
    from aniportrait_b200 import _lib
    from aniportrait_b200.audio_models.pose_decoder import PoseDecoder
    m = _pose_kernels(build_a2p_full())
    _refuses(m, _lib.ApError, "CUDA")                                   # a CPU waveform: no fallback
    _refuses(m, ValueError, "seq_len=601", T=601)                       # beyond the mask / positional table
    _refuses(m, ValueError, "seq_len=0", T=0)
    _refuses(m, TypeError, "id_seed", id_seed=None)
    _refuses(m, IndexError, "out of range", id_seed=torch.tensor([100]))
    _refuses(m, IndexError, "out of range", id_seed=torch.tensor([-1]))
    _refuses(m, NotImplementedError, "batch", id_seed=torch.tensor([1, 2]))
    _refuses(m, NotImplementedError, "batch", x=OA.waveform(4000).repeat(2, 1))
    short = build_a2p(golden(OA.SAMPLES[0]))                          # mask and table cover 42 positions only
    _refuses(_pose_kernels(short), ValueError, "42", T=43)
    dec = PoseDecoder(build_a2p_full())
    with pytest.raises(ValueError, match="fewer than seq_len"):
        dec.decode(features(40).half(), 41, torch.tensor([OA.ID_SEED]))
    with pytest.raises(_lib.ApError, match="CUDA"):
        dec.decode(features(40).half(), 40, torch.tensor([OA.ID_SEED]))


def test_enable_kernels_binds_pose_infer_and_leaves_module_state_alone():
    from aniportrait_b200.audio_models import enable_kernels, enable_kv_cache
    m = build_a2p(golden(OA.SAMPLES[0]))
    sd0 = copy.deepcopy(m.state_dict())
    names0 = [n for n, _ in m.named_parameters()]
    mods0 = [n for n, _ in m.named_modules()]
    enable_kernels(m)
    assert list(m.state_dict()) == list(sd0) and all(torch.equal(m.state_dict()[k], v) for k, v in sd0.items())
    assert [n for n, _ in m.named_parameters()] == names0 and [n for n, _ in m.named_modules()] == mods0
    assert "infer" in vars(m) and "forward" in vars(m.audio_encoder)
    kernel_infer = m.infer
    assert kernel_infer.__func__.__code__.co_varnames[:4] == ("self", "input_value", "seq_len", "id_seed")
    enable_kv_cache(m)                                                # the last rebinding decides
    assert m.infer.__func__ is not kernel_infer.__func__
    enable_kernels(m)
    assert "decoder" in m.infer.__func__.__code__.co_freevars
