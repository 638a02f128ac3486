"""The per-element checks of pose_decoder_reference.py, without a GPU: the fp32 emulation of the decoder kernel passes
them with its unrounded values within half the derived bound, every modelled kernel bug is rejected by a message that
names (step, layer, element), and the fp64 reference run on its own outputs is the module's decoder (kv_cached_infer) in
fp64. Small T and few layers keep it quick; the keys >= 512 models run one layer at one step past 512."""
import re
import types

import pytest
import torch
import torch.nn.functional as F

import pose_decoder_reference as PR

T0, L0, OD0 = 20, 2, 6
ML0, PL0 = 27, 23          # mask_len > pe_len > T: a row stride of T instead of mask_len reads other rows


@pytest.fixture(scope="module")
def params():
    return PR.synthetic_params(L0, OD0, T0, ML0, PL0, seed=1)


CASES = {
    "default": dict(L=L0, od=OD0, T=T0, ml=ML0, pl=PL0),
    "one_layer_one_output": dict(L=1, od=1, T=9, ml=9, pl=9),
    "three_layers_eight_outputs": dict(L=3, od=8, T=13, ml=14, pl=20),
    "causal_mask": dict(L=2, od=6, T=17, ml=17, pl=17, mask="alibi"),
    "eps_1e-3": dict(L=2, od=6, T=12, ml=12, pl=12, eps=1e-3),
}


def _params(c, seed=2):
    return PR.synthetic_params(c["L"], c["od"], c["T"], c["ml"], c["pl"], seed=seed, eps=c.get("eps", 1e-5),
                               mask=c.get("mask", "alibi_finite"))


@pytest.mark.parametrize("name", list(CASES))
def test_emulation_within_half_the_bound(name):
    c = CASES[name]
    P = _params(c)
    out, kv, trace, kv32 = PR.emulate(P, c["T"])
    worst = PR.check(P, c["T"], out, kv, trace, name)
    h = PR.headroom(P, c["T"], out, kv, trace, kv32)
    print(f"\n[checker] {name}: headroom {h:.3f}, worst error / bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert h <= 0.5, h


LONG = ("max_drops_keys_ge_512", "sum_drops_keys_ge_512")


@pytest.mark.parametrize("bug", [b for b in PR.BUGS if b not in LONG])
def test_bug_models_are_rejected(params, bug):
    out, kv, trace, _ = PR.emulate(params, T0, bug=bug)
    with pytest.raises(AssertionError) as ei:
        PR.check(params, T0, out, kv, trace, bug)
    msg = str(ei.value)
    print(f"\n[bug {bug}] {msg[:240]}")
    assert re.search(r"'step': \d+, 'layer': [^,]+, .*'(element|dim)': \d+", msg), msg
    if bug in ("q_fp16", "attn_fp16", "unbiased_var", "no_eps"):       # perturbations of 1e-4 relative or less
        print(f"[bug {bug}] rejected at ratio {float(re.search(r'ratio ([0-9.e+]+)', msg).group(1)):.3g}")


def _one_step_case(i=530, seed=3):
    """One layer at step i > 512: a random fp16 cache of i + 1 rows, a mask row that puts nearly all the weight on keys
    >= 512 (scores of keys < 512 lowered by 200: their exp underflows against the maximum of the others)."""
    T = i + 1
    P = PR.synthetic_params(1, 6, T, T, T, seed=seed)
    g = torch.Generator().manual_seed(seed)
    kc = (torch.randn(PR.HEADS, T, PR.D, generator=g) * 0.5).half()
    vc = torch.randn(PR.HEADS, T, PR.D, generator=g).half()
    m = P["mask"].clone()
    m[:, i, :512] -= 200.0
    P["mask"] = m
    x = torch.randn(PR.E, generator=g)
    return P, i, x, kc, vc


@pytest.mark.parametrize("bug", [None, *LONG])
def test_keys_past_512(bug):
    """The attention stage at step 530: the second score slot of every thread holds keys 512..530."""
    import gemm_reference as GR
    P, i, x, kc, vc = _one_step_case()
    q = PR._gemv32(P["w_qkv"][0][:PR.E], x) + P["vec"][0][:PR.E]
    got = PR._attend32(q.view(PR.HEADS, PR.D), kc, vc, P, i, kc.shape[1], bug).reshape(1, PR.E)
    ref = PR.attn_ref(P, q.view(1, -1), torch.tensor([i]), 0, torch.stack([kc, vc]))
    if bug is None:
        h = GR.headroom(got, ref)
        print(f"\n[checker] step {i}, keys past 512: headroom {h:.3f}")
        assert h <= 0.5
        return
    with pytest.raises(AssertionError, match=r"'step': 530, 'layer': 0, 'stage': 'attention', 'element'"):
        GR.check(got, ref, bug)


class _FeaturesIn:
    def __init__(self, model, feats):
        self._m = model
        self.audio_encoder = lambda *a, **k: types.SimpleNamespace(last_hidden_state=feats, hidden_states=[feats])

    def __getattr__(self, name):
        return getattr(self._m, name)


def test_reference_run_is_the_module_decoder_in_fp64():
    """reference_run on the packed parameters and the per-layer cross rows equals kv_cached_infer in fp64 on the same
    module with its layer weights rounded to fp16 (what the kernel reads)."""
    from aniportrait_b200.audio_models import kv_cached_infer
    from aniportrait_b200.audio_models.pose_decoder import E, pack_decoder
    from pose_decoder_helpers import build_a2p_full, features
    T, idx = 11, 3
    m = build_a2p_full()
    with torch.no_grad():
        for l in m.transformer_decoder.layers:
            for w in (l.self_attn.in_proj_weight, l.self_attn.out_proj.weight, l.linear1.weight, l.linear2.weight):
                w.copy_(w.half().float())
    m = m.double()
    feats = features(T, seed=4).double()
    want = kv_cached_infer(_FeaturesIn(m, feats), None, T, id_seed=torch.tensor([idx]), use_cuda_graph=False)[0]
    pk = pack_decoder(m.float(), True, 1)
    m = m.double()
    with torch.no_grad():
        mem = m.in_fn(feats[0])
        cross = torch.cat([l.multihead_attn.out_proj(F.linear(mem, l.multihead_attn.in_proj_weight[2 * E:],
                                                               l.multihead_attn.in_proj_bias[2 * E:]))
                           for l in m.transformer_decoder.layers], 1)
    P = dict(pk["layers"], pose_map_w=pk["pose_map_w"], pose_map_b=pk["pose_map_b"], pose_map_r_w=pk["pose_map_r_w"],
             pose_map_r_b=pk["pose_map_r_b"], pe=m.PPE.pe.reshape(-1, E), id_row=pk["id_w"][idx],
             mask=m.biased_mask.double(), cross=cross, eps=pk["eps"])
    got, _, _ = PR.reference_run(P, T)
    err = (got - want.double()).abs().max().item()
    print(f"\nreference_run vs kv_cached_infer (fp64): max |diff| {err:.2e}")
    assert err <= 1e-6 * want.abs().max().item()
