"""The wav2vec2 encoder and the Audio2Mesh head on the sm_90a kernels, on the H100: each new op against fp32 torch, the
whole encoder against the reference goldens and the fp32 oracle, the Audio2Pose chain, reproducibility and the launch set."""
import pytest
import torch
import torch.nn.functional as F

from audio_helpers import build_a2m, build_a2p, golden, rel_l2
from oracle import audio as OA

pytestmark = pytest.mark.gpu
OP_TOL = 2e-3


def _f16(t, dev):
    return t.to(dev, torch.float16).contiguous()


def test_stem_and_groupnorm_gelu(cuda_dev):
    """Conv1d(1, 512, 10, 5) and GroupNorm(512, 512) + GELU at T0 = 31999 (a 10 s clip)."""
    from aniportrait_b200 import ops
    g = torch.Generator().manual_seed(11)
    x = OA.waveform(160000)[0].to(cuda_dev)
    w = (0.3 * torch.randn(512, 1, 10, generator=g)).to(cuda_dev)
    gam = (1 + 0.1 * torch.randn(512, generator=g)).to(cuda_dev)
    bet = (0.1 * torch.randn(512, generator=g)).to(cuda_dev)
    y = ops.conv1d_stem(x, w.reshape(512, 10).contiguous())
    ref = F.conv1d(x.view(1, 1, -1), w, stride=5)                                  # [1, 512, T0]
    assert y.shape == (31999, 512)
    assert rel_l2(y.float().t(), ref[0]) < OP_TOL
    z = ops.batch_norm_train(y, gam, bet, 1e-5, act="gelu")
    zref = F.gelu(F.group_norm(y.float().t().unsqueeze(0), 512, gam, bet, 1e-5))[0].t()
    assert rel_l2(z, zref) < OP_TOL
    assert torch.equal(z, ops.batch_norm_train(y, gam, bet, 1e-5, act="gelu"))


def test_gemm_gelu_epilogue(cuda_dev):
    from aniportrait_b200 import ops
    g = torch.Generator().manual_seed(12)
    for M, K, N in [(150, 768, 3072), (77, 1024, 512)]:
        a = torch.randn(M, K, generator=g)
        w = torch.randn(N, K, generator=g) / K ** 0.5
        b = 0.1 * torch.randn(N, generator=g)
        got = ops.gemm(_f16(a, cuda_dev), _f16(w, cuda_dev), bias=b.to(cuda_dev), gelu=True)
        ref = F.gelu(a.half().float() @ w.half().float().t() + b)
        assert rel_l2(got, ref) < OP_TOL, (M, K, N)


@pytest.mark.parametrize("k,T", [(3, 31999), (3, 15998), (3, 999), (2, 499), (2, 500)])
def test_strided_conv_gemm_matches_conv1d(cuda_dev, k, T):
    from aniportrait_b200 import ops
    g = torch.Generator().manual_seed(k * 7 + T)
    x = torch.randn(T, 512, generator=g)
    w = torch.randn(512, 512, k, generator=g) / (512 * k) ** 0.5
    got = ops.conv1d_s2(_f16(x, cuda_dev), ops.pack_conv1d_weight(w.to(cuda_dev)), k, gelu=True)
    ref = F.gelu(F.conv1d(x.half().float().t().unsqueeze(0).to(cuda_dev), w.half().float().to(cuda_dev), stride=2))[0].t()
    assert got.shape == ref.shape and rel_l2(got, ref) < OP_TOL


@pytest.mark.parametrize("T", [42, 150, 300])
def test_positional_conv(cuda_dev, T):
    """x + pos_conv_embed(x) (weight-normalised grouped conv, SamePad, GELU) of the seeded base model, in fp32 torch."""
    from aniportrait_b200 import ops
    from aniportrait_b200.audio_models.wav2vec2 import fold_weight_norm
    pce = build_a2m().audio_encoder.encoder.pos_conv_embed.to(cuda_dev)
    x = torch.randn(1, T, 768, generator=torch.Generator().manual_seed(T)).to(cuda_dev).half().float()
    with torch.no_grad():
        ref = x + pce(x)
    got = ops.pos_conv1d_gelu(_f16(x[0], cuda_dev), ops.pack_pos_conv_weight(fold_weight_norm(pce.conv)),
                              pce.conv.bias.detach().float().contiguous(), pce.conv.groups)
    assert rel_l2(got, ref[0]) < OP_TOL


@pytest.mark.parametrize("t_in,t_out", [(249, 150), (499, 311), (150, 150), (40, 97), (37, 1), (1, 5)])
def test_resample_rows_linear(cuda_dev, t_in, t_out):
    from aniportrait_b200 import ops
    x = torch.randn(t_in, 512, generator=torch.Generator().manual_seed(t_in)).half()
    got = ops.resample_rows_linear(x.to(cuda_dev), t_out)
    ref = F.interpolate(x.float().t().unsqueeze(0), size=t_out, mode="linear", align_corners=True)[0].t()
    assert rel_l2(got, ref) < OP_TOL


def _kernels_a2m(dev):
    from aniportrait_b200.audio_models import enable_kernels
    return enable_kernels(build_a2m().to(dev))


@pytest.mark.parametrize("samples", OA.SAMPLES)
def test_encoder_and_mesh_match_reference_golden(cuda_dev, samples):
    gold = golden(samples)
    m = _kernels_a2m(cuda_dev)
    x = OA.waveform(samples).to(cuda_dev)
    emb = m.audio_encoder(x, seq_len=gold["seq_len"], output_hidden_states=True)
    assert emb.last_hidden_state.dtype == torch.float32 and emb.last_hidden_state.device == x.device
    assert len(emb.hidden_states) == 13 and emb.attentions is None
    assert torch.equal(emb.hidden_states[-1], emb.last_hidden_state)
    e_feat = rel_l2(emb.last_hidden_state, gold["last_hidden_state"])
    mesh = m.infer(x, gold["seq_len"])
    assert mesh.shape == gold["mesh"].shape and mesh.dtype == torch.float32
    e_mesh = rel_l2(mesh, gold["mesh"])
    print(f"S={samples}: last_hidden_state rel-L2 {e_feat:.2e}, a2m {e_mesh:.2e}")
    assert e_feat < 1e-2 and e_mesh < 1e-2


def test_encoder_matches_oracle_on_gpu_long_clip(cuda_dev):
    """A 10.37 s clip (too big to store): kernels against oracle/audio.py in fp32 on the same device."""
    S = 165920
    T = OA.seq_len_of(S)
    m = _kernels_a2m(cuda_dev)
    x = OA.waveform(S).to(cuda_dev)
    want_last, _ = OA.encoder_forward(m.audio_encoder, x, T, output_hidden_states=False)
    want_mesh = OA.mesh_infer(m, x, T)
    got_last = m.audio_encoder(x, seq_len=T).last_hidden_state
    got_mesh = m.infer(x, T)
    e1, e2 = rel_l2(got_last, want_last), rel_l2(got_mesh, want_mesh)
    print(f"10.37 s clip: last_hidden_state rel-L2 {e1:.2e}, a2m {e2:.2e}")
    assert e1 < 1e-2 and e2 < 1e-2


def test_mean_of_hidden_states_head(cuda_dev):
    """only_last_fetures=False: in_fn over the mean of the 13 hidden states."""
    m = _kernels_a2m(cuda_dev)
    m._only_last_features = False
    x = OA.waveform(OA.SAMPLES[0]).to(cuda_dev)
    T = OA.seq_len_of(OA.SAMPLES[0])
    want = OA.mesh_infer(m, x, T)
    assert rel_l2(m.infer(x, T), want) < 1e-2


@pytest.mark.parametrize("order", ["kernels_first", "kv_cache_first"])
def test_pose_chain_matches_reference(cuda_dev, order):
    from aniportrait_b200.audio_models import enable_kernels, enable_kv_cache
    gold = golden(OA.SAMPLES[0])
    m = build_a2p(gold).to(cuda_dev)
    if order == "kernels_first":
        enable_kv_cache(enable_kernels(m))
    else:
        enable_kernels(enable_kv_cache(m))
    x = OA.waveform(OA.SAMPLES[0]).to(cuda_dev)
    T = gold["seq_len"]
    feats = m.audio_encoder(x, seq_len=T, output_hidden_states=True).last_hidden_state
    pose = m.infer(x, T, id_seed=torch.tensor([OA.ID_SEED], device=cuda_dev))
    e_feat, e_pose = rel_l2(feats, gold["pose_features"]), rel_l2(pose, gold["pose"])
    print(f"a2p ({order}): features rel-L2 {e_feat:.2e}, pose rel-L2 {e_pose:.2e}")
    assert e_feat < 1e-2 and e_pose < 1e-2


def test_two_calls_are_byte_identical(cuda_dev):
    m = _kernels_a2m(cuda_dev)
    x = OA.waveform(OA.SAMPLES[1]).to(cuda_dev)
    T = OA.seq_len_of(OA.SAMPLES[1])
    a = m.infer(x, T)
    b = m.infer(x, T)
    assert torch.equal(a, b)
    e1 = m.audio_encoder(x, seq_len=T, output_hidden_states=True)
    e2 = m.audio_encoder(x, seq_len=T, output_hidden_states=True)
    assert all(torch.equal(p, q) for p, q in zip(e1.hidden_states, e2.hidden_states))


def test_run_launches_only_library_kernels(cuda_dev):
    from torch.profiler import ProfilerActivity, profile
    from aniportrait_b200.audio_models.wav2vec2 import pack_encoder, run
    m = build_a2m().to(cuda_dev)
    pk = pack_encoder(m.audio_encoder)
    wave = OA.waveform(OA.SAMPLES[1])[0].to(cuda_dev)
    T = OA.seq_len_of(OA.SAMPLES[1])
    run(pk, wave, T, hidden_states=True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(pk, wave, T, hidden_states=True)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA
             or getattr(e, "self_device_time_total", 0) > 0]
    names = [n for n in names if "memcpy" not in n.lower() and "memset" not in n.lower()]
    foreign = [n for n in names if "ap::" not in n]
    assert names and not foreign, f"non-library kernels in the wav2vec2 encoder: {foreign}"
