"""The Audio2Pose decoder on the sm_90a kernels, on the H100: the one-launch decoder against the fp32 KV-cached torch
decoder (kv_cached_infer) at every chunk length, the whole infer chain against the unmodified reference's stored output,
refusals before any launch, reproducibility, streams, and the launch set."""
import types

import pytest
import torch

from audio_helpers import build_a2p, golden, rel_l2
from oracle import audio as OA
from pose_decoder_helpers import build_a2p_full, features

pytestmark = pytest.mark.gpu
TOL = 2e-3


class _FeaturesIn:
    """The model with its audio encoder replaced by given features, for kv_cached_infer (the decoder alone)."""

    def __init__(self, model, feats):
        self._m = model
        self.audio_encoder = lambda *a, **k: types.SimpleNamespace(last_hidden_state=feats, hidden_states=[feats])

    def __getattr__(self, name):
        return getattr(self._m, name)


@pytest.fixture(scope="module")
def a2p(cuda_dev):
    return build_a2p_full().to(cuda_dev)


def _decoder(model):
    from aniportrait_b200.audio_models.pose_decoder import PoseDecoder
    return PoseDecoder(model)


def _id(dev, i=OA.ID_SEED):
    return torch.tensor([i], device=dev)


@pytest.mark.parametrize("T", [1, 2, 42, 150, 299, 600])
def test_decoder_matches_kv_cached_fp32(cuda_dev, a2p, T):
    from aniportrait_b200.audio_models import kv_cached_infer
    feats = features(T, seed=T).to(cuda_dev)
    want = kv_cached_infer(_FeaturesIn(a2p, feats), None, T, id_seed=_id(cuda_dev))
    got = _decoder(a2p).decode(feats.half(), T, _id(cuda_dev))
    assert got.shape == want.shape == (1, T, 6) and got.dtype == torch.float32
    q = max(1, T // 4)
    err, err_last = rel_l2(got, want), rel_l2(got[:, -q:], want[:, -q:])
    print(f"T={T}: rel-L2 {err:.2e}, last quarter {err_last:.2e}")
    assert err <= TOL and err_last <= TOL


@pytest.mark.parametrize("order", ["kernels_only", "kv_cache_then_kernels"])
def test_infer_chain_matches_reference_golden(cuda_dev, order):
    from aniportrait_b200.audio_models import enable_kernels, enable_kv_cache
    gold = golden(OA.SAMPLES[0])
    m = build_a2p(gold).to(cuda_dev)
    if order == "kv_cache_then_kernels":
        enable_kv_cache(m)
    enable_kernels(m)
    x = OA.waveform(OA.SAMPLES[0]).to(cuda_dev)
    pose = m.infer(x, gold["seq_len"], id_seed=_id(cuda_dev))
    assert pose.shape == gold["pose"].shape and pose.dtype == torch.float32
    err = rel_l2(pose, gold["pose"])
    print(f"infer chain ({order}) vs reference golden: rel-L2 {err:.2e}")
    assert err <= 1e-2


def test_infer_chain_mean_of_hidden_states(cuda_dev):
    """_only_last_features=False: the sum of the 13 states through the fold with 1/13, against the fp32 torch chain
    (oracle/audio.py's encoder, the mean of its hidden states, kv_cached_infer)."""
    from aniportrait_b200.audio_models import enable_kernels, kv_cached_infer
    ref = build_a2p_full(only_last=False).to(cuda_dev)
    m = enable_kernels(build_a2p_full(only_last=False).to(cuda_dev))
    x = OA.waveform(OA.SAMPLES[0]).to(cuda_dev)
    T = OA.seq_len_of(OA.SAMPLES[0])
    _, states = OA.encoder_forward(ref.audio_encoder, x, T, output_hidden_states=True)
    want = kv_cached_infer(_FeaturesIn(ref, sum(states) / len(states)), None, T, id_seed=_id(cuda_dev))
    got = m.infer(x, T, id_seed=_id(cuda_dev))
    err = rel_l2(got, want)
    print(f"only_last_features=False, T={T}: rel-L2 {err:.2e}")
    assert err <= 1e-2


def test_too_long_raises_before_any_launch(cuda_dev, a2p):
    from aniportrait_b200 import ops
    from aniportrait_b200.audio_models import enable_kernels
    m = enable_kernels(build_a2p_full().to(cuda_dev))
    x = OA.waveform(OA.SAMPLES[2]).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    with pytest.raises(ValueError, match="601"):
        m.infer(x, 601, id_seed=_id(cuda_dev))
    with pytest.raises(ValueError, match="601"):
        _decoder(a2p).decode(features(601).to(cuda_dev).half(), 601, _id(cuda_dev))
    assert ops.KERNEL_LAUNCHES == n0


def test_reproducible_and_independent_of_history(cuda_dev, a2p):
    feats = features(299, seed=5).to(cuda_dev).half()
    dec = _decoder(a2p)
    a = dec.decode(feats, 299, _id(cuda_dev))
    b = dec.decode(feats, 299, _id(cuda_dev))
    assert torch.equal(a, b)
    mid = dec.decode(feats, 150, _id(cuda_dev))
    again = dec.decode(feats, 299, _id(cuda_dev))
    assert torch.equal(again, a)
    assert torch.equal(mid, _decoder(a2p).decode(feats, 150, _id(cuda_dev)))
    assert not torch.equal(dec.decode(feats, 299, _id(cuda_dev, OA.ID_SEED + 1)), a)


def test_non_default_stream(cuda_dev, a2p):
    feats = features(150, seed=6).to(cuda_dev).half()
    dec = _decoder(a2p)
    want = dec.decode(feats, 150, _id(cuda_dev))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = dec.decode(feats, 150, _id(cuda_dev))
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(got, want)


def test_cluster_size_is_chosen_once(cuda_dev):
    from aniportrait_b200 import ops
    n = ops.pose_decoder_ctas(0)
    assert n in (8, 16) and ops.pose_decoder_ctas(0) == n
    print(f"pose decoder cluster: {n} CTAs")


@pytest.mark.parametrize("T", [42, 150])
def test_infer_launches_only_library_kernels_and_one_decoder(cuda_dev, T):
    from torch.profiler import ProfilerActivity, profile
    from aniportrait_b200.audio_models import enable_kernels
    m = enable_kernels(build_a2p_full().to(cuda_dev))
    S = {42: OA.SAMPLES[0], 150: OA.SAMPLES[1]}[T]
    x = OA.waveform(S).to(cuda_dev)
    m.infer(x, T, id_seed=_id(cuda_dev))           # packs the weights and copies the mask once
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.infer(x, T, id_seed=_id(cuda_dev))
        torch.cuda.synchronize()
    events = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA
              or getattr(e, "self_device_time_total", 0) > 0]
    events = [e for e in events if "memcpy" not in e.key.lower() and "memset" not in e.key.lower()]
    foreign = [e.key for e in events if "ap::" not in e.key]
    assert events and not foreign, f"non-library kernels in Audio2Pose infer: {foreign}"
    decoder = [e for e in events if "pose_decoder_kernel" in e.key]
    assert len(decoder) == 1 and decoder[0].count == 1, [(e.key, e.count) for e in decoder]
