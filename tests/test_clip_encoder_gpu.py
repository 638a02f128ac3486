"""The CLIP image encoder on the sm_90a kernels, on the H100: patchify and the quick-GELU epilogue against torch, the whole
ViT-L/14 encoder against the same module in fp32, batch independence, reproducibility, the launch set, the C1 pipeline
golden with the kernel encoder, and a session captured on the HF encoder not being replayed after enable_kernels."""
import copy
import os
import warnings

import pytest
import torch

from clip_helpers import (GOLDEN, SMALL_SEED, c1_params, clip_pixels, full_clip_encoder, pipeline_inputs, rel_l2,
                          small_clip_encoder)
from oracle import clip as OC

pytestmark = pytest.mark.gpu
OP_TOL = 2e-3
ENC_TOL = 5e-3


@pytest.fixture(scope="module")
def vit_l(cuda_dev):
    """(fp32 module, fp16 module on the kernels) of the C1 golden's ViT-L/14, on the device."""
    from aniportrait_b200.models.clip_vision import enable_kernels
    m32 = full_clip_encoder(c1_params()["seeds"]["clip"]).to(cuda_dev)
    return m32, enable_kernels(copy.deepcopy(m32).half())


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("B", [1, 3])
def test_patchify_is_bit_exact(cuda_dev, dtype, B):
    from aniportrait_b200 import ops
    px = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(B)).to(cuda_dev, dtype)
    for P in (14, 32):
        got = ops.patchify(px, P)
        want = OC.patchify(px.float(), P, ops.patch_kpad(P)).half()
        assert got.shape == want.shape and torch.equal(got, want), P


@pytest.mark.parametrize("M,K,N", [(257, 1024, 4096), (50, 64, 128)])
def test_gemm_quick_gelu_epilogue(cuda_dev, M, K, N):
    from aniportrait_b200 import ops
    g = torch.Generator().manual_seed(M + N)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = 0.1 * torch.randn(N, generator=g)
    got = ops.gemm(a.to(cuda_dev, torch.float16), w.to(cuda_dev, torch.float16), bias=b.to(cuda_dev), quick_gelu=True)
    y = a.half().float() @ w.half().float().t() + b
    assert rel_l2(got, y * torch.sigmoid(1.702 * y)) < OP_TOL


def test_gemm_refuses_both_gelu_flags(cuda_dev):
    from aniportrait_b200 import _lib, ops
    a = torch.randn(64, 64, device=cuda_dev, dtype=torch.float16)
    w = torch.randn(64, 64, device=cuda_dev, dtype=torch.float16)
    with pytest.raises(_lib.ApError, match="mutually exclusive"):
        ops.gemm(a, w, gelu=True, quick_gelu=True)
    with pytest.raises(_lib.ApError, match="quick-GELU"):
        ops.gemm(a, w, residual=a, quick_gelu=True)


@pytest.mark.parametrize("B", [1, 2])
def test_vit_l_14_matches_fp32_module(cuda_dev, vit_l, B):
    m32, kern = vit_l
    px = clip_pixels(B).to(cuda_dev)
    with torch.no_grad():
        want = m32(px)
        got = kern(px.half())
        hf16 = copy.deepcopy(m32).half()(px.half())
    assert got.image_embeds.dtype == torch.float16 and got.image_embeds.shape == (B, 768)
    assert got.last_hidden_state.shape == (B, 257, 1024)
    e_emb, e_last = rel_l2(got.image_embeds, want.image_embeds), rel_l2(got.last_hidden_state, want.last_hidden_state)
    h_emb, h_last = rel_l2(hf16.image_embeds, want.image_embeds), rel_l2(hf16.last_hidden_state, want.last_hidden_state)
    print(f"ViT-L/14 B={B} vs fp32: kernels image_embeds {e_emb:.2e}, last_hidden_state {e_last:.2e}; "
          f"HF fp16 module image_embeds {h_emb:.2e}, last_hidden_state {h_last:.2e}")
    assert e_emb < ENC_TOL and e_last < ENC_TOL


@pytest.mark.parametrize("B", [1, 2])
def test_small_config_matches_fp32_module(cuda_dev, B):
    from aniportrait_b200.models.clip_vision import enable_kernels
    m32 = small_clip_encoder(SMALL_SEED).to(cuda_dev)
    kern = enable_kernels(copy.deepcopy(m32).half())
    px = clip_pixels(B).to(cuda_dev)
    with torch.no_grad():
        want = m32(px)
        got = kern(px)                                   # fp32 pixels into the fp16 module, as HF allows
    e_emb, e_last = rel_l2(got.image_embeds, want.image_embeds), rel_l2(got.last_hidden_state, want.last_hidden_state)
    print(f"small CLIP B={B}: image_embeds {e_emb:.2e}, last_hidden_state {e_last:.2e}")
    assert e_emb < ENC_TOL and e_last < ENC_TOL


def test_batch_images_are_independent_and_calls_reproducible(cuda_dev, vit_l):
    _, kern = vit_l
    px = clip_pixels(2).to(cuda_dev, torch.float16)
    with torch.no_grad():
        both = kern(px)
        again = kern(px)
        for i in range(2):
            one = kern(px[i:i + 1])
            assert torch.equal(one.image_embeds[0], both.image_embeds[i]), i
            assert torch.equal(one.last_hidden_state[0], both.last_hidden_state[i]), i
    assert torch.equal(both.image_embeds, again.image_embeds)
    assert torch.equal(both.last_hidden_state, again.last_hidden_state)


def test_run_launches_only_library_kernels(cuda_dev, vit_l):
    from torch.profiler import ProfilerActivity, profile
    from aniportrait_b200.models.clip_vision import pack_encoder, run
    pk = pack_encoder(vit_l[1])
    px = clip_pixels(1).to(cuda_dev, torch.float16)
    run(pk, px)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(pk, px)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA
             or getattr(e, "self_device_time_total", 0) > 0]
    names = [n for n in names if "memcpy" not in n.lower() and "memset" not in n.lower()]
    foreign = [n for n in names if "ap::" not in n]
    assert names and not foreign, f"non-library kernels in the CLIP encoder: {foreign}"


def _c1_run(pipe, P, lat0, trace=None):
    ref_image, poses, ref_pose = pipeline_inputs(P["size"], P["L"], P["seeds"]["inputs"])
    kw = dict(callback=lambda i, t, l: trace.append(l.clone()), callback_steps=1) if trace is not None else {}
    out = pipe(ref_image, poses, ref_pose, P["size"], P["size"], P["L"], P["steps"], P["guidance"],
               latents=lat0.clone(), **kw)
    return out.videos, pipe.last_latents.float().cpu()


def test_pipeline_c1_with_kernel_clip_against_reference_golden(cuda_dev):
    from helpers import build_pipeline
    from aniportrait_b200.models.clip_vision import enable_kernels
    gold = torch.load(os.path.join(GOLDEN, "pipeline_c1_full.pt"))
    P = gold["params"]
    pipe = build_pipeline(P, cuda_dev)
    enable_kernels(pipe.image_encoder)
    g = torch.manual_seed(P["seeds"]["latents"])
    lat0 = torch.randn((1, 4, P["L"], P["size"] // 8, P["size"] // 8), generator=g, dtype=torch.float32).half()
    trace = []
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        video, _ = _c1_run(pipe, P, lat0, trace)
    assert not [w for w in caught if "graph-capturable" in str(w.message)], [str(w.message) for w in caught]
    (S,) = pipe._sessions.values()
    assert S.g_embed is not None, "the CLIP / VAE-encode stage was not captured"
    e_first = rel_l2(trace[0], gold["first_step_latents"])
    e_final = rel_l2(trace[-1], gold["final_latents"])
    st = gold.get("video_pixel_stride", 1)
    e_video = rel_l2(video[:, :, [0, P["L"] - 1], ::st, ::st], gold["video_frames"])
    print(f"C1 pipeline with the kernel CLIP, rel-L2: first step {e_first:.3e}, final latents {e_final:.3e}, "
          f"video frames {e_video:.3e}")
    assert e_first < 1e-2 and e_final < 1e-2 and e_video < 1e-2
    v_replay, l_replay = _c1_run(pipe, P, lat0)          # second video: pure graph replay
    pipe.use_cuda_graph = False
    v_eager, l_eager = _c1_run(pipe, P, lat0)
    assert torch.equal(l_replay, l_eager) and torch.equal(v_replay, v_eager)


def test_enable_kernels_after_a_captured_video_takes_effect(cuda_dev):
    """A session captured on the HF encoder must not be replayed once the encoder runs on the kernels: the second video's
    encoder_hidden_states are the kernel path's embedding."""
    from helpers import build_pipeline
    from aniportrait_b200.models.clip_vision import enable_kernels
    P = torch.load(os.path.join(GOLDEN, "pipeline_small.pt"))["params"]
    pipe = build_pipeline(P, cuda_dev)
    L, steps = 4, 2
    ref_image, poses, ref_pose = pipeline_inputs(P["size"], L, P["seeds"]["inputs"])
    lat0 = torch.randn((1, 4, L, P["size"] // 8, P["size"] // 8), generator=torch.manual_seed(3)).half()

    def video():
        pipe(ref_image, poses, ref_pose, P["size"], P["size"], L, steps, P["guidance"], latents=lat0.clone())
        return list(pipe._sessions.values())[-1]
    S_hf = video()
    hf_emb = S_hf.ehs[-1, 0].clone()
    enable_kernels(pipe.image_encoder)
    S = video()
    with torch.no_grad():
        want = pipe.image_encoder(S.clip_in).image_embeds[0].half()
    assert S is not S_hf
    assert torch.equal(S.ehs[-1, 0], want)
    assert not torch.equal(hf_emb, want)
