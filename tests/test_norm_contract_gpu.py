"""The call contract of the normalisation, small-convolution and elementwise kernels, element by element against float64
(norm_reference.py), at the shapes their callers use:

  GroupNorm    ap_groupnorm_nhwc_f16 (statistics pass): UNet levels, two-source up-block concats, the VAE, many small
               frames, HW not a multiple of the rows per block, mean / sigma 0..64, the partial-sum workspace refusal
  LayerNorm    ap_layernorm_f16: every caller width (wide and narrow kernels), the 1536 boundary, partial warps and
               blocks, the motion module's positional-encoding table, constant rows; the narrow kernel again in a child
               process with AP_LAYERNORM_NARROW=1
  BatchNorm    ap_batchnorm_train_nhwc_f16: the PoseGuider stem and stages, wav2vec2's GELU layer at 10 s, chunks at
               AP_BN_MAX_BLOCKS with a partial last chunk, a 64-row call
  direct conv  ap_conv2d_direct_nhwc_f16: the PoseGuider stem chain, odd H / W, with and without bias, exact grid
  audio        ap_conv1d_stem_f32, ap_pos_conv1d_gelu_f16, ap_resample_rows_linear_f16
  small        ap_timestep_embedding_f16, ap_add_f16, ap_add_bcast_f16, ap_silu_f16 (every finite fp16), ap_upsample2x
  refusals     pointers off the 16-byte grid return AP_ERR_INVALID and write nothing

Every call goes through the C ABI into a buffer with a guard band that must stay untouched; it runs twice and both
results must be bit-identical; the inputs must be unchanged. The worst ratio of error to bound is printed per case
(run with -s).
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import gemm_reference as GR
import norm_reference as NR
from test_gemm_contract_gpu import _snapshot, _twice, _unchanged

pytestmark = pytest.mark.gpu

CHILD = "AP_NORM_CONTRACT_CHILD"
NARROW = os.environ.get("AP_LAYERNORM_NARROW") is not None


def _report(family, name, ratio):
    print(f"\n[{family}] {name}: worst error / bound = {ratio:.3f}")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _abi(name, *args):
    """One C-ABI call on the current stream; raises ApError on a non-zero return."""
    from aniportrait_b200 import _lib, ops
    ops._ensure(torch.empty(1, device="cuda"))
    rc = getattr(_lib.lib(), name)(*args, _lib.stream_ptr())
    _lib.check(rc, name)


def _f(v):
    return ctypes.c_float(v)


def _run(name, call, out, inputs):
    snap = _snapshot(*inputs)
    _twice(call, out, name)
    _unchanged(snap, name)
    return out.view


def _f16out(rows, cols, dev, pre=64):
    return GR.Guarded(rows, cols, cols, torch.float16, dev, pre=pre)


# ---------------------------------------------------------------------------------------------------- GroupNorm
def gn_call(x, x2, gamma, beta, groups, eps, silu, out_ptr, ws=None):
    from aniportrait_b200._lib import I, fptr, ptr
    nf, hw, c1 = x.shape
    c2 = x2.shape[2] if x2 is not None else 0
    if ws is None:
        ws = torch.empty(2 * groups * (nf + 2 * NR.GN_MAX_BLOCKS), dtype=torch.float32, device=x.device)
    _abi("ap_groupnorm_nhwc_f16", ptr(x), I(c1), ptr(x2), I(c2), I(nf), I(hw), I(groups), _f(eps), fptr(gamma),
         fptr(beta), I(1 if silu else 0), fptr(ws), out_ptr)


def gn_case(name, nf, hw, c1, c2=0, eps=1e-5, silu=True, mean=0.0):
    return dict(name=name, nf=nf, hw=hw, c1=c1, c2=c2, eps=eps, silu=silu, mean=mean)


GN_CASES = [
    # UNet levels of a 64x64 latent, B = 2 windows of 4 frames (blocks.py:185,194 when no column statistics come along;
    # unet_3d.py:273)
    *[gn_case(f"unet_hw{hw}_c{c}", 8, hw, c) for hw, c in ((4096, 320), (1024, 640), (256, 1280), (64, 1280))],
    gn_case("unet_hw1024_c320_no_silu", 8, 1024, 320, silu=False),           # transformer / motion-module norms
    # up-block skip concats [hidden | skip] (blocks.py:185); 640 + 320 has 30 channels per group: group 21 straddles
    gn_case("up_1280_1280", 4, 64, 1280, 1280), gn_case("up_1280_640", 4, 256, 1280, 640),
    gn_case("up_640_320", 4, 1024, 640, 320), gn_case("up_320_320", 4, 4096, 320, 320),
    # VAE decoder norms, eps 1e-6 (vae.py:98,100,246): 128 / 256 channels at 512x512, 512 at 256x256, Nf = 2;
    # every one doubles rows per block to fit AP_GN_MAX_BLOCKS
    gn_case("vae_512x512_c128", 2, 512 * 512, 128, eps=1e-6), gn_case("vae_512x512_c256", 2, 512 * 512, 256, eps=1e-6),
    gn_case("vae_256x256_c512", 2, 256 * 256, 512, eps=1e-6),
    gn_case("many_frames_1200", 1200, 64, 320),                                # rows per block reaches HW
    gn_case("hw1000_partial_chunk", 3, 1000, 320), gn_case("hw1000_two_source", 3, 1000, 640, 320, eps=1e-6),
    *[gn_case(f"mean_over_sigma_{m}", 4, 1024, 320, mean=float(m)) for m in (0, 1, 4, 16, 64)],
    *[gn_case(f"vae_mean_over_sigma_{m}", 2, 512 * 512, 128, eps=1e-6, mean=float(m)) for m in (16, 64)],
]


def _gn_operands(c, dev, seed=11):
    g = _gen(seed)
    x = (torch.randn(c["nf"], c["hw"], c["c1"], generator=g) + c["mean"]).half().to(dev)
    x2 = (torch.randn(c["nf"], c["hw"], c["c2"], generator=g) + c["mean"]).half().to(dev) if c["c2"] else None
    C = c["c1"] + c["c2"]
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev)
    beta = (0.1 * torch.randn(C, generator=g)).to(dev)
    return x, x2, gamma, beta


@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: c["name"])
def test_groupnorm(cuda_dev, case):
    from aniportrait_b200._lib import ptr
    c = case
    x, x2, gamma, beta = _gn_operands(c, cuda_dev)
    C = c["c1"] + c["c2"]
    out = _f16out(c["nf"] * c["hw"], C, cuda_dev)
    got = _run(c["name"], lambda: gn_call(x, x2, gamma, beta, 32, c["eps"], c["silu"], ptr(out.view)), out,
               (x, x2, gamma, beta))
    k, rpb, chunks = NR.gn_geometry(c["hw"], c["c1"], c["nf"])
    ref = NR.gn_ref(x, x2, gamma, beta, 32, c["eps"], c["silu"])
    ratio = GR.check(got, ref, c["name"])
    _report(f"group norm mean/sigma={c['mean']:g}", f"{c['name']} (k {k}, rows/block {rpb}, chunks {chunks})", ratio)


def test_groupnorm_workspace_refusal(cuda_dev):
    """2400 frames of 64 rows need 2400 partial-sum blocks even at rows per block >= HW: AP_ERR_INVALID, nothing written."""
    from aniportrait_b200._lib import ApError, ptr
    nf, hw = 2400, 64
    assert NR.gn_refused(hw, (320,), nf)
    x, _, gamma, beta = _gn_operands(gn_case("r", nf, hw, 320), cuda_dev)
    out = _f16out(nf * hw, 320, cuda_dev)
    with pytest.raises(ApError, match=r"rc=-1\)"):
        gn_call(x, None, gamma, beta, 32, 1e-5, True, ptr(out.view))
    torch.cuda.synchronize()
    assert bool((out.bits == out.sentinel).all()), "the output was written"


# ---------------------------------------------------------------------------------------------------- LayerNorm
def ln_call(x, gamma, beta, eps, pe, rows_per_pe, pe_period, out_ptr, rows=None, C=None):
    from aniportrait_b200._lib import I, LL, fptr, ptr
    _abi("ap_layernorm_f16", ptr(x), LL(rows or x.shape[0]), I(C or x.shape[1]), _f(eps), fptr(gamma), fptr(beta),
         fptr(pe), I(rows_per_pe), I(pe_period), out_ptr)


def ln_case(name, rows, C, F=0, N=0, mean=0.0, const=False):
    return dict(name=name, rows=rows, C=C, F=F, N=N, mean=mean, const=const)


LN_CASES = [
    # UNet transformer norms at the three widths (blocks.py:353,397,568): LPR 8 / 16 / 32; 4101 rows leave a partial
    # warp and a partial block
    *[ln_case(f"unet_c{c}", 4101, c) for c in (320, 640, 1280)],
    ln_case("w2v_c512", 300, 512),                 # wav2vec2.py:121 feature projection LN, 10 s at 30 fps
    ln_case("w2v_c768", 301, 768),                 # wav2vec2.py:124,133,136: LPR 16, 6 vectors per lane (MAXV)
    ln_case("clip_c1024", 2 * 257, 1024),          # clip_vision.py:120,123,128,131: B = 2 images of 257 tokens
    ln_case("boundary_c1536", 1001, 1536),
    *[ln_case(f"narrow_c{c}", 1001, c) for c in (1544, 2048, 322)],
    # motion module: pe[(row // N) % F], rows (b F + f) N + p, B = 2 (blocks.py:564)
    *[ln_case(f"motion_pe_F{F}", 2 * F * 256, 320, F=F, N=256) for F in (4, 16, 24)],
    ln_case("motion_pe_F16_c1280", 2 * 16 * 64, 1280, F=16, N=64),
    *[ln_case(f"mean_over_sigma_{m}", 1001, 320, mean=float(m)) for m in (1, 4, 16, 64)],
    ln_case("constant_rows_c320_pe", 2 * 4 * 64, 320, F=4, N=64, const=True),
    ln_case("constant_rows_c322", 333, 322, const=True),
    ln_case("constant_rows_c768", 301, 768, const=True),
]


def _ln_operands(c, dev, seed=12):
    g = _gen(seed)
    rows, C = c["rows"], c["C"]
    x = torch.randn(rows, C, generator=g) + c["mean"] * torch.randn(rows, 1, generator=g).sign()
    if c["const"]:                                # every other row constant (var = 0), at a few magnitudes
        x[::2] = (torch.randn(rows, 1, generator=g) * 16)[::2]
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev)
    beta = (0.1 * torch.randn(C, generator=g)).to(dev)
    pe = torch.randn(c["F"], C, generator=g).to(dev) if c["F"] else None
    return x.half().to(dev), gamma, beta, pe


@pytest.mark.parametrize("case", LN_CASES, ids=lambda c: c["name"])
def test_layernorm(cuda_dev, case):
    from aniportrait_b200._lib import ptr
    c = case
    x, gamma, beta, pe = _ln_operands(c, cuda_dev)
    rpp, per = (c["N"], c["F"]) if c["F"] else (0, 0)
    out = _f16out(c["rows"], c["C"], cuda_dev)
    got = _run(c["name"], lambda: ln_call(x, gamma, beta, 1e-5, pe, rpp, per, ptr(out.view)), out, (x, gamma, beta, pe))
    ref = NR.ln_ref(x, gamma, beta, 1e-5, pe, max(rpp, 1), max(per, 1), narrow=NARROW)
    ratio = GR.check(got, ref, c["name"])
    if c["const"]:
        want = NR.ln_constant_rows(gamma, beta, pe, c["rows"], max(rpp, 1), max(per, 1))
        bad = (got[::2] != want[::2]).sum().item()
        assert bad == 0, f"{c['name']}: {bad} elements of constant rows differ from fp16(beta + pe)"
    kind = NR.ln_kernel(c["C"], NARROW)
    _report(f"layer norm{' narrow' if NARROW else ''}", f"{c['name']} {kind[0]}<{kind[1]}>", ratio)


def test_layernorm_narrow_in_child_process(cuda_dev):
    """AP_LAYERNORM_NARROW is read at every call but set per process here: every LayerNorm case again in a child pytest,
    where every width takes layernorm_kernel<MAXV>."""
    if os.environ.get(CHILD):
        pytest.skip("already running in the child")
    env = dict(os.environ, AP_LAYERNORM_NARROW="1", **{CHILD: "1"})
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__),
           "-k", "test_layernorm and not child"]
    r = subprocess.run(cmd, env=env, cwd=root, timeout=900, capture_output=True, text=True)
    tail = (r.stdout + r.stderr)
    for line in tail.splitlines():
        if line.startswith("[layer norm narrow]"):
            print("\n" + line)
    assert r.returncode == 0, tail[-4000:]
    assert "[layer norm narrow]" in tail and " passed" in tail


# ---------------------------------------------------------------------------------------------------- BatchNorm
ACT = {"none": 0, "relu": 1, "gelu": 2}


def bn_call(x, gamma, beta, eps, act, out_ptr, rows=None, C=None):
    from aniportrait_b200._lib import I, LL, fptr, ptr
    rows, C = rows or x.shape[0], C or x.shape[1]
    ws = torch.empty(2 * C * (NR.BN_MAX_BLOCKS + 1), dtype=torch.float32, device=x.device)
    _abi("ap_batchnorm_train_nhwc_f16", ptr(x), LL(rows), I(C), fptr(gamma), fptr(beta), _f(eps), I(ACT[act]), fptr(ws),
         LL(ws.numel()), out_ptr)


def bn_case(name, rows, C, act="relu", mean=0.0, pad=0):
    return dict(name=name, rows=rows, C=C, act=act, mean=mean, pad=pad)


BN_CASES = [
    # PoseGuider stem, 3 frames of 512x512 (pose_guider.py:48-49,98,135): conv0 at 512^2 (3 channels padded to 8),
    # then 16 at 256^2, 32 at 128^2, 64 and 128 at 64^2
    bn_case("stem_c8_512x512_pad5", 3 * 512 * 512, 8, pad=5), bn_case("stem_c16_256x256", 3 * 256 * 256, 16),
    bn_case("stem_c32_128x128", 3 * 128 * 128, 32), bn_case("stem_c64_64x64", 3 * 64 * 64, 64),
    bn_case("stem_c128_64x64", 3 * 64 * 64, 128),
    # the 320..1280-wide stages (pose_guider.py:55-58)
    bn_case("stage_c320_32x32", 3 * 32 * 32, 320), bn_case("stage_c640_16x16", 3 * 16 * 16, 640),
    bn_case("stage_c1280_8x8", 3 * 8 * 8, 1280),
    bn_case("w2v_c512_gelu_10s", 31999, 512, act="gelu"),      # wav2vec2.py:117 (conv0 frames of 160000 samples)
    bn_case("act_none", 5000, 64, act="none"),
    bn_case("max_blocks_partial_last", 2048 * 320 - 5, 64),    # 2048 chunks of 320 rows, the last one 315 rows
    bn_case("rows_64", 64, 64),                                # biased and unbiased variance differ by 1/63
    *[bn_case(f"mean_over_sigma_{m}", 3 * 64 * 64, 64, mean=float(m)) for m in (1, 4, 16, 64)],
]


@pytest.mark.parametrize("case", BN_CASES, ids=lambda c: c["name"])
def test_batchnorm(cuda_dev, case):
    from aniportrait_b200._lib import ptr
    c = case
    g = _gen(13)
    x = torch.randn(c["rows"], c["C"], generator=g) + c["mean"]
    gamma, beta = 1 + 0.2 * torch.randn(c["C"], generator=g), 0.1 * torch.randn(c["C"], generator=g)
    if c["pad"]:              # the PoseGuider's padded channels: zero input, gamma = beta = 0 (pose_guider.py:106-107)
        x[:, -c["pad"]:], gamma[-c["pad"]:], beta[-c["pad"]:] = 0, 0, 0
    x, gamma, beta = x.half().to(cuda_dev), gamma.to(cuda_dev), beta.to(cuda_dev)
    out = _f16out(c["rows"], c["C"], cuda_dev)
    got = _run(c["name"], lambda: bn_call(x, gamma, beta, 1e-5, c["act"], ptr(out.view)), out, (x, gamma, beta))
    k, rpb, chunks = NR.bn_geometry(c["rows"], c["C"])
    ratio = GR.check(got, NR.bn_ref(x, gamma, beta, 1e-5, c["act"]), c["name"])
    if c["pad"]:
        assert bool((got[:, -c["pad"]:].float() == 0).all()), "padded channels are not exactly 0"
    _report(f"batch norm {c['act']} mean/sigma={c['mean']:g}", f"{c['name']} (rows/block {rpb}, chunks {chunks})", ratio)


# ---------------------------------------------------------------------------------------------------- direct conv
def dc_call(x, w, bias, stride, pad, out_ptr):
    from aniportrait_b200._lib import I, fptr, ptr
    nf, H, W, cin = x.shape
    _abi("ap_conv2d_direct_nhwc_f16", ptr(x), I(cin), I(nf), I(H), I(W), ptr(w), I(w.shape[0]), I(w.shape[1]),
         I(stride), I(pad), fptr(bias), out_ptr)


def dc_case(name, cin, cout, K, S, nf, H, W, real_cin=0, real_cout=0, bias=True):
    return dict(name=name, cin=cin, cout=cout, K=K, S=S, nf=nf, H=H, W=W, real_cin=real_cin or cin,
                real_cout=real_cout or cout, bias=bias)


DC_CASES = [
    # the PoseGuider stem chain (pose_guider.py:48-49 spec, :97-100 channel padding: cin_have / cout_p), 2 frames at 512^2
    dc_case("stem0_3to3_k3", 8, 8, 3, 1, 2, 512, 512, real_cin=3, real_cout=3),
    dc_case("stem1_3to16_k4s2", 8, 16, 4, 2, 2, 512, 512, real_cin=3),
    dc_case("stem2_16to16_k3", 16, 16, 3, 1, 2, 256, 256),
    dc_case("stem3_16to32_k4s2", 16, 32, 4, 2, 2, 256, 256),
    dc_case("stem4_32to32_k3", 32, 32, 3, 1, 2, 128, 128),
    dc_case("stem5_32to64_k4s2", 32, 64, 4, 2, 2, 128, 128),
    # odd H and W for every stride-2 K = 4 variant; no bias
    *[dc_case(f"odd_{cin}_k4s2", cin, 32, 4, 2, 3, 37, 53) for cin in (8, 16, 32)],
    *[dc_case(f"no_bias_{cin}_k{K}s{S}", cin, ct * 2, K, S, 2, 33, 31, bias=False)
      for cin, K, S, ct in NR.DIRECT_CONV_VARIANTS],
]


@pytest.mark.parametrize("case", DC_CASES, ids=lambda c: c["name"])
def test_direct_conv(cuda_dev, case):
    from aniportrait_b200._lib import ptr
    c = case
    ho, wo = NR.direct_out_hw(c["H"], c["W"], c["K"], c["S"], 1)
    for grid in (True, False):
        g = _gen(14)
        mk_a, mk_w, mk_b, _ = (GR.grid_operands if grid else GR.gauss_operands)(c["K"] ** 2 * c["cin"])
        x = mk_a((c["nf"], c["H"], c["W"], c["cin"]), g)
        w = mk_w((c["cout"], c["K"], c["K"], c["cin"]), g)
        b = mk_b((c["cout"],), g) if c["bias"] else None
        x[..., c["real_cin"]:] = 0
        w[..., c["real_cin"]:] = 0
        w[c["real_cout"]:] = 0
        if b is not None:
            b[c["real_cout"]:] = 0
        x, w = x.to(cuda_dev), w.to(cuda_dev)
        b = b.to(cuda_dev) if b is not None else None
        out = _f16out(c["nf"] * ho * wo, c["cout"], cuda_dev)
        got = _run(c["name"], lambda: dc_call(x, w, b, c["S"], 1, ptr(out.view)), out, (x, w, b))
        ratio = GR.check_both(got, NR.direct_conv_ref(x, w, b, c["S"], 1, exact=grid), c["name"])
        if c["real_cout"] < c["cout"]:
            assert bool((got[:, c["real_cout"]:].float() == 0).all()), "padded output channels are not exactly 0"
        _report("direct conv", f"{c['name']} {'grid' if grid else 'gauss'}", ratio)


# ---------------------------------------------------------------------------------------------------- audio
@pytest.mark.parametrize("samples", [10, 11, 14, 15, 16 * 5 + 10, 160000])
@pytest.mark.parametrize("cout", [512, 64])
def test_conv1d_stem(cuda_dev, samples, cout):
    """wav2vec2.py:116: Conv1d(1, Cout, 10, 5) over the waveform; 90 samples give 17 frames (a partial second block of
    16), 160000 samples (10 s) 31999."""
    from aniportrait_b200._lib import I, LL, fptr, ptr
    T0 = NR.stem_frames(samples)
    for grid in (True, False):
        g = _gen(15)
        if grid:
            wave = torch.randint(-4, 5, (samples,), generator=g) / 4.0
            w = torch.randint(-32, 33, (cout, 10), generator=g) / 32.0
        else:
            wave, w = torch.randn(samples, generator=g), torch.randn(cout, 10, generator=g) * 0.3
        wave, w = wave.float().to(cuda_dev), w.float().to(cuda_dev)
        out = _f16out(T0, cout, cuda_dev)
        name = f"stem S={samples} Cout={cout}"
        got = _run(name, lambda: _abi("ap_conv1d_stem_f32", fptr(wave), LL(samples), fptr(w), I(cout), ptr(out.view)),
                   out, (wave, w))
        ratio = GR.check_both(got, NR.stem_ref(wave, w, exact=grid), name)
        _report("conv1d stem", f"{name} {'grid' if grid else 'gauss'}", ratio)


@pytest.mark.parametrize("T", [1, 31, 32, 33, 63, 64, 65, 600, 1500])
def test_pos_conv(cuda_dev, T):
    """wav2vec2.py:123: x + GELU(Conv1d(768, 768, 128, padding=64, groups=16)[:-1] + b); T < K / 2 included."""
    from aniportrait_b200._lib import I, LL, fptr, ptr
    g = _gen(16)
    K, C = 128, 768
    x = torch.randn(T, C, generator=g).half().to(cuda_dev)
    w = (torch.randn(C, 48, K, generator=g) * (48 * K) ** -0.5).permute(0, 2, 1).half().contiguous().to(cuda_dev)
    b = (0.5 * torch.randn(C, generator=g)).to(cuda_dev)
    out = _f16out(T, C, cuda_dev)
    name = f"pos conv T={T}"
    got = _run(name, lambda: _abi("ap_pos_conv1d_gelu_f16", ptr(x), LL(T), I(C), I(16), I(K), ptr(w), fptr(b),
                                  ptr(out.view)), out, (x, w, b))
    _report("pos conv", name, GR.check(got, NR.pos_conv_ref(x, w, b), name))


# (T_in, T_out): the encoder's (T0 after the feature extractor, seq_len) at 21920 / 80000 / 85920 / 160000 samples
# (oracle/audio.py:35-41, wav2vec2.py:120), up-sampling, a single output row and a single input row
RESAMPLE_CASES = [(68, 42), (249, 150), (268, 162), (499, 300), (42, 68), (150, 499), (68, 1), (1, 42), (1, 1)]


@pytest.mark.parametrize("t_in,t_out", RESAMPLE_CASES)
def test_resample(cuda_dev, t_in, t_out):
    from aniportrait_b200._lib import I, LL, ptr
    x = torch.randn(t_in, 512, generator=_gen(17)).half().to(cuda_dev)
    out = _f16out(t_out, 512, cuda_dev)
    name = f"resample {t_in}->{t_out}"
    got = _run(name, lambda: _abi("ap_resample_rows_linear_f16", ptr(x), LL(t_in), I(512), ptr(out.view), LL(t_out)),
               out, (x,))
    ratio = GR.check(got, NR.resample_ref(x, t_out), name)
    emu = NR.emulate_resample(x, t_out)
    bad = (got.view(torch.int16) != emu.view(torch.int16)).sum().item()
    assert bad == 0, f"{name}: {bad} elements differ from the kernel's formula in fp32"
    _report("resample", name, ratio)


# ---------------------------------------------------------------------------------------------------- small kernels
def _ddim_leading(n, offset):
    """DDIM 'leading' spacing (pipelines/scheduler.py:73): arange(n) * (1000 // n) + steps_offset."""
    return [i * (1000 // n) + offset for i in range(n)]


def test_timestep_embedding(cuda_dev):
    """unet_3d.py:238 / unet_2d_condition.py:142 at dim 320: t in {0, 1, 999} and every leading DDIM timestep of 25 and
    30 steps with steps_offset 0 and 1."""
    from aniportrait_b200._lib import I, fptr, ptr
    ts = sorted({0, 1, 999, *[t for n in (25, 30) for o in (0, 1) for t in _ddim_leading(n, o)]})
    t = torch.tensor(ts, dtype=torch.float32, device=cuda_dev)
    out = _f16out(len(ts), 320, cuda_dev)
    got = _run("timestep", lambda: _abi("ap_timestep_embedding_f16", fptr(t), I(len(ts)), I(320), ptr(out.view)),
               out, (t,))
    _report("timestep embedding", f"{len(ts)} timesteps, dim 320", GR.check(got, NR.timestep_ref(t, 320), "timestep"))


def test_silu_every_finite_f16(cuda_dev):
    from aniportrait_b200._lib import LL, ptr
    x = NR.all_finite_f16(cuda_dev)
    n = x.numel()
    out = _f16out(n, 1, cuda_dev)
    got = _run("silu", lambda: _abi("ap_silu_f16", ptr(x), ptr(out.view), LL(n)), out, (x,))
    _report("silu", f"all {n} finite fp16 values", GR.check(got, NR.silu_ref(x), "silu"))


def test_add_and_add_bcast_cfg_layout(cuda_dev):
    """unet_3d.py:253: the PoseGuider feature [F, 64, 64, 320] added to both CFG halves of [2F, 64, 64, 320] (add_bcast,
    dup = 2), and ap_add_f16 when the shapes match; both bit-identical to torch's fp16 add."""
    from aniportrait_b200._lib import LL, ptr
    g = _gen(18)
    F_, hw, c = 4, 64 * 64, 320
    a = torch.randn(2 * F_ * hw, c, generator=g).half().to(cuda_dev)
    p = torch.randn(F_ * hw, c, generator=g).half().to(cuda_dev)
    out = _f16out(2 * F_ * hw, c, cuda_dev)
    got = _run("add_bcast", lambda: _abi("ap_add_bcast_f16", ptr(a), ptr(p), ptr(out.view), LL(a.numel()),
                                         LL(p.numel())), out, (a, p))
    assert torch.equal(got.view(torch.int16), NR.add_ref(a, p, 2).view(torch.int16)), "add_bcast != torch a + b"
    assert not torch.equal(got, NR.emulate_add_bcast(a, p, 2, bug="interleave"))
    b = torch.randn(2 * F_ * hw, c, generator=g).half().to(cuda_dev)
    out2 = _f16out(2 * F_ * hw, c, cuda_dev)
    got2 = _run("add", lambda: _abi("ap_add_f16", ptr(a), ptr(b), ptr(out2.view), LL(a.numel())), out2, (a, b))
    assert torch.equal(got2.view(torch.int16), (a + b).view(torch.int16)), "add != torch a + b"
    _report("add", "add_bcast dup 2 and add, 2 x 4 x 64 x 64 x 320", 0.0)


def test_upsample2x(cuda_dev):
    from aniportrait_b200._lib import I, ptr
    x = torch.randn(3, 9, 7, 64, generator=_gen(19)).half().to(cuda_dev)
    out = _f16out(3 * 18 * 14, 64, cuda_dev)
    got = _run("upsample2x", lambda: _abi("ap_upsample2x_nhwc_f16", ptr(x), ptr(out.view), I(3), I(9), I(7), I(64)),
               out, (x,))
    want = x.repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1, 64)
    assert torch.equal(got, want)


# ---------------------------------------------------------------------------------------------------- refusals
def _off(t, off):
    """A copy of t as a view `off` elements past the 16-byte grid."""
    flat = torch.zeros(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = torch.as_strided(flat, t.shape, t.stride(), off)
    v.copy_(t)
    return v


def _refusal_call(dev, name, off):
    """(Guarded output, call(out_ptr)) with one pointer of the named entry point `off` elements off the 16-byte grid."""
    from aniportrait_b200._lib import I, LL, ptr
    g = _gen(20)
    entry, arg = name.split(":")
    nf, hw, C = 2, 64, 320
    x = torch.randn(nf, hw, C, generator=g).half().to(dev)
    x2 = torch.randn(nf, hw, C, generator=g).half().to(dev)
    gamma, beta = torch.randn(2 * C, generator=g).to(dev), torch.randn(2 * C, generator=g).to(dev)
    bump = lambda t, a: _off(t, off) if arg == a else t  # noqa: E731
    pre = 64 + off if arg == "out" else 64
    if entry == "groupnorm":
        out = GR.Guarded(nf * hw, 2 * C, 2 * C, torch.float16, dev, pre=pre)
        return out, lambda: gn_call(bump(x, "x"), bump(x2, "x2"), gamma, beta, 32, 1e-5, True, ptr(out.view))
    if entry == "groupnorm_apply":
        cs = torch.zeros(nf * hw // 32, C, 2, device=dev)
        ws = torch.empty(2 * 32 * nf, device=dev)
        out = GR.Guarded(nf * hw, 2 * C, 2 * C, torch.float16, dev, pre=pre)
        from aniportrait_b200._lib import fptr
        return out, lambda: _abi("ap_groupnorm_apply_nhwc_f16", ptr(bump(x, "x")), I(C), ptr(cs), LL(C),
                                 ptr(bump(x2, "x2")), I(C), ptr(cs), LL(C), I(nf), I(hw), I(32), _f(1e-5), fptr(gamma),
                                 fptr(beta), I(1), fptr(ws), ptr(out.view))
    if entry == "layernorm":
        xl = x.view(-1, C)
        pe = torch.randn(4, C, generator=g).to(dev)
        out = GR.Guarded(nf * hw, C, C, torch.float16, dev, pre=pre)
        return out, lambda: ln_call(bump(xl, "x"), bump(gamma[:C].contiguous(), "gamma"),
                                    bump(beta[:C].contiguous(), "beta"), 1e-5, bump(pe, "pe"), 32, 4, ptr(out.view))
    if entry == "batchnorm":
        out = GR.Guarded(nf * hw, C, C, torch.float16, dev, pre=pre)
        return out, lambda: bn_call(bump(x.view(-1, C), "x"), gamma[:C].contiguous(), beta[:C].contiguous(), 1e-5,
                                    "relu", ptr(out.view))
    n = nf * hw * C
    if entry == "add":
        out = GR.Guarded(nf * hw, C, C, torch.float16, dev, pre=pre)
        return out, lambda: _abi("ap_add_f16", ptr(bump(x, "a")), ptr(bump(x2, "b")), ptr(out.view), LL(n))
    if entry == "add_bcast":
        out = GR.Guarded(2 * nf * hw, C, C, torch.float16, dev, pre=pre)
        a = torch.cat([x, x2])
        return out, lambda: _abi("ap_add_bcast_f16", ptr(bump(a, "a")), ptr(bump(x, "b")), ptr(out.view), LL(2 * n),
                                 LL(n))
    if entry == "upsample2x":
        out = GR.Guarded(nf * 4 * hw, C, C, torch.float16, dev, pre=pre)
        return out, lambda: _abi("ap_upsample2x_nhwc_f16", ptr(bump(x.view(nf, 8, 8, C), "x")), ptr(out.view), I(nf),
                                 I(8), I(8), I(C))
    raise KeyError(name)


REFUSALS = ["groupnorm:x", "groupnorm:x2", "groupnorm:out", "groupnorm_apply:x", "groupnorm_apply:x2",
            "groupnorm_apply:out", "layernorm:x", "layernorm:out", "layernorm:gamma", "layernorm:beta", "layernorm:pe",
            "batchnorm:x", "batchnorm:out", "add:a", "add:b", "add:out", "add_bcast:a", "add_bcast:b", "add_bcast:out",
            "upsample2x:x", "upsample2x:out"]


@pytest.mark.parametrize("off", [1, 2])
@pytest.mark.parametrize("name", REFUSALS)
def test_misaligned_refusal(cuda_dev, name, off):
    """A pointer one or two elements off the 16-byte grid is refused with AP_ERR_INVALID before any launch: the output's
    guard band and body keep their sentinels."""
    from aniportrait_b200._lib import ApError
    out, call = _refusal_call(cuda_dev, name, off)
    torch.cuda.synchronize()
    with pytest.raises(ApError, match=r"rc=-1\)"):
        call()
    torch.cuda.synchronize()
    out.check(name)
    assert bool((out.bits == out.sentinel).all()), f"{name}: the output was written"
