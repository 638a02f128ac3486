"""The call contract of the wgmma GEMM / implicit-GEMM conv kernel (ap_gemm_f16, ap_conv3x3_nhwc_f16), element by
element against float64 (gemm_reference.py), at every tile width, epilogue and caller layout:

  variant matrix   every BN of the linear epilogue, GEGLU at BN 64 / 128, M and K edges, each epilogue feature alone,
                   and outputs / residuals whose bases TMA cannot address (direct-store epilogue)
  caller layouts   UNet resnet / up-block / downsample / conv_in / conv_out convs, the LayerNorm-folded qkv, GEGLU and
                   temporal GEMMs, VAE mid-attention, CLIP, wav2vec2, the pose decoder's cross GEMM, conv grids that
                   are not powers of two
  statistics       row / column partials against fp64 sums of the stored output, GroupNorm from column statistics
  switches         the TMA-less epilogue, single-buffered staging and PDL launches, each in a child process
  refusals         argument combinations the kernel cannot honour return AP_ERR_INVALID and write nothing

Every call writes into a buffer with a guard band (rows after M, columns between n_valid and ldo, elements before the
output) that must stay untouched; inputs must be unchanged, and a second call must give identical bits. Linear
epilogues run twice: on exact-grid operands (bit-exact check) and on Gaussian ones (bounded check). The worst ratio of
error to bound is printed per case (run with -s).
"""
import os
import subprocess
import sys

import pytest
import torch

import gemm_reference as GR

pytestmark = pytest.mark.gpu

CHILD = "AP_GEMM_CONTRACT_CHILD"


def _report(family, name, ratio):
    print(f"\n[{family}] {name}: worst error / bound = {ratio:.3f}")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).clone()


def _snapshot(*ts):
    return [(t, _bits(t)) for t in ts if t is not None]


def _unchanged(snap, what):
    for t, b in snap:
        assert torch.equal(_bits(t), b), f"{what}: an input was modified"


def _twice(call, out: GR.Guarded, what):
    """Runs call() twice into the guarded output; both results must be bit-identical, the guard band intact."""
    call()
    torch.cuda.synchronize()
    first = out.bits.clone()
    call()
    torch.cuda.synchronize()
    assert torch.equal(first, out.bits), f"{what}: two calls differ"
    out.check(what)


def _family(act, out_f32):
    return "fp32 output" if out_f32 else (act or "linear")


def _run_gemm(name, a, w, call, out, refkw, grid):
    from aniportrait_b200 import ops
    snap = _snapshot(a, w, call.get("a2"), call.get("bias"), call.get("residual"))
    _twice(lambda: ops.gemm(a, w, out=out.view, **call), out, name)
    _unchanged(snap, name)
    ref = GR.gemm_ref(a, w, **refkw)
    ratio = GR.check_both(out.view, ref, f"{name} ({'exact grid' if grid else 'gaussian'})")
    _report(_family(refkw.get("act"), refkw.get("out_f32")), f"{name} {'grid' if grid else 'gauss'}", ratio)
    return ratio


# ---------------------------------------------------------------------------------------------------- variant matrix
@pytest.mark.parametrize("case", GR.GEMM_CASES, ids=lambda c: c["name"])
def test_gemm_variant(cuda_dev, case):
    for grid in ((True, False) if case["act"] is None else (False,)):
        a, w, call, out, refkw = GR.build_gemm_case(case, cuda_dev, grid, seed=11)
        _run_gemm(case["name"], a, w, call, out, refkw, grid)


# ---------------------------------------------------------------------------------------------------- caller GEMMs
def _ops(K, grid):
    return GR.grid_operands(K) if grid else GR.gauss_operands(K)


def _caller_gemm(name, dev, grid):
    """(a, w, call, out, refkw) of one caller's GEMM, as the caller lays it out."""
    g = _gen(sum(map(ord, name)))
    if name == "shortcut_1x1_two_source":        # blocks.py:196-199: [x | skip] @ ws.T + bs, 32x32 up-block
        M, K1, K2, N = 2 * 32 * 32, 640, 320, 640
        mk_a, mk_w, mk_b, _ = _ops(K1 + K2, grid)
        a, a2, w, b = mk_a((M, K1), g), mk_a((M, K2), g), mk_w((N, K1 + K2), g), mk_b((N,), g)
        a, a2, w, b = a.to(dev), a2.to(dev), w.to(dev), b.to(dev)
        call = dict(a2=a2, bias=b)
        refkw = dict(a2=a2, bias=b)
    elif name == "vae_wv_xt":                     # vae.py:116: V^T = Wv . X^T  [c, n]
        c, n = 512, 1024
        mk_a, mk_w, _, _ = _ops(c, grid)
        a, w = mk_w((c, c), g).to(dev), mk_a((n, c), g).to(dev)
        M, N = c, n
        call, refkw = {}, {}
    elif name == "vae_scores_n_valid":            # vae.py:117-118: keys zero padded to a multiple of 32, n_valid = n
        n, npad, c = 400, 416, 512
        mk_a, mk_w, _, _ = _ops(c, grid)
        a = mk_a((n, c), g).to(dev)
        k = torch.zeros(npad, c, dtype=torch.float16)
        k[:n] = mk_w((n, c), g)
        w = k.to(dev)
        M, N = n, npad
        call, refkw = dict(n_valid=n), dict(n_valid=n)
    elif name == "vae_pv_k4096":                  # vae.py:120: P . V with K = n = 4096 keys
        n, c = 4096, 512
        mk_a, mk_w, _, _ = _ops(n, grid)
        a, w = mk_a((n, n), g).to(dev), mk_w((c, n), g).to(dev)
        M, N = n, c
        call, refkw = {}, {}
    elif name == "clip_fc1_quick_gelu":           # clip_vision.py:129: fc1 over B * 257 tokens
        M, K, N = 2 * 257, 1024, 4096
        _, mk_w, mk_b, _ = _ops(K, False)
        mk_a = GR.gauss_operands(K)[0]
        a, w, b = mk_a((M, K), g).to(dev), mk_w((N, K), g).to(dev), mk_b((N,), g).to(dev)
        call, refkw = dict(bias=b, quick_gelu=True), dict(bias=b, act="quick_gelu")
    elif name == "clip_proj_strided_cls":         # clip_vision.py:133: projection over the CLS rows, a strided A view
        B, T, K, N = 2, 257, 1024, 768
        mk_a, mk_w, _, _ = _ops(K, grid)
        h = mk_a((B * T, K), g).to(dev)
        a = h.view(B, T, K)[:, 0]
        w = mk_w((N, K), g).to(dev)
        M = B
        call, refkw = {}, {}
    elif name == "w2v_conv1d_s2_gelu":            # ops.py:428-430: overlapping frame pairs + frame 2m+2 as source 2
        T, c, co = 101, 512, 512
        mk_a, mk_w, _, _ = _ops(3 * c, False)
        x = mk_a((T, c), g).to(dev)
        to = (T - 3) // 2 + 1
        a = x.as_strided((to, 2 * c), (2 * c, 1))
        a2 = x[2:].as_strided((to, c), (2 * c, 1))
        w = mk_w((co, 3 * c), g).to(dev)
        M, N = to, co
        call, refkw = dict(a2=a2, gelu=True), dict(a2=a2, act="gelu")
    elif name == "w2v_ffn_gelu":                  # wav2vec2.py:134: feed-forward up-projection
        M, K, N = 101, 1024, 4096
        mk_a, mk_w, mk_b, _ = _ops(K, False)
        a, w, b = mk_a((M, K), g).to(dev), mk_w((N, K), g).to(dev), mk_b((N,), g).to(dev)
        call, refkw = dict(bias=b, gelu=True), dict(bias=b, act="gelu")
    elif name == "w2v_head_f32_n_valid":          # wav2vec2.py:215: N = 1404 padded to 1408, fp32 output
        M, K, N, nv = 101, 1024, 1408, 1404
        mk_a, mk_w, mk_b, _ = _ops(K, grid)
        a, w, b = mk_a((M, K), g).to(dev), mk_w((N, K), g).to(dev), mk_b((N,), g).to(dev)
        call = dict(bias=b, n_valid=nv, out_f32=True)
        refkw = dict(bias=b, n_valid=nv, out_f32=True)
    elif name == "pose_cross_f32":                # pose_decoder.py:162: [T, 768] x [layers * 512, 768], fp32 output
        M, K, N = 150, 768, 6 * 512
        mk_a, mk_w, mk_b, _ = _ops(K, grid)
        a, w, b = mk_a((M, K), g).to(dev), mk_w((N, K), g).to(dev), mk_b((N,), g).to(dev)
        call, refkw = dict(bias=b, out_f32=True), dict(bias=b, out_f32=True)
    else:
        raise KeyError(name)
    M = a.shape[0]
    act = refkw.get("act")
    nv = refkw.get("n_valid") or (w.shape[0] // 2 if act == "geglu" else w.shape[0])
    dtype = torch.float32 if refkw.get("out_f32") else torch.float16
    out = GR.Guarded(M, nv, nv, dtype, dev)
    return a, w, call, out, dict(refkw, exact=grid)


CALLER_GEMMS = ["shortcut_1x1_two_source", "vae_wv_xt", "vae_scores_n_valid", "vae_pv_k4096", "clip_fc1_quick_gelu",
                "clip_proj_strided_cls", "w2v_conv1d_s2_gelu", "w2v_ffn_gelu", "w2v_head_f32_n_valid",
                "pose_cross_f32"]
_NONLINEAR = {"clip_fc1_quick_gelu", "w2v_conv1d_s2_gelu", "w2v_ffn_gelu"}


@pytest.mark.parametrize("name", CALLER_GEMMS)
def test_caller_gemm(cuda_dev, name):
    for grid in ((False,) if name in _NONLINEAR else (True, False)):
        a, w, call, out, refkw = _caller_gemm(name, cuda_dev, grid)
        _run_gemm(name, a, w, call, out, refkw, grid)


# ---------------------------------------------------------------------------------------------------- convs
def conv_case(name, nf, h, w, c1, c2, cout, stride=1, bias="row", frames=0, res=False, bn=0, res_off=0):
    """bias 'temb': a [B, 3 Cout_p] table sliced at column Cout_p, bias_group_rows = frames * Ho * Wo (the time
    embedding of blocks.py:189-190). res_off: the residual's base sits res_off elements past the 16-byte grid."""
    return dict(name=name, nf=nf, h=h, w=w, c1=c1, c2=c2, cout=cout, stride=stride, bias=bias, frames=frames, res=res,
                bn=bn, res_off=res_off)


CONV_CASES = [
    # UNet resnet conv1 with the time-embedding table slice, B = 2 windows of F = 3 frames (blocks.py:189-190)
    conv_case("resnet_64_temb", 6, 64, 64, 320, 0, 320, bias="temb", frames=3),
    conv_case("resnet_32_temb", 6, 32, 32, 640, 0, 640, bias="temb", frames=3),
    conv_case("resnet_16_temb", 6, 16, 16, 1280, 0, 1280, bias="temb", frames=3),
    conv_case("resnet_8_temb", 6, 8, 8, 1280, 0, 1280, bias="temb", frames=3),
    conv_case("resnet_conv2_residual", 3, 32, 32, 640, 0, 640, res=True),              # blocks.py:203
    # up-block resnets: GroupNorm'd [hidden | skip] as two conv sources (blocks.py:185-203)
    conv_case("up_640_320", 2, 32, 32, 640, 320, 640, res=True),
    conv_case("up_1280_640", 2, 16, 16, 1280, 640, 1280),
    conv_case("up_1280_1280", 2, 8, 8, 1280, 1280, 1280),
    # stride 2: downsample (blocks.py:219), two sources with C1 != C2 and C1 == C2, odd Ho / Wo
    conv_case("down_s2_320", 2, 64, 64, 320, 0, 320, stride=2),
    conv_case("down_s2_640", 3, 32, 32, 640, 0, 640, stride=2),
    conv_case("s2_two_source_64_128", 2, 16, 16, 64, 128, 128, stride=2),
    conv_case("s2_two_source_320_640", 2, 16, 16, 320, 640, 320, stride=2),
    conv_case("s2_two_source_128_64_odd", 3, 10, 14, 128, 64, 64, stride=2),
    conv_case("s2_two_source_128_128", 2, 16, 16, 128, 128, 128, stride=2),
    conv_case("s2_odd_ho", 3, 10, 14, 128, 0, 64, stride=2),
    # conv_in (unet_3d.py:255; 4 latent channels padded to 64) and conv_out to 4 channels (unet_3d.py:274; n_valid = 4:
    # the direct epilogue)
    conv_case("conv_in", 2, 64, 64, 64, 0, 320),
    conv_case("conv_out_4", 2, 64, 64, 320, 0, 4),
    # grids that are not powers of two; frames that do not divide the 128-row box
    conv_case("w48", 3, 24, 48, 64, 0, 64),
    conv_case("w40", 5, 20, 40, 128, 0, 96),
    conv_case("w6", 7, 6, 6, 64, 64, 64),
    conv_case("w5", 3, 5, 5, 64, 0, 64, res=True),
    # the residual off the 16-byte grid: direct-store epilogue, scalar residual loads
    conv_case("residual_unaligned", 2, 16, 16, 128, 0, 128, res=True, res_off=1),
    conv_case("bn32", 2, 16, 16, 128, 0, 128, bn=32, res=True),
]


def _build_conv(case, dev, grid, seed=21):
    from aniportrait_b200 import ops
    c = case
    g = _gen(seed)
    K = 9 * (c["c1"] + c["c2"])
    mk_a, mk_w, mk_b, mk_r = _ops(K, grid)
    x = mk_a((c["nf"], c["h"], c["w"], c["c1"]), g).to(dev)
    x2 = mk_a((c["nf"], c["h"], c["w"], c["c2"]), g).to(dev) if c["c2"] else None
    wp = ops.pack_conv3x3_weight(mk_w((c["cout"], c["c1"] + c["c2"], 3, 3), g)).to(dev)
    cp = wp.shape[0]
    ho, wo = c["h"] // c["stride"], c["w"] // c["stride"]
    M = c["nf"] * ho * wo
    bias, gr = None, 0
    if c["bias"] == "row":
        bias = mk_b((cp,), g).to(dev)
    elif c["bias"] == "temb":
        gr = c["frames"] * ho * wo
        bias = mk_b((c["nf"] // c["frames"], 3 * cp), g).to(dev)[:, cp:2 * cp]
    res = None
    if c["res"]:
        r = mk_r((M * c["cout"],), g)
        flat = torch.zeros(M * c["cout"] + 8, dtype=torch.float16)
        flat[c["res_off"]:c["res_off"] + r.numel()] = r
        res = flat.to(dev)[c["res_off"]:c["res_off"] + r.numel()].view(c["nf"], ho, wo, c["cout"])
    out = GR.Guarded(M, c["cout"], c["cout"], torch.float16, dev)
    call = dict(bias=bias, residual=res, x2=x2, stride=c["stride"], bias_group_rows=gr, block_n=c["bn"],
                out=out.view.view(c["nf"], ho, wo, c["cout"]))
    return x, wp, call, out


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c["name"])
def test_conv_case(cuda_dev, case):
    from aniportrait_b200 import ops
    for grid in (True, False):
        x, wp, call, out = _build_conv(case, cuda_dev, grid)
        snap = _snapshot(x, wp, call["x2"], call["bias"], call["residual"])
        _twice(lambda: ops.conv3x3(x, wp, case["cout"], **call), out, case["name"])
        _unchanged(snap, case["name"])
        ref = GR.conv_ref(x, wp, case["cout"], x2=call["x2"], stride=case["stride"], bias=call["bias"],
                          bias_group_rows=call["bias_group_rows"], residual=call["residual"], exact=grid)
        ratio = GR.check_both(out.view, ref, f"{case['name']} ({'exact grid' if grid else 'gaussian'})")
        _report(f"conv s{case['stride']}", f"{case['name']} {'grid' if grid else 'gauss'}", ratio)


# ---------------------------------------------------------------------------------------------------- statistics
def _stats_operands(dev, M, N, K, seed):
    g = _gen(seed)
    mk_a, mk_w, mk_b, mk_r = GR.gauss_operands(K)
    return (mk_a((M, K), g).to(dev), mk_w((N, K), g).to(dev), mk_b((N,), g).to(dev),
            (mk_r((M, N), g) + 0.5).to(dev))


@pytest.mark.parametrize("M", [31, 129, 4101])
@pytest.mark.parametrize("bn", [32, 64, 160])
def test_row_stats(cuda_dev, M, bn):
    """Row partials of the epilogue == fp64 sums of the stored fp16 output per (part, row), incl. M tails and BN = 32
    (whose odd column half has no chunk and writes zeros)."""
    from aniportrait_b200 import ops
    N, K = 320, 320
    a, w, b, r = _stats_operands(cuda_dev, M, N, K, 31 + bn)
    out = GR.Guarded(M, N, N, torch.float16, cuda_dev)
    res = {}

    def call():
        res["rs"] = ops.gemm(a, w, bias=b, residual=r, out=out.view, block_n=bn, row_stats=True)[1]
        res.setdefault("first", res["rs"].buf[:, :M].clone())
    _twice(call, out, f"row stats M={M} bn={bn}")
    rs = res["rs"]
    assert torch.equal(res["first"], rs.buf[:, :M]), "row partials differ between two calls"
    GR.check_both(out.view, GR.gemm_ref(a, w, bias=b, residual=r, bn=bn), "row stats output")
    want, bnd = GR.row_stats_ref(out.view, bn, rs.parts)
    ratio = GR.check_stats(rs.buf[:, :M], want, bnd, f"row stats M={M} bn={bn}")
    _report("statistics", f"row M={M} bn={bn}", ratio)


@pytest.mark.parametrize("M", [33, 129, 4101])
@pytest.mark.parametrize("bn", [32, 128])
def test_gemm_col_stats(cuda_dev, M, bn):
    from aniportrait_b200 import ops
    N, K = 384, 256
    a, w, b, r = _stats_operands(cuda_dev, M, N, K, 41 + bn)
    out = GR.Guarded(M, N, N, torch.float16, cuda_dev)
    res = {}

    def call():
        res["cs"] = ops.gemm(a, w, bias=b, residual=r, out=out.view, block_n=bn, col_stats=True)[1]
        res.setdefault("first", res["cs"].buf.clone())
    _twice(call, out, "col stats")
    cs = res["cs"]
    assert torch.equal(res["first"], cs.buf), "column partials differ between two calls"
    want, bnd = GR.col_stats_ref(out.view, GR.gemm_box_rows(M, (M + 127) // 128, cuda_dev))
    ratio = GR.check_stats(cs.buf[:want.shape[0]], want, bnd, f"col stats M={M} bn={bn}")
    _report("statistics", f"col M={M} bn={bn}", ratio)


def test_ff2_residual_col_stats(cuda_dev):
    """FeedForward's second GEMM (blocks.py:127): K = 1280 -> 320 with the residual and column statistics."""
    from aniportrait_b200 import ops
    M, N, K = 2048, 320, 1280
    a, w, b, r = _stats_operands(cuda_dev, M, N, K, 51)
    out = GR.Guarded(M, N, N, torch.float16, cuda_dev)
    res = {}

    def call():
        res["cs"] = ops.gemm(a, w, bias=b, residual=r, out=out.view, col_stats=True)[1]
        res.setdefault("first", res["cs"].buf.clone())
    _twice(call, out, "ff2")
    assert torch.equal(res["first"], res["cs"].buf), "column partials differ between two calls"
    _report("linear", "ff2 output", GR.check(out.view, GR.gemm_ref(a, w, bias=b, residual=r), "ff2"))
    want, bnd = GR.col_stats_ref(out.view, GR.gemm_box_rows(M, M // 128, cuda_dev))
    _report("statistics", "ff2 col", GR.check_stats(res["cs"].buf, want, bnd, "ff2 col stats"))


def _group_norm_twice(y, gamma, beta, what, **kw):
    """ops.group_norm into a guarded output, twice (identical bits); returns the [rows, C] output view."""
    from aniportrait_b200 import ops
    c = gamma.numel()
    rows = y.numel() // y.shape[-1]
    out = GR.Guarded(rows, c, c, torch.float16, y.device)
    _twice(lambda: ops.group_norm(y, gamma, beta, 32, 1e-5, True, out=out.view.view(*y.shape[:-1], c), **kw), out, what)
    return out.view


@pytest.mark.parametrize("mu", [0, 16])
@pytest.mark.parametrize("nf,h,w,cin,cout,stride", [
    (4, 32, 32, 320, 320, 1), (3, 16, 16, 640, 640, 1), (6, 8, 8, 1280, 1280, 1), (2, 64, 64, 320, 320, 2),
    (5, 16, 24, 128, 320, 1), (8, 4, 8, 256, 256, 1), (3, 24, 48, 64, 128, 1)])
def test_conv_col_stats_group_norm(cuda_dev, nf, h, w, cin, cout, stride, mu):
    """Conv column partials per 32-row sub-box == fp64 sums of the stored output; GroupNorm fed with them == fp64.
    mu: channel means of the conv output (sigma ~ 1), for the E[x^2] - mean^2 cancellation of the GroupNorm."""
    from aniportrait_b200 import ops
    g = _gen(61)
    mk_a, mk_w, mk_b, _ = GR.gauss_operands(9 * cin)
    x = mk_a((nf, h, w, cin), g).to(cuda_dev)
    wp = ops.pack_conv3x3_weight(mk_w((cout, cin, 3, 3), g)).to(cuda_dev)
    b = (0.2 * mk_b((cout,), g) + mu).to(cuda_dev)
    ho, wo = h // stride, w // stride
    assert ops.conv_col_stats_ok(nf, ho, wo)
    out = GR.Guarded(nf * ho * wo, cout, cout, torch.float16, cuda_dev)
    y = out.view.view(nf, ho, wo, cout)
    res = {}

    def call():
        res["cs"] = ops.conv3x3(x, wp, cout, bias=b, stride=stride, col_stats=True, out=y)[1]
        res.setdefault("first", res["cs"].buf.clone())
    _twice(call, out, "conv col stats")
    cs = res["cs"]
    assert torch.equal(res["first"], cs.buf), "conv column partials differ between two calls"
    rows = GR.conv_box_rows(nf, ho, wo, cuda_dev)
    want, bnd = GR.col_stats_ref(out.view, rows)
    ratio = GR.check_stats(cs.buf[:want.shape[0]], want, bnd, "conv col stats")
    _report("statistics", f"conv col {nf}x{ho}x{wo}x{cout} mu={mu}", ratio)
    gamma = torch.randn(cout, generator=g).to(cuda_dev)
    beta = torch.randn(cout, generator=g).to(cuda_dev)
    fused = _group_norm_twice(y, gamma, beta, "group norm", stats=cs)
    ref = GR.group_norm_ref(y.view(nf, ho * wo, cout), gamma, beta, 32, 1e-5, True)
    _report(f"group norm mu/sigma={mu}", f"conv {nf}x{ho}x{wo}x{cout}", GR.check(fused, ref, "group norm"))


@pytest.mark.parametrize("mu", [0, 1, 4, 16, 64])
def test_up_block_two_source_group_norm(cuda_dev, mu):
    """GroupNorm over [GEMM output with residual | conv output], each with its own column statistics; groups straddle
    the two sources (C = 640 + 320, 30 channels per group). mu: the mean of both sources (sigma ~ 1)."""
    from aniportrait_b200 import ops
    nf, h, w = 4, 16, 16
    g = _gen(71)
    a = torch.randn(nf * h * w, 640, generator=g).half().to(cuda_dev)
    w1 = (torch.randn(640, 640, generator=g) * 640 ** -0.5).half().to(cuda_dev)
    r1 = (0.5 * torch.randn(nf * h * w, 640, generator=g) + mu).half().to(cuda_dev)
    xin = torch.randn(nf, h, w, 320, generator=g).half().to(cuda_dev)
    wc = ops.pack_conv3x3_weight((torch.randn(320, 320, 3, 3, generator=g) * (9 * 320) ** -0.5).half()).to(cuda_dev)
    bc = torch.full((320,), float(mu)).to(cuda_dev)
    o1 = GR.Guarded(nf * h * w, 640, 640, torch.float16, cuda_dev)
    o2 = GR.Guarded(nf * h * w, 320, 320, torch.float16, cuda_dev)
    st = {}

    def gemm_call():
        st["cs1"] = ops.gemm(a, w1, residual=r1, col_stats=True, out=o1.view)[1]
        st.setdefault("first1", st["cs1"].buf.clone())

    def conv_call():
        st["cs2"] = ops.conv3x3(xin, wc, 320, bias=bc, col_stats=True, out=o2.view.view(nf, h, w, 320))[1]
        st.setdefault("first2", st["cs2"].buf.clone())
    _twice(gemm_call, o1, "up-block gemm")
    _twice(conv_call, o2, "up-block conv")
    assert torch.equal(st["first1"], st["cs1"].buf) and torch.equal(st["first2"], st["cs2"].buf)
    gamma = torch.randn(960, generator=g).to(cuda_dev)
    beta = torch.randn(960, generator=g).to(cuda_dev)
    x1, x2 = o1.view.view(nf, h, w, 640), o2.view.view(nf, h, w, 320)
    fused = _group_norm_twice(x1, gamma, beta, "two-source group norm", x2=x2, stats=st["cs1"], stats2=st["cs2"])
    cat = torch.cat([o1.view.view(nf, h * w, 640), o2.view.view(nf, h * w, 320)], -1)
    ref = GR.group_norm_ref(cat, gamma, beta, 32, 1e-5, True)
    _report(f"group norm mu/sigma={mu}", "up-block two-source", GR.check(fused, ref, "two-source group norm"))


# ---------------------------------------------------------------------------------------------------- LayerNorm fold
def _ln_producer(dev, M, C, mu_over_sigma, seed):
    """x = a @ w0 + r with rows of mean +-mu_over_sigma and sigma ~ 1, produced with row statistics."""
    from aniportrait_b200 import ops
    g = _gen(seed)
    a = torch.randn(M, C, generator=g).half().to(dev)
    w0 = (torch.randn(C, C, generator=g) * C ** -0.5).half().to(dev)
    r = (mu_over_sigma * torch.randn(M, 1, generator=g).sign().expand(M, C)).half().contiguous().to(dev)
    x, rs = ops.gemm(a, w0, residual=r, row_stats=True)
    torch.cuda.synchronize()
    bn = C // (rs.parts // 2)
    want, bnd = GR.row_stats_ref(x, bn, rs.parts)
    _report("statistics", f"LN producer mean/sigma={mu_over_sigma}", GR.check_stats(rs.buf[:, :M], want, bnd, "rows"))
    return x, rs, g


@pytest.mark.parametrize("mu_over_sigma", [0, 1, 4, 16, 64])
@pytest.mark.parametrize("layout", ["qkv_head_padded", "geglu", "temporal_qkv_pe"])
def test_ln_fold(cuda_dev, layout, mu_over_sigma):
    """The LayerNorm folded into its consumer against fp64 LayerNorm + the original fp32 linear layer:
    qkv_head_padded  blocks.py:351 (heads of d = 40 padded to 64 rows, no bias)
    geglu            blocks.py:123 (FeedForward's GEGLU projection, C = 320 -> 2 x 1280)
    temporal_qkv_pe  blocks.py:555 (a per-frame positional-encoding bias table, bias_group_rows = tokens)"""
    from aniportrait_b200 import ops
    from aniportrait_b200.models.blocks import fold_layer_norm
    C, eps = 320, 1e-5
    M = 2 * 3 * 96 if layout == "temporal_qkv_pe" else 1000
    x, rs, g = _ln_producer(cuda_dev, M, C, mu_over_sigma, 81)
    gamma = (1.0 + 0.2 * torch.randn(C, generator=g)).to(cuda_dev)
    beta = (0.1 * torch.randn(C, generator=g)).to(cuda_dev)
    gr, act = 0, None
    if layout == "qkv_head_padded":
        heads, d = 8, 40
        dpad = ops.head_pad(d)
        w = torch.zeros(3, heads, dpad, C)
        w[:, :, :d] = torch.randn(3, heads, d, C, generator=g) * C ** -0.5
        w = w.reshape(3 * heads * dpad, C).to(cuda_dev)
        b = None
        wg, bias = fold_layer_norm(w, b, gamma, beta)
    elif layout == "geglu":
        w = (torch.randn(8 * C, C, generator=g) * C ** -0.5).to(cuda_dev)
        b = (0.1 * torch.randn(8 * C, generator=g)).to(cuda_dev)
        wg, bias = ops.interleave_geglu(*fold_layer_norm(w, b, gamma, beta))
        w, b = ops.interleave_geglu(w, b)
        act = "geglu"
    else:
        frames, tokens = 6, 96
        w = (torch.randn(3 * C, C, generator=g) * C ** -0.5).to(cuda_dev)
        b = (0.5 * torch.randn(frames, 3 * C, generator=g)).to(cuda_dev)            # per-frame PE @ W^T
        wg, fb = fold_layer_norm(w, None, gamma, beta)
        bias = (fb[None, :] + b).contiguous()
        gr = tokens
    out = GR.Guarded(M, wg.shape[0] // (2 if act else 1), wg.shape[0] // (2 if act else 1), torch.float16, cuda_dev)
    _twice(lambda: ops.gemm(x, wg, bias=bias, geglu=act == "geglu", bias_group_rows=gr, out=out.view,
                            ln=ops.LNFold(rs, eps)), out, layout)
    ref = GR.ln_fold_ref(x, w, b, gamma, beta, eps, wg, act=act, bias_group_rows=gr)
    ratio = GR.check(out.view, ref, f"LN fold {layout} mean/sigma={mu_over_sigma}")
    _report(f"LN fold mean/sigma={mu_over_sigma}", layout, ratio)


# ---------------------------------------------------------------------------------------------------- switches
@pytest.mark.parametrize("env,select", [
    ({"AP_GEMM_NO_TMA_EPI": "1"}, "test_gemm_variant or test_conv_case"),
    ({"AP_GEMM_EPI_DOUBLE": "0"}, "test_gemm_variant or test_conv_case"),
    ({"AP_PDL": "1"}, "test_ln_fold or test_conv_col_stats_group_norm or test_up_block"),
], ids=["no_tma_epilogue", "single_buffered_staging", "pdl"])
def test_switches_in_child_process(env, select):
    """The switches are read once per process: re-run a subset in a child pytest with each one set."""
    if os.environ.get(CHILD):
        pytest.skip("already running under a switch")
    full = dict(os.environ, **env, **{CHILD: "1"})
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__),
           "-k", f"({select}) and not switches"]
    r = subprocess.run(cmd, env=full, cwd=root, timeout=900, capture_output=True, text=True)
    tail = (r.stdout + r.stderr)[-4000:]
    print(f"\n[switch {env}] {tail.strip().splitlines()[-1] if tail.strip() else ''}")
    assert r.returncode == 0, tail


# ---------------------------------------------------------------------------------------------------- refusals
def _refusals(dev):
    from aniportrait_b200 import ops
    M, N, K = 129, 320, 320
    g = _gen(91)
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
    wgeglu = (torch.randn(2 * N, K, generator=g) * K ** -0.5).half().to(dev)
    r = torch.randn(M, N, generator=g).half().to(dev)
    flat = torch.randn(N + 8, generator=g).to(dev)
    table = torch.randn(2, N + 2, generator=g).to(dev)
    x = torch.randn(2, 6, 6, 64, generator=g).half().to(dev)
    wc = ops.pack_conv3x3_weight((torch.randn(64, 64, 3, 3, generator=g) * 0.05).half()).to(dev)
    f16 = lambda cols=N: GR.Guarded(M, cols, cols, torch.float16, dev)  # noqa: E731
    return {
        "bias_unaligned": (f16(), lambda o: ops.gemm(a, w, bias=flat[1:1 + N], out=o)),
        "bias_ld_not_multiple_of_4": (f16(), lambda o: ops.gemm(a, w, bias=table[:, :N], bias_group_rows=64, out=o)),
        "conv_bias_unaligned": (GR.Guarded(72, 64, 64, torch.float16, dev),
                                lambda o: ops.conv3x3(x, wc, 64, bias=flat[1:1 + 64], out=o.view(2, 6, 6, 64))),
        "row_stats_n_valid": (f16(288), lambda o: ops.gemm(a, w, n_valid=288, out=o, row_stats=True)),
        "col_stats_n_valid": (f16(288), lambda o: ops.gemm(a, w, n_valid=288, out=o, col_stats=True)),
        "geglu_bn32": (f16(), lambda o: ops.gemm(a, wgeglu, geglu=True, block_n=32, out=o)),
        "geglu_bn160": (f16(), lambda o: ops.gemm(a, wgeglu, geglu=True, block_n=160, out=o)),
        "geglu_f32": (GR.Guarded(M, N, N, torch.float32, dev),
                      lambda o: ops.gemm(a, wgeglu, geglu=True, out_f32=True, out=o)),
        "gelu_residual": (f16(), lambda o: ops.gemm(a, w, residual=r, gelu=True, out=o)),
        "gelu_and_quick_gelu": (f16(), lambda o: ops.gemm(a, w, gelu=True, quick_gelu=True, out=o)),
        "unsupported_bn": (f16(), lambda o: ops.gemm(a, w, block_n=96, out=o)),
        "conv_col_stats_geometry": (GR.Guarded(72, 64, 64, torch.float16, dev),
                                    lambda o: ops.conv3x3(x, wc, 64, out=o.view(2, 6, 6, 64), col_stats=True)),
    }


REFUSALS = ["bias_unaligned", "bias_ld_not_multiple_of_4", "conv_bias_unaligned", "row_stats_n_valid",
            "col_stats_n_valid", "geglu_bn32", "geglu_bn160", "geglu_f32", "gelu_residual", "gelu_and_quick_gelu",
            "unsupported_bn", "conv_col_stats_geometry"]


@pytest.mark.parametrize("name", REFUSALS)
def test_refusal(cuda_dev, name):
    """Refused with AP_ERR_INVALID before any launch: the output's sentinels stay intact."""
    from aniportrait_b200._lib import ApError
    out, call = _refusals(cuda_dev)[name]
    torch.cuda.synchronize()
    with pytest.raises(ApError, match=r"rc=-1\)"):
        call(out.view)
    torch.cuda.synchronize()
    out.check(name)
    assert bool((out.bits == out.sentinel).all()), f"{name}: the output was written"
