"""The normalisation / small-convolution / elementwise checker itself, without a GPU (norm_reference.py): every fp32
emulation passes its bounded check on the GPU case table at reduced sizes, with its unrounded values within half of the
derived pre-rounding bound; every modelled bug is rejected with a message that names the element; every fp64 reference
matches torch's own fp64 operator."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_reference as GR
import norm_reference as NR
from aniportrait_b200 import ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rejected(fn) -> str:
    try:
        fn()
    except AssertionError as e:
        return str(e).splitlines()[0][:200]
    return ""


def _within(out, ref, y32, what):
    ratio = GR.check(out, ref, what)
    head = GR.headroom(y32, ref)
    print(f"\n[emulation] {what}: worst error / bound = {ratio:.3f}, unrounded / pre-rounding bound = {head:.3f}")
    assert head <= 0.5, f"{what}: headroom {head:.3f}"


# ------------------------------------------------------------------------------------------------------ GroupNorm
# (Nf, HW, C1, C2, groups, eps, silu, mean, max_blocks): the GPU table at reduced HW / Nf. A small max_blocks makes the
# reduced shapes reach the rows-per-block doubling loop of gn_launch_geometry, as the VAE and many-frame cases do.
GN_CPU = [
    (2, 256, 320, 0, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS),
    (2, 64, 1280, 0, 32, 1e-5, False, 0.0, NR.GN_MAX_BLOCKS),
    (2, 64, 640, 320, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS),       # 30 channels per group: group 21 straddles
    (2, 64, 1280, 640, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS),
    (2, 1000, 320, 0, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS),       # HW not a multiple of rows per block
    (2, 4096, 128, 0, 32, 1e-6, True, 0.0, 40),                      # rows per block doubled
    (40, 64, 320, 0, 32, 1e-5, True, 0.0, 40),                       # rows per block reaches HW
    *[(2, 256, 320, 0, 32, 1e-5, True, float(m), NR.GN_MAX_BLOCKS) for m in (1, 4, 16, 64)],
]


def _gn_operands(nf, hw, c1, c2, mean, seed=1):
    g = _gen(seed)
    x = (torch.randn(nf, hw, c1, generator=g) + mean).half()
    x2 = (torch.randn(nf, hw, c2, generator=g) + mean).half() if c2 else None
    gamma = 1 + 0.2 * torch.randn(c1 + c2, generator=g)
    beta = 0.1 * torch.randn(c1 + c2, generator=g)
    return x, x2, gamma, beta


@pytest.mark.parametrize("nf,hw,c1,c2,groups,eps,silu,mean,mb", GN_CPU)
def test_gn_emulation_within_bound(nf, hw, c1, c2, groups, eps, silu, mean, mb):
    x, x2, gamma, beta = _gn_operands(nf, hw, c1, c2, mean)
    ref = NR.gn_ref(x, x2, gamma, beta, groups, eps, silu, max_blocks=mb)
    out = NR.emulate_gn(x, x2, gamma, beta, groups, eps, silu, max_blocks=mb)
    y32 = NR.emulate_gn(x, x2, gamma, beta, groups, eps, silu, max_blocks=mb, unrounded=True)
    _within(out, ref, y32, f"GN {nf}x{hw}x{c1}+{c2} mean={mean} max_blocks={mb}")


def test_gn_geometry_reaches_doubling_and_refusal():
    """The restated gn_launch_geometry at the GPU shapes: the VAE's 512x512 level doubles rows per block, 1200 frames of
    64 rows need rows per block >= HW, and 2400 such frames are refused."""
    assert NR.gn_geometry(512 * 512, 128, 2) == (16, 256, 1024)
    k, rpb, chunks = NR.gn_geometry(64, 320, 1200)
    assert rpb >= 64 and chunks == 1
    assert NR.gn_refused(64, (320,), 2400) and not NR.gn_refused(64, (320,), 1200)


@pytest.mark.parametrize("bug,case", [
    ("drop_last_chunk", (2, 1000, 320, 0, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS)),
    ("drop_last_chunk", (2, 4096, 128, 0, 32, 1e-6, True, 0.0, 40)),
    ("straddle_one_source", (2, 64, 640, 320, 32, 1e-5, True, 0.0, NR.GN_MAX_BLOCKS)),
])
def test_gn_bug_rejected(bug, case):
    nf, hw, c1, c2, groups, eps, silu, mean, mb = case
    x, x2, gamma, beta = _gn_operands(nf, hw, c1, c2, mean)
    out = NR.emulate_gn(x, x2, gamma, beta, groups, eps, silu, bug=bug, max_blocks=mb)
    msg = _rejected(lambda: GR.check(out, NR.gn_ref(x, x2, gamma, beta, groups, eps, silu, max_blocks=mb), bug))
    print(f"\n[bug {bug}] {msg}")
    assert "element" in msg and "group" in msg


def test_gn_reference_matches_torch():
    x, x2, gamma, beta = _gn_operands(2, 48, 64, 32, 2.0)
    ref = NR.gn_ref(x, x2, gamma, beta, 16, 1e-6, True)
    cat = torch.cat([x, x2], -1).double().permute(0, 2, 1)
    want = F.silu(F.group_norm(cat, 16, gamma.double(), beta.double(), 1e-6)).permute(0, 2, 1).reshape(-1, 96)
    assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ LayerNorm
# (rows, C, narrow, pe_period, mean): every caller width at reduced rows, the 1536 boundary, the narrow widths.
LN_CPU = [(r, c, False, 0, 0.0) for r, c in ((77, 320), (77, 640), (77, 1280), (45, 512), (45, 768), (40, 1024),
                                             (21, 1536))]
LN_CPU += [(37, c, False, 0, 0.0) for c in (1544, 2048, 322)]
LN_CPU += [(37, c, True, 0, 0.0) for c in (320, 768, 1280)]
LN_CPU += [(2 * 4 * 16, 320, False, 4, 0.0), (2 * 16 * 4, 640, True, 16, 0.0)]
LN_CPU += [(64, 320, False, 0, m) for m in (16.0, 64.0)]


def _ln_operands(rows, C, pe_period, mean, seed=2):
    g = _gen(seed)
    x = (torch.randn(rows, C, generator=g) + mean * torch.randn(rows, 1, generator=g).sign()).half()
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    pe = torch.randn(pe_period, C, generator=g) if pe_period else None
    return x, gamma, beta, pe


def _ln_rows_per_pe(rows, pe_period):
    return rows // (2 * pe_period) if pe_period else 1          # B = 2 windows of pe_period frames


@pytest.mark.parametrize("rows,C,narrow,pe_period,mean", LN_CPU)
def test_ln_emulation_within_bound(rows, C, narrow, pe_period, mean):
    x, gamma, beta, pe = _ln_operands(rows, C, pe_period, mean)
    rpp = _ln_rows_per_pe(rows, pe_period)
    kw = dict(pe=pe, rows_per_pe=rpp, pe_period=max(pe_period, 1), narrow=narrow)
    ref = NR.ln_ref(x, gamma, beta, 1e-5, **kw)
    out = NR.emulate_ln(x, gamma, beta, 1e-5, **kw)
    y32 = NR.emulate_ln(x, gamma, beta, 1e-5, unrounded=True, **kw)
    _within(out, ref, y32, f"LN {rows}x{C} {NR.ln_kernel(C, narrow)} pe={pe_period} mean={mean}")


@pytest.mark.parametrize("C,narrow", [(320, False), (768, False), (322, False), (1280, True)])
def test_ln_constant_rows_exact(C, narrow):
    g = _gen(4)
    rows, period = 2 * 4 * 8, 4
    x = torch.randn(rows, 1, generator=g).mul(8).half().expand(rows, C).contiguous()
    gamma, beta, pe = torch.randn(C, generator=g), torch.randn(C, generator=g), torch.randn(period, C, generator=g)
    kw = dict(pe=pe, rows_per_pe=8, pe_period=period)
    out = NR.emulate_ln(x, gamma, beta, 1e-5, narrow=narrow, **kw)
    assert torch.equal(out, NR.ln_constant_rows(gamma, beta, rows=rows, **kw))


@pytest.mark.parametrize("bug,rows,C,narrow,pe_period", [
    ("pe_row", 2 * 4 * 16, 320, False, 4), ("pe_row", 2 * 16 * 4, 640, True, 16),
    ("last_vec", 37, 1280, False, 0), ("last_vec", 37, 1544, False, 0), ("last_vec", 37, 768, True, 0),
])
def test_ln_bug_rejected(bug, rows, C, narrow, pe_period):
    x, gamma, beta, pe = _ln_operands(rows, C, pe_period, 0.0)
    kw = dict(pe=pe, rows_per_pe=_ln_rows_per_pe(rows, pe_period), pe_period=max(pe_period, 1), narrow=narrow)
    out = GR.Guarded(rows, C, C, torch.float16, torch.device("cpu"))
    NR.emulate_ln(x, gamma, beta, 1e-5, bug=bug, out=out.view, **kw)
    msg = _rejected(lambda: GR.check(out.view, NR.ln_ref(x, gamma, beta, 1e-5, **kw), bug))
    print(f"\n[bug {bug} C={C}] {msg}")
    assert "element" in msg and "row" in msg


def test_ln_reference_matches_torch():
    x, gamma, beta, _ = _ln_operands(33, 322, 0, 3.0)
    ref = NR.ln_ref(x, gamma, beta, 1e-5)
    want = F.layer_norm(x.double(), (322,), gamma.double(), beta.double(), 1e-5)
    assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ BatchNorm
BN_CPU = [(2 * 64 * 64, 8, "relu", 0.0), (2 * 64 * 64, 16, "relu", 0.0), (4096, 64, "relu", 4.0),
          (1024, 320, "relu", 0.0), (256, 1280, "none", 0.0), (3999, 512, "gelu", 0.0), (64, 64, "relu", 0.0),
          *[(2048, 64, "relu", m) for m in (1.0, 16.0, 64.0)]]


def _bn_operands(rows, C, mean, seed=3, pad=0):
    g = _gen(seed)
    x = (torch.randn(rows, C, generator=g) + mean).half()
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    if pad:
        x[:, -pad:] = 0
        gamma[-pad:] = 0
        beta[-pad:] = 0
    return x, gamma, beta


@pytest.mark.parametrize("rows,C,act,mean", BN_CPU)
def test_bn_emulation_within_bound(rows, C, act, mean):
    x, gamma, beta = _bn_operands(rows, C, mean)
    ref = NR.bn_ref(x, gamma, beta, 1e-5, act)
    out = NR.emulate_bn(x, gamma, beta, 1e-5, act)
    _within(out, ref, NR.emulate_bn(x, gamma, beta, 1e-5, act, unrounded=True), f"BN {rows}x{C} {act} mean={mean}")


def test_bn_padded_channels_exactly_zero():
    x, gamma, beta = _bn_operands(1024, 16, 0.0, pad=5)
    assert bool((NR.emulate_bn(x, gamma, beta, 1e-5, "relu")[:, -5:] == 0).all())


def test_bn_geometry_partial_last_chunk():
    """31999 rows at C = 512 (wav2vec2, 10 s): rows per block 64, and a partial last chunk at 2^21 + 5 rows x 64."""
    assert NR.bn_geometry(31999, 512) == (4, 32, 1000)
    k, rpb, chunks = NR.bn_geometry(2 ** 21 + 5, 64)
    assert chunks <= NR.BN_MAX_BLOCKS and (2 ** 21 + 5) % rpb


@pytest.mark.parametrize("bug,rows,C,mb", [("unbiased", 64, 64, NR.BN_MAX_BLOCKS), ("drop_last_chunk", 1000, 64, 8),
                                            ("drop_last_chunk", 3999, 512, NR.BN_MAX_BLOCKS)])
def test_bn_bug_rejected(bug, rows, C, mb):
    x, gamma, beta = _bn_operands(rows, C, 0.0)
    out = NR.emulate_bn(x, gamma, beta, 1e-5, "relu", bug=bug, max_blocks=mb)
    msg = _rejected(lambda: GR.check(out, NR.bn_ref(x, gamma, beta, 1e-5, "relu"), bug))
    print(f"\n[bug {bug} rows={rows}] {msg}")
    assert "element" in msg and "channel" in msg


def test_bn_reference_matches_torch():
    x, gamma, beta = _bn_operands(300, 24, 1.5)
    ref = NR.bn_ref(x, gamma, beta, 1e-5, "gelu")
    want = F.batch_norm(x.double(), None, None, gamma.double(), beta.double(), training=True, eps=1e-5)
    assert torch.allclose(ref.o, F.gelu(want), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ direct conv
def _dc_operands(cin, K, cout, nf, H, W, grid, bias=True, seed=5):
    g = _gen(seed)
    n = K * K * cin
    mk_a, mk_w, mk_b, _ = GR.grid_operands(n) if grid else GR.gauss_operands(n)
    x, w = mk_a((nf, H, W, cin), g), mk_w((cout, K, K, cin), g)
    return x, w, (mk_b((cout,), g) if bias else None)


@pytest.mark.parametrize("cin,K,S,ct", NR.DIRECT_CONV_VARIANTS)
@pytest.mark.parametrize("bias", [True, False])
def test_direct_conv_emulation(cin, K, S, ct, bias):
    for grid in (True, False):
        x, w, b = _dc_operands(cin, K, 2 * ct, 2, 13, 11, grid, bias)
        ref = NR.direct_conv_ref(x, w, b, S, 1, exact=grid)
        out = NR.emulate_direct_conv(x, w, b, S, 1)
        GR.check_both(out, ref, f"direct conv {cin} K{K} S{S}")
        assert GR.headroom(NR.emulate_direct_conv(x, w, b, S, 1, unrounded=True), ref) <= 0.5


@pytest.mark.parametrize("bug", ["flip_tap", "pad_off"])
@pytest.mark.parametrize("cin,K,S", [(8, 3, 1), (32, 4, 2)])
def test_direct_conv_bug_rejected(bug, cin, K, S):
    for grid in (True, False):
        x, w, b = _dc_operands(cin, K, 16, 2, 12, 9, grid)
        out = NR.emulate_direct_conv(x, w, b, S, 1, bug=bug)
        msg = _rejected(lambda: GR.check_both(out, NR.direct_conv_ref(x, w, b, S, 1, exact=grid), bug))
        print(f"\n[bug {bug} K{K} S{S} grid={grid}] {msg}")
        assert "element" in msg and "frame" in msg


@pytest.mark.parametrize("cin,K,S,ct", NR.DIRECT_CONV_VARIANTS)
def test_direct_conv_reference_matches_torch(cin, K, S, ct):
    x, w, b = _dc_operands(cin, K, 16, 2, 9, 7, False)
    ref = NR.direct_conv_ref(x, w, b, S, 1)
    want = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), b.double(), stride=S, padding=1)
    assert torch.allclose(ref.o, want.permute(0, 2, 3, 1).reshape(-1, 16), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ audio
@pytest.mark.parametrize("samples", [10, 11, 14, 15, 90, 4001])
def test_stem_emulation(samples):
    g = _gen(6)
    wave, w = torch.randn(samples, generator=g), torch.randn(64, 10, generator=g) * 0.3
    ref = NR.stem_ref(wave, w)
    _within(NR.emulate_stem(wave, w), ref, NR.emulate_stem(wave, w, unrounded=True), f"stem {samples}")
    want = F.conv1d(wave.double()[None, None], w.double()[:, None], stride=5)[0].t()
    assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12)
    wg = (torch.randint(-32, 33, (64, 10), generator=g) / 32.0)
    xg = (torch.randint(-4, 5, (samples,), generator=g) / 4.0)
    GR.check_exact(NR.emulate_stem(xg, wg), NR.stem_ref(xg, wg, exact=True), "stem exact grid")


def _pos_operands(T, seed=7, K=128):
    g = _gen(seed)
    x = torch.randn(T, 768, generator=g).half()
    w = (torch.randn(768, 48, K, generator=g) * (48 * K) ** -0.5)
    return x, ops.pack_pos_conv_weight(w), torch.randn(768, generator=g) * 0.5


@pytest.mark.parametrize("T", [1, 33, 65])
def test_pos_conv_emulation(T):
    x, wp, b = _pos_operands(T)
    ref = NR.pos_conv_ref(x, wp, b)
    _within(NR.emulate_pos_conv(x, wp, b), ref, NR.emulate_pos_conv(x, wp, b, unrounded=True), f"pos conv T={T}")


@pytest.mark.parametrize("bug", ["trim_side", "group_offset"])
def test_pos_conv_bug_rejected(bug):
    x, wp, b = _pos_operands(40)
    msg = _rejected(lambda: GR.check(NR.emulate_pos_conv(x, wp, b, bug=bug), NR.pos_conv_ref(x, wp, b), bug))
    print(f"\n[bug {bug}] {msg}")
    assert "element" in msg and "group" in msg


def test_pos_conv_reference_matches_torch():
    K, T = 16, 21
    x, wp, b = _pos_operands(T, K=K)
    ref = NR.pos_conv_ref(x, wp, b)
    w = wp.double().permute(0, 2, 1)                                   # [C, 48, K]
    conv = F.conv1d(x.double().t()[None], w, b.double(), padding=K // 2, groups=16)[0, :, :-1].t()
    assert torch.allclose(ref.o, x.double() + F.gelu(conv), rtol=1e-12, atol=1e-12)


RESAMPLE_CPU = [(68, 42), (249, 150), (268, 162), (499, 300), (42, 68), (7, 1), (1, 9), (5, 5), (3, 200)]


@pytest.mark.parametrize("t_in,t_out", RESAMPLE_CPU)
def test_resample_emulation(t_in, t_out):
    """The kernel's fp32 formula is within bound, and its fp64 reference is F.interpolate(linear, align_corners=True).
    torch's own fp32 interpolation is NOT the kernel's formula bit for bit (it differs in the last fp32 bit on a few
    percent of the values), so the GPU contract asserts bit-identity with this emulation, not with torch."""
    x = torch.randn(t_in, 64, generator=_gen(8)).half()
    ref = NR.resample_ref(x, t_out)
    out = NR.emulate_resample(x, t_out)
    _within(out, ref, NR.emulate_resample(x, t_out, unrounded=True), f"resample {t_in}->{t_out}")
    want64 = F.interpolate(x.double().t()[None], size=t_out, mode="linear", align_corners=True)[0].t()
    assert torch.allclose(ref.o, want64, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("t_in,t_out", [(68, 42), (42, 68)])
def test_resample_align_corners_false_rejected(t_in, t_out):
    x = torch.randn(t_in, 64, generator=_gen(8)).half()
    msg = _rejected(lambda: GR.check(NR.emulate_resample(x, t_out, bug="align_false"), NR.resample_ref(x, t_out), "ac"))
    print(f"\n[bug align_false {t_in}->{t_out}] {msg}")
    assert "element" in msg and "i0" in msg


# ------------------------------------------------------------------------------------------------------ small kernels
def test_timestep_emulation_and_swap():
    t = torch.tensor([0.0, 1.0, 999.0, 981.0, 501.0])
    ref = NR.timestep_ref(t, 320)
    _within(NR.emulate_timestep(t, 320), ref, NR.emulate_timestep(t, 320, unrounded=True), "timestep embedding")
    msg = _rejected(lambda: GR.check(NR.emulate_timestep(t, 320, bug="swap"), ref, "swap"))
    print(f"\n[bug swap] {msg}")
    assert "element" in msg and "freq" in msg
    half = 160
    w = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64) / half)
    want = torch.cat([torch.cos(t.double()[:, None] * w), torch.sin(t.double()[:, None] * w)], 1)
    assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12)


def test_silu_emulation_every_finite_value():
    x = NR.all_finite_f16()
    assert x.numel() == 63488
    ref = NR.silu_ref(x)
    _within(NR.emulate_silu(x), ref, NR.emulate_silu(x, unrounded=True), "silu")
    assert torch.allclose(ref.o[:, 0], F.silu(x.double()), rtol=1e-12, atol=1e-300)


def test_add_bcast_interleave_rejected():
    g = _gen(9)
    a, b = torch.randn(2 * 6, 40, generator=g).half(), torch.randn(6, 40, generator=g).half()
    assert torch.equal(NR.emulate_add_bcast(a, b, 2), NR.add_ref(a.float(), b.float(), 2).half())
    assert not torch.equal(NR.emulate_add_bcast(a, b, 2, bug="interleave"), NR.add_ref(a, b, 2))
