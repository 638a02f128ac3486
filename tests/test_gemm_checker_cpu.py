"""The GEMM / conv checker itself, without a GPU (gemm_reference.py): the fp32 emulation of the kernel passes both checks
on the GPU case table at reduced M, and its unrounded values use at most half of the derived bound; every modelled bug is rejected by at least one check, the exact-grid
generator refuses budgets that could round, and the nine-tap conv reference matches F.conv2d in float64."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_reference as GR

CPU = torch.device("cpu")
M_CPU = 257       # reduced M: keeps a partial last tile, a 32-row tail and more than one 128-row tile


def _m(case):
    return min(case["M"], M_CPU)


def _emulate_case(case, grid, bug=None, seed=0, unrounded=False):
    a, w, call, out, refkw = GR.build_gemm_case(case, CPU, grid, seed, M=_m(case))
    kw = dict(a2=call["a2"], bias=call["bias"], bias_group_rows=call["bias_group_rows"], residual=call["residual"],
              act=case["act"], n_valid=case["n_valid"], out_f32=case["out_f32"], bn=case["bn"] or 128, bug=bug)
    GR.emulate_gemm(a, w, out=out.view, **kw)
    ref = GR.gemm_ref(a, w, **refkw)
    if unrounded:
        return out, ref, GR.emulate_gemm(a, w, unrounded=True, **kw)
    return out, ref


@pytest.mark.parametrize("case", GR.GEMM_CASES, ids=lambda c: c["name"])
def test_emulation_passes_bounded_check(case):
    out, ref, y32 = _emulate_case(case, grid=False, unrounded=True)
    ratio = GR.check(out.view, ref, case["name"])
    out.check(case["name"])
    head = GR.headroom(y32, ref)
    print(f"\n[emulation] {case['name']}: worst error / bound = {ratio:.3f}, unrounded / pre-rounding bound = {head:.3f}")
    assert head <= 0.5


@pytest.mark.parametrize("case", [c for c in GR.GEMM_CASES if c["act"] is None], ids=lambda c: c["name"])
def test_emulation_exact_on_grid(case):
    out, ref, y32 = _emulate_case(case, grid=True, unrounded=True)
    GR.check_exact(out.view, ref, case["name"])
    GR.check(out.view, ref, case["name"])
    assert torch.equal(y32.double(), ref.o), "fp32 accumulation on the grid must be exact"


def test_exact_grid_rounds_and_stays_exact_at_large_k():
    """K = 23040 at M = 300: fp32 accumulation equals fp64 exactly, and most outputs need a rounding to fp16 (so round to
    nearest even and its ties are exercised)."""
    K, M, N = 23040, 300, 64
    mk_a, mk_w, _, _ = GR.grid_operands(K)
    g = torch.Generator().manual_seed(5)
    a, w = mk_a((M, K), g), mk_w((N, K), g)
    acc32 = GR._mm_steps(a.float(), w.float())
    acc64 = a.double() @ w.double().t()
    assert torch.equal(acc32.double(), acc64)
    needs_rounding = (acc64.half().double() != acc64).double().mean().item()
    print(f"\nK={K}: {needs_rounding:.0%} of the outputs need rounding to fp16")
    assert needs_rounding > 0.5


def test_exact_grid_refuses_overflowing_budget():
    GR.grid_operands(32736 - 40)
    with pytest.raises(AssertionError, match="2\\*\\*22"):
        GR.grid_operands(32768)
    with pytest.raises(AssertionError, match="2\\*\\*22"):
        GR.grid_operands(20000, j_max=64)


# ------------------------------------------------------------------------------------------------------ conv
CONV_CPU = [  # (nf, h, w, c1, c2, cout, stride)
    (2, 8, 8, 64, 0, 64, 1), (2, 8, 6, 64, 64, 96, 1), (3, 5, 5, 64, 0, 32, 1), (2, 8, 8, 64, 128, 64, 2),
    (2, 10, 14, 128, 64, 64, 2), (1, 6, 40, 64, 0, 64, 1),
]


def _conv_operands(nf, h, w, c1, c2, cout, grid, seed=0):
    from aniportrait_b200 import ops
    K = 9 * (c1 + c2)
    mk_a, mk_w, mk_b, _ = GR.grid_operands(K) if grid else GR.gauss_operands(K)
    g = torch.Generator().manual_seed(seed)
    x = mk_a((nf, h, w, c1), g)
    x2 = mk_a((nf, h, w, c2), g) if c2 else None
    wt = mk_w((cout, c1 + c2, 3, 3), g)
    wp = ops.pack_conv3x3_weight(wt)
    bias = mk_b((wp.shape[0],), g)
    return x, x2, wt, wp, bias


@pytest.mark.parametrize("nf,h,w,c1,c2,cout,stride", CONV_CPU)
def test_conv_reference_matches_conv2d(nf, h, w, c1, c2, cout, stride):
    x, x2, wt, wp, bias = _conv_operands(nf, h, w, c1, c2, cout, grid=False)
    ref = GR.conv_ref(x, wp, cout, x2=x2, stride=stride, bias=bias)
    xc = x if x2 is None else torch.cat([x, x2], -1)
    want = F.conv2d(xc.double().permute(0, 3, 1, 2), wt.double(), bias[:cout].double(), stride=stride, padding=1)
    want = want.permute(0, 2, 3, 1).reshape(-1, cout)
    assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("nf,h,w,c1,c2,cout,stride", CONV_CPU)
def test_conv_emulation_passes_both_checks(nf, h, w, c1, c2, cout, stride):
    for grid in (True, False):
        x, x2, wt, wp, bias = _conv_operands(nf, h, w, c1, c2, cout, grid)
        out = GR.emulate_conv(x, wp, cout, x2=x2, stride=stride, bias=bias)
        ref = GR.conv_ref(x, wp, cout, x2=x2, stride=stride, bias=bias, exact=grid)
        GR.check_both(out, ref, f"conv {nf}x{h}x{w} {c1}+{c2} s{stride}")
        y32 = GR.emulate_conv(x, wp, cout, x2=x2, stride=stride, bias=bias, unrounded=True)
        assert GR.headroom(y32, ref) <= 0.5


# ------------------------------------------------------------------------------------------------------ LayerNorm fold
def _ln_fold_emulate(mu_over_sigma, act=None, bug=None, M=200, K=320, N=640, seed=3, unrounded=False):
    """The folded-LN chain in fp32: the producer's fp16 x and its row partials, ln_finalize (E[x^2] - mean^2, hi/lo split
    of -mean), the folded weights of models.blocks.fold_layer_norm, and the GEMM emulation with the rstd epilogue."""
    from aniportrait_b200 import ops
    from aniportrait_b200.models.blocks import fold_layer_norm
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g) + mu_over_sigma * torch.randn(M, 1, generator=g).sign()).half()
    gamma = 1.0 + 0.2 * torch.randn(K, generator=g)
    beta = 0.1 * torch.randn(K, generator=g)
    w = torch.randn(N, K, generator=g) * K ** -0.5
    b = 0.1 * torch.randn(N, generator=g)
    xf = x.float()
    S, Q = xf.sum(1), (xf * xf).sum(1)
    mean = S * (1.0 / K)
    rstd = torch.rsqrt(torch.clamp(Q * (1.0 / K) - mean * mean, min=0) + 1e-5)
    hi = (-mean).half()
    lo = (-mean - hi.float()).half()
    a2 = torch.zeros(M, ops.LN_EXTRA_K, dtype=torch.float16)
    a2[:, 0], a2[:, 1], a2[:, 2] = hi, lo, hi
    wg, bias = fold_layer_norm(w, b, gamma, beta)
    wref, bref = w, b
    if act == "geglu":
        wg, bias = ops.interleave_geglu(wg, bias)
        wref, bref = ops.interleave_geglu(w, b)
    out = GR.emulate_gemm(x, wg, a2=a2, bias=bias, act=act, ln_rstd=rstd, bug=bug, unrounded=unrounded)
    ref = GR.ln_fold_ref(x, wref, bref, gamma, beta, 1e-5, wg, act=act)
    return out, ref


@pytest.mark.parametrize("ratio_ms", [0, 1, 4, 16, 64])
@pytest.mark.parametrize("act", [None, "geglu"])
def test_ln_fold_emulation_within_bound(ratio_ms, act):
    out, ref = _ln_fold_emulate(ratio_ms, act)
    r = GR.check(out, ref, f"LN fold mean/sigma={ratio_ms}")
    y32, _ = _ln_fold_emulate(ratio_ms, act, unrounded=True)
    head = GR.headroom(y32, ref)
    print(f"\n[emulation] LN fold mean/sigma={ratio_ms} {act}: worst error / bound = {r:.3f}, unrounded = {head:.3f}")
    assert head <= 0.5


# ------------------------------------------------------------------------------------------------------ modelled bugs
def _case(name):
    return next(c for c in GR.GEMM_CASES if c["name"] == name)


def _rejected(fn) -> str:
    try:
        fn()
    except AssertionError as e:
        return str(e).splitlines()[0][:160]
    return ""


def _gemm_bug_rejected(case, bug):
    msgs = []
    for grid in ((True, False) if case["act"] is None else (False,)):
        out, ref = _emulate_case(case, grid, bug=bug)
        msgs.append(_rejected(lambda: GR.check_both(out.view, ref, case["name"])))
        msgs.append(_rejected(lambda: out.check(case["name"])))
    return [m for m in msgs if m]


@pytest.mark.parametrize("bug,name", [
    ("m_tail", "m129"), ("m_tail", "bn160_m4101"), ("res_box", "bn64_bias_res_m129"), ("bias_tile", "bias_group_100"),
    ("bias_tile", "bias_group_72_bn32"), ("bias_ld", "bias_table_slice"), ("src2_kb", "k1280_plus8_src2"),
    ("src2_kb", "two_source_640_320"), ("bn160_chunk", "bn160_bias_res_m129"), ("bn160_chunk", "bn160_m4101"),
    ("geglu_swap", "geglu_bn64"), ("geglu_swap", "geglu_bn128_m4101"), ("n_valid", "n_valid_301"),
    ("n_valid", "n_valid_296"), ("n_valid", "out_f32_nvalid"),
])
def test_gemm_bug_rejected(bug, name):
    msgs = _gemm_bug_rejected(_case(name), bug)
    print(f"\n[bug {bug} on {name}] rejected by: {msgs}")
    assert msgs, f"modelled bug {bug} on {name} passed every check"


def test_conv_stride2_phase_bug_rejected():
    """Defect 1: the odd x-phase of source 2 addressed at C1 + c instead of C2 + c (C1 != C2)."""
    for nf, h, w, c1, c2, cout, stride in [(2, 8, 8, 64, 128, 64, 2), (2, 10, 14, 128, 64, 64, 2)]:
        for grid in (True, False):
            x, x2, wt, wp, bias = _conv_operands(nf, h, w, c1, c2, cout, grid)
            out = GR.emulate_conv(x, wp, cout, x2=x2, stride=stride, bias=bias, bug="phase_c1")
            ref = GR.conv_ref(x, wp, cout, x2=x2, stride=stride, bias=bias, exact=grid)
            msg = _rejected(lambda: GR.check_both(out, ref, "conv s2 two-source"))
            print(f"\n[bug phase_c1 {c1}+{c2} grid={grid}] {msg}")
            assert msg


@pytest.mark.parametrize("act", [None, "geglu"])
def test_ln_rstd_neighbour_row_rejected(act):
    out, ref = _ln_fold_emulate(1, act, bug="ln_row")
    msg = _rejected(lambda: GR.check(out, ref, "LN fold rstd of the next row"))
    print(f"\n[bug ln_row {act}] {msg}")
    assert msg


@pytest.mark.parametrize("bn", [32, 64, 160])
def test_row_stats_including_clipped_columns_rejected(bn):
    """Defect 3: row partials formed from every computed column although the store clips those >= n_valid."""
    M, N, nv = 129, 320, 288
    g = torch.Generator().manual_seed(7)
    full = torch.randn(M, N, generator=g).half()
    stored = full[:, :nv]
    parts = 2 * (N // bn)
    want, bnd = GR.row_stats_ref(stored, bn, parts)
    good = GR.emulate_row_stats(full, bn, parts, nv)
    assert GR.check_stats(good, want, bnd, "row stats") <= 1.0
    bad = GR.emulate_row_stats(full, bn, parts, nv, bug="stats_clipped")
    msg = _rejected(lambda: GR.check_stats(bad, want, bnd, "row stats with clipped columns"))
    print(f"\n[bug stats_clipped bn={bn}] {msg}")
    assert msg


def test_box_rows_cover_every_output_once():
    """The statistics box maps of gemm_box_rows / conv_box_rows name every output row exactly once."""
    for M in (1, 129, 4101):
        r = GR.gemm_box_rows(M, (M + 127) // 128, CPU)
        assert torch.equal(r[r >= 0].sort().values, torch.arange(M))
    for nf, ho, wo in [(4, 32, 32), (3, 16, 24), (8, 4, 8), (5, 5, 6), (3, 24, 48)]:
        r = GR.conv_box_rows(nf, ho, wo, CPU)
        assert torch.equal(r[r >= 0].sort().values, torch.arange(nf * ho * wo))


def test_group_norm_reference_matches_torch():
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(2, 64, 96, generator=g) * 2 + 3).half()
    gamma, beta = torch.randn(96, generator=g), torch.randn(96, generator=g)
    ref = GR.group_norm_ref(x, gamma, beta, 32, 1e-5, True)
    want = F.silu(F.group_norm(x.double().permute(0, 2, 1), 32, gamma.double(), beta.double(), 1e-5))
    assert torch.allclose(ref.o, want.permute(0, 2, 1).reshape(-1, 96), rtol=1e-12, atol=1e-12)
    assert math.isfinite(ref.bound.max().item())
