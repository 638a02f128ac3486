"""Python-side operator wrappers over the C ABI (torch tensors in, torch tensors out).

torch is used for device memory and streams only; every arithmetic op below is a hand-written sm_90a kernel in
aniportrait_b200/csrc reached through libaniportrait_b200.so. Activations are fp16 channels-last token matrices.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import I, LL, check, fptr, lib, ptr, stream_ptr

SHAPE_LOG = None  # dev aid: set to a list to record (kind, M, N, K, flags) of every GEMM / conv launch
GN_MAX_BLOCKS = 2368  # AP_GN_MAX_BLOCKS in include/aniportrait_b200.h
KERNEL_LAUNCHES = 0  # incremented by every wrapper; bench.py reports it as gpu_launches


def _count(n=1):
    global KERNEL_LAUNCHES
    KERNEL_LAUNCHES += n


def _ensure(t: torch.Tensor):
    if not t.is_cuda:
        raise _lib.ApError("aniportrait_b200 ops need CUDA tensors (no CPU fallback)")
    _lib.init(t.device.index if t.device.index is not None else torch.cuda.current_device())


# --------------------------------------------------------------------------------------------------------------
# weight repacking (done once at load time)
# --------------------------------------------------------------------------------------------------------------
def pack_conv3x3_weight(w: torch.Tensor, cin_pad_to: int = 64, cout_pad_to: int = 32) -> torch.Tensor:
    """[Cout, Cin, 3, 3] -> [Cout_p, 9*Cin_p] fp16, tap-major / channel-minor, zero padded."""
    cout, cin = w.shape[0], w.shape[1]
    cin_p = (cin + cin_pad_to - 1) // cin_pad_to * cin_pad_to
    cout_p = (cout + cout_pad_to - 1) // cout_pad_to * cout_pad_to
    wp = torch.zeros(cout_p, 3, 3, cin_p, dtype=torch.float16, device=w.device)
    wp[:cout, :, :, :cin] = w.permute(0, 2, 3, 1).to(torch.float16)
    return wp.reshape(cout_p, 9 * cin_p).contiguous()


def interleave_geglu(w: torch.Tensor, b: torch.Tensor | None):
    """FeedForward.net.0.proj weight [8C, C] (value half then gate half) -> rows interleaved in blocks of 16:
    [v0..15, g0..15, v16..31, g16..31, ...] so that a 32-column accumulator chunk holds matching value/gate pairs."""
    n2 = w.shape[0]
    half = n2 // 2
    assert half % 16 == 0
    idx = torch.arange(half, device=w.device).reshape(-1, 16)
    order = torch.cat([idx, idx + half], dim=1).reshape(-1)
    wi = w[order].contiguous()
    bi = b[order].contiguous() if b is not None else None
    return wi, bi


# --------------------------------------------------------------------------------------------------------------
# GEMM / conv
# --------------------------------------------------------------------------------------------------------------
class RowStats:
    """Per-row {sum, sumsq} partials of a GEMM output, written by its epilogue: the LayerNorm statistics of the next op."""

    def __init__(self, buf: torch.Tensor, parts: int, ld: int):
        self.buf, self.parts, self.ld = buf, parts, ld


class ColStats:
    """Per-channel {sum, sumsq} partials over 32-row blocks of a GEMM / conv output: the GroupNorm statistics of the next
    op. buf: fp32 [entries, C, 2]."""

    def __init__(self, buf: torch.Tensor):
        self.buf = buf


LN_EXTRA_K = 8    # columns the LayerNorm folding appends to K: (-mean_hi, -mean_lo, -mean_hi, 0 x 5) x (cs_hi, cs_hi, cs_lo, 0 x 5)


class LNFold:
    """LayerNorm folded into the consuming GEMM. The GEMM's weights are [W diag(gamma) | colsum_hi, colsum_hi, colsum_lo, 0..]
    (K + LN_EXTRA_K columns: models.blocks.fold_layer_norm), its bias beta.W^T + b; `stats` are the RowStats of the A
    operand x from its producer's epilogue. ops.gemm turns them into the [M, 8] operand (-mean_hi, -mean_lo, -mean_hi, 0..)
    and the per-row rstd (ap_layernorm_finalize_f16), appends the operand as a second K source, and the epilogue applies
    out = rstd * acc + bias."""

    def __init__(self, stats: RowStats, eps: float = 1e-5):
        self.stats, self.eps = stats, eps

    def operands(self, M: int, K: int):
        """(a2 [M, 8] fp16, rstd [M] fp32); computed once per RowStats."""
        cached = getattr(self.stats, "_ln_ops", None)
        if cached is None:
            dev = self.stats.buf.device
            a2 = torch.empty(M, LN_EXTRA_K, dtype=torch.float16, device=dev)
            rstd = torch.empty(M, dtype=torch.float32, device=dev)
            check(lib().ap_layernorm_finalize_f16(ptr(self.stats.buf), I(self.stats.parts), LL(self.stats.ld), LL(M), I(K),
                                                  _lib.c_float(self.eps), ptr(a2), fptr(rstd), stream_ptr()),
                  "ap_layernorm_finalize_f16")
            _count()
            cached = (a2, rstd)
            self.stats._ln_ops = cached
        return cached


def _epilogue_ext(M, N, device, row_stats, col_stats, ln, bias, flags, K, block_n):
    """Builds the ap_epilogue_ext for a call; returns (ext | None, RowStats | None, ColStats | None)."""
    bias_ld = 0
    if bias is not None and bias.dim() == 2 and bias.stride(0) != bias.shape[1]:
        bias_ld = bias.stride(0)           # a column slice of a wider table shared by several ops
    if not (row_stats or col_stats or ln is not None or bias_ld):
        return None, None, None
    ext = _lib.EpilogueExt()
    m_pad = (M + 127) // 128 * 128
    rs = cs = None
    if row_stats:
        parts = lib().ap_gemm_row_stat_parts(LL(M), I(N), I(K), I(flags), I(block_n))
        if parts <= 0:
            check(parts if parts < 0 else -1, "ap_gemm_row_stat_parts")
        rs = RowStats(torch.empty(2 * parts, m_pad, 2, dtype=torch.float32, device=device), 2 * parts, m_pad)
        ext.row_stat_out, ext.row_stat_ld = rs.buf.data_ptr(), m_pad
    if col_stats:
        cs = ColStats(torch.empty(m_pad // 32, N, 2, dtype=torch.float32, device=device))
        ext.col_stat_out, ext.col_stat_ld = cs.buf.data_ptr(), N
    if ln is not None:
        ext.ln_rstd = ln.rstd.data_ptr()
    ext.bias_ld = bias_ld
    return ext, rs, cs


def _with_stats(out, rs, cs, row_stats, col_stats):
    if not (row_stats or col_stats):
        return out
    res = [out]
    if row_stats:
        res.append(rs)
    if col_stats:
        res.append(cs)
    return tuple(res)


def gemm(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, residual: torch.Tensor | None = None,
         a2: torch.Tensor | None = None, geglu: bool = False, out: torch.Tensor | None = None,
         bias_group_rows: int = 0, n_valid: int = 0, block_n: int = 0, out_f32: bool = False,
         row_stats: bool = False, col_stats: bool = False, ln: LNFold | None = None, gelu: bool = False,
         quick_gelu: bool = False):
    """out = [a | a2] @ w.T (+bias) (+residual); a:[M,K1] fp16 (row stride may exceed K1), w:[N,K1+K2] fp16.
    gelu: out = gelu_erf(a @ w.T + bias) (AP_GEMM_GELU; not with a residual, GEGLU or `ln`).
    quick_gelu: out = y * sigmoid(1.702 y), y = a @ w.T + bias (AP_GEMM_QUICK_GELU; same restrictions, not with gelu).
    row_stats / col_stats: also return the epilogue's RowStats / ColStats of `out` (-> (out, RowStats?, ColStats?)).
    ln: fold a LayerNorm of `a` into this GEMM (see LNFold). bias may be a column slice of a wider fp32 table."""
    _ensure(a)
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and a.dim() == 2 and w.dim() == 2
    assert a.stride(1) == 1 and w.is_contiguous()
    M, K1 = a.shape
    N = w.shape[0]
    K2 = 0
    if ln is not None:
        assert a2 is None and bias is not None, "LayerNorm folding: single-source A, folded bias required"
        a2, ln.rstd = ln.operands(M, K1)
    if a2 is not None:
        assert a2.dtype == torch.float16 and a2.shape[0] == M and a2.stride(1) == 1
        K2 = a2.shape[1]
    assert w.shape[1] == K1 + K2, (w.shape, K1, K2)
    nout = N // 2 if geglu else N
    if n_valid:
        nout = n_valid
    if out is None:
        out = torch.empty(M, nout, dtype=torch.float32 if out_f32 else torch.float16, device=a.device)
    assert out.stride(1) == 1 and out.dtype == (torch.float32 if out_f32 else torch.float16)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.stride(-1) == 1 and bias.shape[-1] == N
        assert bias.is_contiguous() or bias.dim() == 2
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.stride(1) == 1 and residual.shape[0] == M
    flags = (1 if geglu else 0) | (2 if out_f32 else 0) | (4 if gelu else 0) | (8 if quick_gelu else 0)
    ext, rs, cs = _epilogue_ext(M, N, a.device, row_stats, col_stats, ln, bias, flags, K1 + K2, block_n)
    rc = lib().ap_gemm_f16(ptr(a), LL(a.stride(0)), I(K1), ptr(a2), LL(a2.stride(0) if a2 is not None else 0), I(K2),
                           ptr(w), LL(M), I(N), fptr(bias), LL(bias_group_rows), ptr(residual),
                           LL(residual.stride(0) if residual is not None else 0), ptr(out), LL(out.stride(0)),
                           I(nout), I(flags), I(block_n), stream_ptr(), _lib.ext_ptr(ext))
    check(rc, "ap_gemm_f16")
    if SHAPE_LOG is not None:
        kind = "gemm_geglu" if geglu else ("gemm_gelu" if gelu else ("gemm_quick_gelu" if quick_gelu else "gemm"))
        SHAPE_LOG.append((kind, M, N, K1 + K2, int(residual is not None)))
    _count()
    return _with_stats(out, rs, cs, row_stats, col_stats)


def conv_col_stats_ok(nf: int, ho: int, wo: int) -> bool:
    """Can a 3x3 conv with this output grid emit GroupNorm column statistics from its epilogue? (mirrors the tile-box choice
    of ap_conv3x3_nhwc_f16: every 32-row sub-box of a tile must lie in one frame, entries frame-major)."""
    def pow2_div(v, cap):
        d = 1
        while d * 2 <= cap and v % (d * 2) == 0:
            d *= 2
        return d
    bw = pow2_div(wo, 128)
    bh = pow2_div(ho, 128 // bw)
    bnf = 128 // (bw * bh)
    tiles = (wo // bw) * (ho // bh)
    return (ho * wo) % 32 == 0 and bw * bh >= 32 and (bnf == 1 or tiles == 1)


def conv_m_tiles(nf: int, ho: int, wo: int) -> int:
    def pow2_div(v, cap):
        d = 1
        while d * 2 <= cap and v % (d * 2) == 0:
            d *= 2
        return d
    bw = pow2_div(wo, 128)
    bh = pow2_div(ho, 128 // bw)
    bnf = 128 // (bw * bh)
    return (nf + bnf - 1) // bnf * (wo // bw) * (ho // bh)


def conv3x3(x: torch.Tensor, w_packed: torch.Tensor, cout: int, bias: torch.Tensor | None = None,
            residual: torch.Tensor | None = None, x2: torch.Tensor | None = None, stride: int = 1,
            out: torch.Tensor | None = None, bias_group_rows: int = 0, block_n: int = 0, col_stats: bool = False):
    """x: [Nf, H, W, C1] fp16 channels-last (C1 % 64 == 0); w_packed: pack_conv3x3_weight(...); returns
    [Nf, H/stride, W/stride, cout] (and, with col_stats, the ColStats of the output for the next GroupNorm: only where
    conv_col_stats_ok(...) holds). bias may be a column slice of a wider fp32 table."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    nf, h, wd, c1 = x.shape
    c2 = 0
    if x2 is not None:
        assert x2.is_contiguous() and x2.shape[:3] == x.shape[:3]
        c2 = x2.shape[3]
    cout_p = w_packed.shape[0]
    assert w_packed.shape[1] == 9 * (c1 + c2), (w_packed.shape, c1, c2)
    ho, wo = h // stride, wd // stride
    if out is None:
        out = torch.empty(nf, ho, wo, cout, dtype=torch.float16, device=x.device)
    assert out.is_contiguous()
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.stride(-1) == 1 and bias.shape[-1] == cout_p
        assert bias.is_contiguous() or bias.dim() == 2
    if residual is not None:
        assert residual.is_contiguous() and residual.shape == out.shape
    ext, cs = None, None
    bias_ld = bias.stride(0) if (bias is not None and bias.dim() == 2 and bias.stride(0) != bias.shape[1]) else 0
    if col_stats or bias_ld:
        ext = _lib.EpilogueExt()
        ext.bias_ld = bias_ld
        if col_stats:
            assert cout == cout_p, "column statistics need an unpadded output width"
            cs = ColStats(torch.empty(4 * conv_m_tiles(nf, ho, wo), cout, 2, dtype=torch.float32, device=x.device))
            ext.col_stat_out, ext.col_stat_ld = cs.buf.data_ptr(), cout
    rc = lib().ap_conv3x3_nhwc_f16(ptr(x), I(c1), ptr(x2), I(c2), I(nf), I(h), I(wd), I(stride), ptr(w_packed),
                                   I(cout_p), fptr(bias), LL(bias_group_rows), ptr(residual), ptr(out), LL(cout),
                                   I(cout), I(block_n), stream_ptr(), _lib.ext_ptr(ext))
    check(rc, "ap_conv3x3_nhwc_f16")
    if SHAPE_LOG is not None:
        SHAPE_LOG.append((f"conv3x3_s{stride}", nf * ho * wo, cout_p, 9 * (c1 + c2), int(residual is not None)))
    _count()
    return (out, cs) if col_stats else out


# --------------------------------------------------------------------------------------------------------------
# normalisation
# --------------------------------------------------------------------------------------------------------------
_stats_ws = {}


def _stats_workspace(device, n):
    key = (device.index, torch.cuda.current_stream().cuda_stream)
    buf = _stats_ws.get(key)
    if buf is None or buf.numel() < n:
        # sized once for any realistic frame count: CUDA graphs keep this pointer, so it must never be re-allocated
        buf = torch.empty(max(n, 2 * 32 * (4096 + 2 * GN_MAX_BLOCKS)), dtype=torch.float32, device=device)
        _stats_ws[key] = buf
    return buf


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool,
               x2: torch.Tensor | None = None, out: torch.Tensor | None = None, stats: ColStats | None = None,
               stats2: ColStats | None = None) -> torch.Tensor:
    """x: [Nf, HW, C1] (or [Nf,H,W,C1]) fp16 channels-last; optional x2 concatenated along C. gamma/beta fp32 [C].
    stats / stats2: ColStats written by the epilogue of the op that produced x / x2: when every source has them, the
    statistics pass over the activation is skipped (finalize from the partials + apply only)."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    nf, c1 = x.shape[0], x.shape[-1]
    hw = x.numel() // (nf * c1)
    c2 = 0
    if x2 is not None:
        assert x2.is_contiguous() and x2.shape[0] == nf
        c2 = x2.shape[-1]
    c = c1 + c2
    assert gamma.dtype == torch.float32 and gamma.numel() == c and beta.numel() == c
    if out is None:
        out = torch.empty(*x.shape[:-1], c, dtype=torch.float16, device=x.device)
    fused = stats is not None and (x2 is None or stats2 is not None) and hw % 32 == 0 and groups <= 32
    ws = _stats_workspace(x.device, 2 * groups * (nf + 2 * GN_MAX_BLOCKS))
    if fused:
        for st, cc in ((stats, c1), (stats2, c2)):
            if st is not None:
                assert st.buf.shape[1] == cc and st.buf.shape[0] >= nf * hw // 32, (st.buf.shape, nf, hw, cc)
        rc = lib().ap_groupnorm_apply_nhwc_f16(ptr(x), I(c1), ptr(stats.buf), LL(c1), ptr(x2), I(c2),
                                               ptr(stats2.buf if stats2 is not None else None), LL(c2), I(nf), I(hw),
                                               I(groups), _lib.c_float(eps), fptr(gamma), fptr(beta),
                                               I(1 if silu else 0), fptr(ws), ptr(out), stream_ptr())
        check(rc, "ap_groupnorm_apply_nhwc_f16")
        _count(3 if x2 is not None else 2)
        return out
    stats = ws
    rc = lib().ap_groupnorm_nhwc_f16(ptr(x), I(c1), ptr(x2), I(c2), I(nf), I(hw), I(groups), _lib.c_float(eps),
                                     fptr(gamma), fptr(beta), I(1 if silu else 0), fptr(stats), ptr(out),
                                     stream_ptr())
    check(rc, "ap_groupnorm_nhwc_f16")
    _count(5 if x2 is not None else 3)
    return out


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5,
               pe: torch.Tensor | None = None, rows_per_pe: int = 0, pe_period: int = 0,
               out: torch.Tensor | None = None) -> torch.Tensor:
    """x: [rows, C] fp16; pe: optional fp32 [pe_period, C] added after the affine (row r uses pe[(r//rows_per_pe)%period])."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 2
    rows, c = x.shape
    if out is None:
        out = torch.empty_like(x)
    if pe is not None:
        assert pe.dtype == torch.float32 and pe.is_contiguous() and pe.shape[-1] == c and pe.shape[0] >= pe_period
    rc = lib().ap_layernorm_f16(ptr(x), LL(rows), I(c), _lib.c_float(eps), fptr(gamma), fptr(beta), fptr(pe),
                                I(rows_per_pe), I(pe_period), ptr(out), stream_ptr())
    check(rc, "ap_layernorm_f16")
    _count()
    return out


BN_MAX_BLOCKS = 2048  # AP_BN_MAX_BLOCKS in include/aniportrait_b200.h
_bn_ws = {}


ACTIVATIONS = {"none": 0, "relu": 1, "gelu": 2}   # AP_ACT_* in include/aniportrait_b200.h


def batch_norm_train(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, relu: bool = True,
                     out: torch.Tensor | None = None, act: str | None = None) -> torch.Tensor:
    """nn.BatchNorm2d in TRAIN mode (batch statistics over every row of the call, biased variance) + optional activation.
    x: [..., C] fp16 channels-last, C % 8 == 0; gamma/beta fp32 [C]. act: "none", "relu" or "gelu" (erf); when not
    given, `relu` chooses between ReLU and none."""
    if act is None:
        act = "relu" if relu else "none"
    if act not in ACTIVATIONS:
        raise ValueError(f"act {act!r} is not one of {list(ACTIVATIONS)}")
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    c = x.shape[-1]
    rows = x.numel() // c
    assert gamma.dtype == torch.float32 and gamma.numel() == c and beta.dtype == torch.float32 and beta.numel() == c
    if out is None:
        out = torch.empty_like(x)
    key = (x.device.index, torch.cuda.current_stream().cuda_stream)
    ws = _bn_ws.get(key)
    if ws is None:   # sized once for the widest layer: CUDA graphs keep this pointer
        ws = torch.empty(2 * 2048 * (BN_MAX_BLOCKS + 1), dtype=torch.float32, device=x.device)
        _bn_ws[key] = ws
    rc = lib().ap_batchnorm_train_nhwc_f16(ptr(x), LL(rows), I(c), fptr(gamma), fptr(beta), _lib.c_float(eps),
                                           I(ACTIVATIONS[act]), fptr(ws), LL(ws.numel()), ptr(out), stream_ptr())
    check(rc, "ap_batchnorm_train_nhwc_f16")
    _count(3)
    return out


def pack_conv_direct_weight(w: torch.Tensor, cin_pad: int, cout_pad: int) -> torch.Tensor:
    """[Cout, Cin, K, K] -> [cout_pad, K, K, cin_pad] fp16 (zero padded) for conv2d_direct."""
    cout, cin, k, _ = w.shape
    wp = torch.zeros(cout_pad, k, k, cin_pad, dtype=torch.float16, device=w.device)
    wp[:cout, :, :, :cin] = w.permute(0, 2, 3, 1).to(torch.float16)
    return wp.contiguous()


def conv2d_direct(x: torch.Tensor, w_packed: torch.Tensor, stride: int, pad: int = 1,
                  bias: torch.Tensor | None = None) -> torch.Tensor:
    """Small-channel direct convolution. x: [Nf, H, W, Cin] fp16 (Cin in {8, 16, 32}); w_packed from
    pack_conv_direct_weight; returns [Nf, Ho, Wo, Cout]."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4 and w_packed.dtype == torch.float16
    nf, h, wd, cin = x.shape
    cout, k, _, cin_w = w_packed.shape
    assert cin_w == cin and w_packed.is_contiguous()
    ho, wo = (h + 2 * pad - k) // stride + 1, (wd + 2 * pad - k) // stride + 1
    out = torch.empty(nf, ho, wo, cout, dtype=torch.float16, device=x.device)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == cout
    rc = lib().ap_conv2d_direct_nhwc_f16(ptr(x), I(cin), I(nf), I(h), I(wd), ptr(w_packed), I(cout), I(k), I(stride),
                                         I(pad), fptr(bias), ptr(out), stream_ptr())
    check(rc, "ap_conv2d_direct_nhwc_f16")
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------
# wav2vec2 audio encoder
# --------------------------------------------------------------------------------------------------------------
def conv1d_stem(wave: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Conv1d(1 -> Cout, kernel 10, stride 5, no bias) of an fp32 waveform [S] with fp32 weights [Cout, 10] (or the
    module's [Cout, 1, 10]) -> fp16 [T0, Cout], T0 = (S - 10) // 5 + 1."""
    _ensure(wave)
    assert wave.dtype == torch.float32 and wave.is_contiguous() and wave.dim() == 1
    w = w.reshape(w.shape[0], -1)
    assert w.dtype == torch.float32 and w.is_contiguous() and w.shape[1] == 10
    S, cout = wave.numel(), w.shape[0]
    if S < 10:
        raise ValueError(f"conv1d_stem: {S} samples give no output frame (need >= 10)")
    out = torch.empty((S - 10) // 5 + 1, cout, dtype=torch.float16, device=wave.device)
    check(lib().ap_conv1d_stem_f32(fptr(wave), LL(S), fptr(w), I(cout), ptr(out), stream_ptr()), "ap_conv1d_stem_f32")
    _count()
    return out


def pack_conv1d_weight(w: torch.Tensor) -> torch.Tensor:
    """Conv1d weight [Cout, Cin, k] -> [Cout, k*Cin] fp16, tap-major / channel-minor: a stride-2 conv over channels-last
    frames x [T, Cin] is then a GEMM whose A row m is frames 2m .. 2m+k-1 (see conv1d_s2)."""
    return w.permute(0, 2, 1).reshape(w.shape[0], -1).to(torch.float16).contiguous()


def conv1d_s2(x: torch.Tensor, w_packed: torch.Tensor, k: int, gelu: bool = True) -> torch.Tensor:
    """Conv1d(Cin -> Cout, kernel k in {2, 3}, stride 2, no padding) over x [T, Cin] fp16 (contiguous), as one GEMM
    without an im2col buffer: A row m = frames (2m, 2m+1) read with row stride 2 Cin, plus for k = 3 the second source
    frame 2m + 2 (a2 = x shifted by two frames, same row stride). Returns [(T - k) // 2 + 1, Cout] (GELU applied)."""
    assert x.is_contiguous() and x.dim() == 2 and k in (2, 3)
    T, c = x.shape
    to = (T - k) // 2 + 1
    if to < 1:
        raise ValueError(f"conv1d_s2: {T} frames give no output for kernel {k}")
    assert w_packed.shape[1] == k * c, (w_packed.shape, k, c)
    pairs = x.as_strided((to, 2 * c), (2 * c, 1))
    a2 = x[2:].as_strided((to, c), (2 * c, 1)) if k == 3 else None
    return gemm(pairs, w_packed, a2=a2, gelu=gelu)


def pack_pos_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """Grouped Conv1d weight [C, C / groups, K] (the weight norm already folded in) -> fp16 [C, K, C / groups]."""
    return w.permute(0, 2, 1).to(torch.float16).contiguous()


def pos_conv1d_gelu(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, groups: int) -> torch.Tensor:
    """x + GELU(Conv1d(C, C, K, padding=K/2, groups)(x)[:-1] + bias) over x [T, C] fp16 (the positional convolution of
    the wav2vec2 encoder with its SamePad trim and residual). w_packed from pack_pos_conv_weight; bias fp32 [C]."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 2
    T, c = x.shape
    assert w_packed.dtype == torch.float16 and w_packed.is_contiguous() and w_packed.shape[0] == c
    assert w_packed.shape[2] * groups == c and bias.dtype == torch.float32 and bias.numel() == c
    out = torch.empty_like(x)
    check(lib().ap_pos_conv1d_gelu_f16(ptr(x), LL(T), I(c), I(groups), I(w_packed.shape[1]), ptr(w_packed), fptr(bias),
                                       ptr(out), stream_ptr()), "ap_pos_conv1d_gelu_f16")
    _count()
    return out


def resample_rows_linear(x: torch.Tensor, t_out: int) -> torch.Tensor:
    """F.interpolate(mode="linear", align_corners=True) along the rows of x [T_in, C] fp16 -> [t_out, C]."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 2
    if t_out < 1:
        raise ValueError(f"resample_rows_linear: t_out={t_out} must be >= 1")
    out = torch.empty(t_out, x.shape[1], dtype=torch.float16, device=x.device)
    check(lib().ap_resample_rows_linear_f16(ptr(x), LL(x.shape[0]), I(x.shape[1]), ptr(out), LL(t_out), stream_ptr()),
          "ap_resample_rows_linear_f16")
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------
# CLIP vision encoder
# --------------------------------------------------------------------------------------------------------------
def patch_kpad(patch: int) -> int:
    """Width of the patch-embedding GEMM operand: 3 P^2 pixel columns plus the CLS column, padded to a multiple of 64."""
    return (3 * patch * patch + 1 + 63) // 64 * 64


def patchify(pixels: torch.Tensor, patch: int) -> torch.Tensor:
    """NCHW pixels [B, 3, H, W] (fp16 or fp32, contiguous) -> fp16 [B * (1 + Gh Gw), patch_kpad(patch)]: per image a CLS row
    (1.0 in column 3 P^2) then the patches in flatten(2) order, columns (c, ky, kx), zero padded (ap_patchify_nchw_f16)."""
    _ensure(pixels)
    assert pixels.dim() == 4 and pixels.shape[1] == 3 and pixels.is_contiguous()
    assert pixels.dtype in (torch.float16, torch.float32), pixels.dtype
    B, _, H, W = pixels.shape
    kpad = patch_kpad(patch)
    out = torch.empty(B * (1 + (H // patch) * (W // patch)), kpad, dtype=torch.float16, device=pixels.device)
    check(lib().ap_patchify_nchw_f16(ptr(pixels), I(1 if pixels.dtype == torch.float32 else 0), I(B), I(H), I(W),
                                     I(patch), ptr(out), I(kpad), stream_ptr()), "ap_patchify_nchw_f16")
    _count()
    return out


def softmax_rows(x: torch.Tensor) -> torch.Tensor:
    """In-place row softmax of an fp16 matrix [rows, cols] (cols even)."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.dim() == 2 and x.stride(1) == 1
    check(lib().ap_softmax_rows_f16(ptr(x), ptr(x), LL(x.shape[0]), I(x.shape[1]), LL(x.stride(0)), stream_ptr()),
          "ap_softmax_rows_f16")
    _count()
    return x


# --------------------------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------------------------
def head_pad(d: int) -> int:
    """Head dim padded to a whole number of 64-column swizzle atoms (40->64, 80->128, 88->128, 160->192)."""
    p = (d + 63) // 64 * 64
    if p > 192:
        raise _lib.ApError(f"head_dim {d} > 192 is not supported by the fused attention kernel")
    return p


def pad_head_rows(w: torch.Tensor, heads: int, dpad: int) -> torch.Tensor:
    """Projection weight [heads*d, K] -> [heads*dpad, K] with zero rows after each head's d rows."""
    hd, k = w.shape
    d = hd // heads
    out = torch.zeros(heads, dpad, k, dtype=w.dtype, device=w.device)
    out[:, :d] = w.view(heads, d, k)
    return out.reshape(heads * dpad, k).contiguous()


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, n_frames: int, tokens: int, heads: int,
              head_dim: int, dpad: int, bank_k: torch.Tensor | None = None, bank_v: torch.Tensor | None = None,
              bank_tokens: int = 0, n_banks: int = 0, first_bank_frame: int = 0, frames_per_bank: int = 1,
              scale: float | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
    """q/k/v: column-slices [n_frames*tokens, heads*dpad] of one fp16 buffer (same row stride); returns
    [n_frames*tokens, heads*head_dim]."""
    _ensure(q)
    rows = n_frames * tokens
    for t in (q, k, v):
        assert t.dtype == torch.float16 and t.shape == (rows, heads * dpad) and t.stride(1) == 1
        assert t.stride(0) == q.stride(0)
    if out is None:
        out = torch.empty(rows, heads * head_dim, dtype=torch.float16, device=q.device)
    ld_bank = 0
    if bank_k is not None:
        assert bank_k.shape == (n_banks * bank_tokens, heads * dpad) and bank_k.stride(1) == 1
        assert bank_v.shape == bank_k.shape and bank_v.stride(0) == bank_k.stride(0)
        ld_bank = bank_k.stride(0)
    if scale is None:
        scale = head_dim ** -0.5
    rc = lib().ap_attention_f16(ptr(q), ptr(k), ptr(v), LL(q.stride(0)), ptr(bank_k), ptr(bank_v), LL(ld_bank),
                                I(bank_tokens), I(n_banks), I(n_frames), I(tokens), I(heads), I(head_dim), I(dpad),
                                I(first_bank_frame), I(frames_per_bank), _lib.c_float(scale), ptr(out),
                                LL(out.stride(0)), stream_ptr())
    check(rc, "ap_attention_f16")
    _count()
    return out


def temporal_attention(qkv: torch.Tensor, B: int, F: int, N: int, C: int, heads: int,
                       out: torch.Tensor | None = None) -> torch.Tensor:
    _ensure(qkv)
    assert qkv.dtype == torch.float16 and qkv.shape == (B * F * N, 3 * C) and qkv.stride(1) == 1
    if out is None:
        out = torch.empty(B * F * N, C, dtype=torch.float16, device=qkv.device)
    scale = (C // heads) ** -0.5
    rc = lib().ap_temporal_attention_f16(ptr(qkv), LL(qkv.stride(0)), ptr(out), LL(out.stride(0)), I(B), I(F), I(N),
                                         I(C), I(heads), _lib.c_float(scale), stream_ptr())
    check(rc, "ap_temporal_attention_f16")
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------
# elementwise / layout
# --------------------------------------------------------------------------------------------------------------
def add(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    _ensure(a)
    assert a.dtype == torch.float16 and a.shape == b.shape and a.is_contiguous() and b.is_contiguous()
    if out is None:
        out = torch.empty_like(a)
    check(lib().ap_add_f16(ptr(a), ptr(b), ptr(out), LL(a.numel()), stream_ptr()), "ap_add_f16")
    _count()
    return out


def add_bcast(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """a: [dup*n...], b: [n...] broadcast over the leading duplicate (CFG) dimension."""
    _ensure(a)
    assert a.dtype == torch.float16 and a.is_contiguous() and b.is_contiguous() and a.numel() % b.numel() == 0
    if out is None:
        out = torch.empty_like(a)
    check(lib().ap_add_bcast_f16(ptr(a), ptr(b), ptr(out), LL(a.numel()), LL(b.numel()), stream_ptr()),
          "ap_add_bcast_f16")
    _count()
    return out


def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """t: fp32 [B] on device -> fp16 [B, dim] (cos | sin)."""
    _ensure(t)
    assert t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty(t.numel(), dim, dtype=torch.float16, device=t.device)
    check(lib().ap_timestep_embedding_f16(fptr(t), I(t.numel()), I(dim), ptr(out), stream_ptr()),
          "ap_timestep_embedding_f16")
    _count()
    return out


def silu(x: torch.Tensor) -> torch.Tensor:
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    out = torch.empty_like(x)
    check(lib().ap_silu_f16(ptr(x), ptr(out), LL(x.numel()), stream_ptr()), "ap_silu_f16")
    _count()
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    _ensure(x)
    nf, h, w, c = x.shape
    assert x.dtype == torch.float16 and x.is_contiguous()
    out = torch.empty(nf, 2 * h, 2 * w, c, dtype=torch.float16, device=x.device)
    check(lib().ap_upsample2x_nhwc_f16(ptr(x), ptr(out), I(nf), I(h), I(w), I(c), stream_ptr()), "ap_upsample2x")
    _count()
    return out


def ncfhw_to_nhwc(x: torch.Tensor, cpad: int) -> torch.Tensor:
    """[B, C, F, H, W] -> [(B F), H, W, cpad] (zero padded channels)."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 5
    b, c, f, h, w = x.shape
    out = torch.empty(b * f, h, w, cpad, dtype=torch.float16, device=x.device)
    check(lib().ap_ncfhw_to_nhwc_f16(ptr(x), ptr(out), I(b), I(c), I(f), I(h * w), I(cpad), stream_ptr()),
          "ap_ncfhw_to_nhwc_f16")
    _count()
    return out


def nhwc_to_ncfhw(x: torch.Tensor, B: int, C: int, F: int) -> torch.Tensor:
    """[(B F), H, W, ld>=C] -> [B, C, F, H, W]."""
    _ensure(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4 and x.shape[0] == B * F
    _, h, w, ld = x.shape
    out = torch.empty(B, C, F, h, w, dtype=torch.float16, device=x.device)
    check(lib().ap_nhwc_to_ncfhw_f16(ptr(x), ptr(out), I(B), I(C), I(F), I(h * w), I(ld), stream_ptr()),
          "ap_nhwc_to_ncfhw_f16")
    _count()
    return out


def gather_window(latents: torch.Tensor, frame_idx: torch.Tensor, dup: int, cpad: int = 64) -> torch.Tensor:
    """latents [L, H, W, 4] fp16 -> UNet input [(dup F), H, W, cpad]."""
    _ensure(latents)
    L, h, w, c = latents.shape
    assert c == 4 and latents.dtype == torch.float16 and latents.is_contiguous() and frame_idx.dtype == torch.int32
    F = frame_idx.numel()
    out = torch.empty(dup * F, h, w, cpad, dtype=torch.float16, device=latents.device)
    check(lib().ap_gather_window_f16(ptr(latents), _lib.ctypes.cast(_lib.c_void_p(frame_idx.data_ptr()),
                                                                     _lib.POINTER(_lib.c_int)),
                                     ptr(out), I(dup), I(F), I(h * w), I(cpad), stream_ptr()), "ap_gather_window_f16")
    _count()
    return out


def gather_window_scaled(latents: torch.Tensor, frame_idx: torch.Tensor, scale: torch.Tensor, dup: int,
                         cpad: int = 64) -> torch.Tensor:
    """gather_window with the latents multiplied by scale[0] (an fp32 device scalar read by the kernel, so a captured
    graph sees the value of every step) and rounded to fp16 once: EulerDiscreteScheduler.scale_model_input."""
    _ensure(latents)
    L, h, w, c = latents.shape
    assert c == 4 and latents.dtype == torch.float16 and latents.is_contiguous() and frame_idx.dtype == torch.int32
    assert scale.dtype == torch.float32 and scale.is_cuda and scale.numel() >= 1
    F = frame_idx.numel()
    out = torch.empty(dup * F, h, w, cpad, dtype=torch.float16, device=latents.device)
    check(lib().ap_gather_window_scaled_f16(ptr(latents), _lib.ctypes.cast(_lib.c_void_p(frame_idx.data_ptr()),
                                                                            _lib.POINTER(_lib.c_int)),
                                            fptr(scale), ptr(out), I(dup), I(F), I(h * w), I(cpad), stream_ptr()),
          "ap_gather_window_scaled_f16")
    _count()
    return out


def scatter_accumulate(pred: torch.Tensor, frame_idx: torch.Tensor, acc: torch.Tensor):
    """pred [(B F), H, W, ld] fp16 (first 4 channels) accumulated into acc fp32 [B, L, H, W, 4] at frame_idx."""
    _ensure(pred)
    B, L, h, w, _ = acc.shape
    F = frame_idx.numel()
    assert pred.shape[0] == B * F and acc.dtype == torch.float32 and acc.is_contiguous() and pred.is_contiguous()
    check(lib().ap_scatter_accumulate_f16(ptr(pred), I(pred.shape[-1]),
                                          _lib.ctypes.cast(_lib.c_void_p(frame_idx.data_ptr()), _lib.POINTER(_lib.c_int)),
                                          fptr(acc), I(B), I(F), I(L), I(h * w), stream_ptr()),
          "ap_scatter_accumulate_f16")
    _count()


PREDICTION_TYPES = {"v_prediction": 0, "epsilon": 1, "sample": 2}   # AP_PRED_* in include/aniportrait_b200.h


def cfg_ddim_step(acc: torch.Tensor, inv_count: torch.Tensor, guidance: float, alpha_t: float, alpha_prev: float,
                  latents: torch.Tensor, prediction_type: str = "v_prediction", clip_range: float = 0.0):
    """In place: latents <- DDIM (eta = 0) step of the CFG-combined prediction acc * inv_count; acc zeroed.
    inv_count holds per-frame weights: 1 / count (the overlap average) under CFG, 1 without CFG, where the reference steps
    on the sum of the windows' predictions (sharding.step_weights). clip_range > 0 clamps the predicted x0
    (DDIMScheduler clip_sample)."""
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type {prediction_type!r} is not one of {sorted(PREDICTION_TYPES)}")
    _ensure(latents)
    B, L, h, w, _ = acc.shape
    assert latents.shape == (L, h, w, 4) and latents.dtype == torch.float16 and inv_count.dtype == torch.float32
    check(lib().ap_cfg_ddim_step_f16(fptr(acc), fptr(inv_count), I(1 if B == 2 else 0), _lib.c_float(guidance),
                                     _lib.c_float(alpha_t), _lib.c_float(alpha_prev),
                                     I(PREDICTION_TYPES[prediction_type]), _lib.c_float(clip_range), ptr(latents),
                                     I(L), I(h * w), stream_ptr()), "ap_cfg_ddim_step_f16")
    _count()


def cfg_multistep_step(acc: torch.Tensor, inv_count: torch.Tensor, guidance: float, coef, latents: torch.Tensor,
                       hist: torch.Tensor):
    """In place: one step of a multistep sampler on the CFG-combined prediction v = acc * inv_count (weights as in
    cfg_ddim_step); acc zeroed. coef: pipelines.scheduler.MultistepCoefficients (m = c_xx x + c_xv v, latents <- k_x x +
    k_0 m + k_1 hist, hist <- m if coef.store). hist: fp32 [L, H, W, 4], read only when k_1 != 0."""
    _ensure(latents)
    B, L, h, w, _ = acc.shape
    assert latents.shape == (L, h, w, 4) and latents.dtype == torch.float16 and inv_count.dtype == torch.float32
    assert hist.shape == (L, h, w, 4) and hist.dtype == torch.float32 and hist.is_contiguous()
    f = _lib.c_float
    check(lib().ap_cfg_multistep_step_f16(fptr(acc), fptr(inv_count), I(1 if B == 2 else 0), f(guidance), f(coef.c_xx),
                                          f(coef.c_xv), f(coef.k_x), f(coef.k_0), f(coef.k_1), I(1 if coef.store else 0),
                                          fptr(hist), ptr(latents), I(L), I(h * w), stream_ptr()),
          "ap_cfg_multistep_step_f16")
    _count()


def pack_frames_u8(video: torch.Tensor, rescale: bool = False) -> torch.Tensor:
    """video [B, 3, F, H, W] fp16 (any strides, e.g. the decoder's [F, 3, H, W] frames viewed as a video) -> [B, F, H, W, 3]
    uint8 on the device: the bytes `save_videos_grid` (reference src/utils/util.py:87-104) makes on the host from the fp32
    copy, `(x * 255).astype(uint8)` after `(x + 1) / 2` if rescale."""
    _ensure(video)
    assert video.dim() == 5 and video.shape[1] == 3 and video.dtype == torch.float16, "pack_frames_u8: [B, 3, F, H, W] fp16"
    B, _, F, H, W = video.shape
    out = torch.empty(B, F, H, W, 3, dtype=torch.uint8, device=video.device)
    strides = (_lib.c_longlong * 5)(*video.stride())
    check(lib().ap_pack_frames_u8(ptr(video), strides, I(B), I(F), I(H), I(W), I(1 if rescale else 0), ptr(out),
                                  stream_ptr()), "ap_pack_frames_u8")
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------
# Face-mesh projection and landmark pose frames
# --------------------------------------------------------------------------------------------------------------
LMK_CANVAS = 512       # AP_LMK_CANVAS
LMK_MAX_EDGES = 255    # AP_LMK_MAX_EDGES


def project_points(base: torch.Tensor, matrices: torch.Tensor, proj, width: float, height: float,
                   offsets: torch.Tensor | None = None) -> torch.Tensor:
    """fp64 pixel coordinates [L, N, 2] of base fp64 [N, 3] or [L, N, 3] (+ offsets fp32 [L, N, 3], added in fp64) under
    the per-frame fp64 matrices [L, 4, 4] and the projection `proj` (16 host floats, row-major P): ap_project_points_f64."""
    _ensure(matrices)
    L = matrices.shape[0]
    N = base.shape[-2]
    assert matrices.dtype == torch.float64 and matrices.is_contiguous() and tuple(matrices.shape) == (L, 4, 4)
    assert base.dtype == torch.float64 and base.is_contiguous() and base.device == matrices.device
    assert tuple(base.shape) in ((N, 3), (L, N, 3)), base.shape
    if offsets is not None:
        assert offsets.dtype == torch.float32 and offsets.is_contiguous() and tuple(offsets.shape) == (L, N, 3)
        assert offsets.device == matrices.device
    p = (_lib.ctypes.c_double * 16)(*[float(v) for v in proj])
    out = torch.empty(L, N, 2, dtype=torch.float64, device=matrices.device)
    dp = _lib.ctypes.POINTER(_lib.ctypes.c_double)
    check(lib().ap_project_points_f64(fptr(offsets), _lib.ctypes.cast(ptr(base), dp), I(1 if base.dim() == 3 else 0),
                                      _lib.ctypes.cast(ptr(matrices), dp), p, I(L), I(N),
                                      _lib.ctypes.c_double(width), _lib.ctypes.c_double(height),
                                      _lib.ctypes.cast(ptr(out), dp), stream_ptr()), "ap_project_points_f64")
    _count()
    return out


def draw_landmarks(keypoints: torch.Tensor, size_x: float, size_y: float, normed: bool, edges, colors,
                   thickness: int = 2) -> torch.Tensor:
    """Landmark pose frames uint8 [L, 512, 512, 3] of fp64 keypoints [L, N, 2] in one launch (ap_draw_landmarks_u8).
    edges: int32 [E, 2] and colors: uint8 [E, 3] host arrays in draw order (numpy or CPU tensors)."""
    import numpy as np
    _ensure(keypoints)
    assert keypoints.dtype == torch.float64 and keypoints.is_contiguous() and keypoints.dim() == 3
    assert keypoints.shape[2] == 2
    L, N, _ = keypoints.shape
    e = np.ascontiguousarray(edges, dtype=np.int32).reshape(-1, 2)
    c = np.ascontiguousarray(colors, dtype=np.uint8).reshape(-1, 3)
    assert len(e) == len(c)
    out = torch.empty(L, LMK_CANVAS, LMK_CANVAS, 3, dtype=torch.uint8, device=keypoints.device)
    check(lib().ap_draw_landmarks_u8(_lib.ctypes.cast(ptr(keypoints), _lib.ctypes.POINTER(_lib.ctypes.c_double)), I(L),
                                     I(N), _lib.ctypes.c_double(size_x), _lib.ctypes.c_double(size_y),
                                     I(1 if normed else 0), e.ctypes.data_as(_lib.ctypes.POINTER(_lib.ctypes.c_int)),
                                     c.ctypes.data_as(_lib.ctypes.POINTER(_lib.ctypes.c_ubyte)), I(len(e)),
                                     I(thickness), ptr(out), stream_ptr()), "ap_draw_landmarks_u8")
    _count()
    return out


RESIZE_MAX_SIDE = 8192   # AP_RESIZE_MAX_SIDE


def resize_linear_u8(src: torch.Tensor, size, mid=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """cv2.resize(frame, size) (INTER_LINEAR) of every frame of uint8 src [L, h, w, 3] -> [L, H, W, 3] for size = (W, H),
    in one launch (ap_resize_linear_u8). mid = (w', h'): cv2.resize(cv2.resize(frame, mid), size), the intermediate never
    stored. out: a contiguous uint8 [L, H, W, 3] to write into instead of a new tensor."""
    _ensure(src)
    assert src.dtype == torch.uint8 and src.is_contiguous() and src.dim() == 4 and src.shape[3] == 3, (src.dtype, src.shape)
    L, h, w, _ = src.shape
    W, H = (int(v) for v in size)
    mw, mh = (0, 0) if mid is None else (int(v) for v in mid)
    for what, sides in (("source", (w, h)), ("intermediate", () if mid is None else (mw, mh)), ("output", (W, H))):
        if not all(1 <= v <= RESIZE_MAX_SIDE for v in sides):   # refused before the output is allocated
            raise ValueError(f"resize_linear_u8: {what} size {sides}: every side must lie in [1, {RESIZE_MAX_SIDE}]")
    if out is None:
        out = torch.empty(L, H, W, 3, dtype=torch.uint8, device=src.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (L, H, W, 3), (out.dtype, out.shape)
    assert out.device == src.device
    check(lib().ap_resize_linear_u8(ptr(src), I(L), I(w), I(h), I(mw), I(mh), I(W), I(H), ptr(out), stream_ptr()),
          "ap_resize_linear_u8")
    _count()
    return out


RESIZE_PIL_MAX_SCALE = 32   # AP_RESIZE_PIL_MAX_SCALE


def resize_pil_bilinear_u8(src: torch.Tensor, size, out: torch.Tensor | None = None) -> torch.Tensor:
    """Image.resize(size, Image.BILINEAR) (Pillow's 8-bit resampler) of every frame of uint8 RGB src [L, h, w, 3] ->
    [L, H, W, 3] for size = (W, H), in one launch (ap_resize_pil_bilinear_u8); a same-size call is a device copy and no
    launch. Every side lies in [1, RESIZE_MAX_SIDE] and no axis shrinks by more than RESIZE_PIL_MAX_SCALE. out: a contiguous
    uint8 [L, H, W, 3] to write into instead of a new tensor."""
    _ensure(src)
    assert src.dtype == torch.uint8 and src.is_contiguous() and src.dim() == 4 and src.shape[3] == 3, (src.dtype, src.shape)
    L, h, w, _ = src.shape
    W, H = (int(v) for v in size)
    for what, sides in (("source", (w, h)), ("output", (W, H))):
        if not all(1 <= v <= RESIZE_MAX_SIDE for v in sides):   # refused before the output is allocated
            raise ValueError(f"resize_pil_bilinear_u8: {what} size {sides}: every side must lie in [1, {RESIZE_MAX_SIDE}]")
    if w > RESIZE_PIL_MAX_SCALE * W or h > RESIZE_PIL_MAX_SCALE * H:
        raise ValueError(f"resize_pil_bilinear_u8: {(w, h)} -> {(W, H)} shrinks an axis by more than "
                         f"{RESIZE_PIL_MAX_SCALE}x")
    if out is None:
        out = torch.empty(L, H, W, 3, dtype=torch.uint8, device=src.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (L, H, W, 3), (out.dtype, out.shape)
    assert out.device == src.device
    check(lib().ap_resize_pil_bilinear_u8(ptr(src), I(L), I(w), I(h), I(W), I(H), ptr(out), stream_ptr()),
          "ap_resize_pil_bilinear_u8")
    if (w, h) != (W, H):
        _count()
    return out


GRID_MAX_TILES = 16   # AP_GRID_MAX_TILES
_GRID_DTYPES = {torch.uint8: 0, torch.float16: 1, torch.float32: 2}   # AP_GRID_U8 / AP_GRID_F16 / AP_GRID_F32


def grid_shape(B: int, n_rows: int, H: int, W: int):
    """(GH, GW) of torchvision.utils.make_grid(padding=2) for B tiles of H x W; B = 1 is the tile itself."""
    if B == 1:
        return H, W
    xmaps = min(n_rows, B)
    return -(-B // xmaps) * (H + 2) + 2, xmaps * (W + 2) + 2


def video_grid_u8(tiles, n_rows: int, T: int, bgr=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """save_videos_grid's frames of torch.cat(tiles) as uint8 [T, GH, GW, 3], in one launch (ap_video_grid_u8).
    tiles: CUDA uint8 [T' >= T or 1, H, W, 3] frame bytes (T' = 1 repeats the frame; bgr[i] swaps their channels) or
    fp16 / fp32 videos [1, 3, T' >= T, H, W] in [0, 1], any strides. out: a contiguous uint8 [T, GH, GW, 3] to reuse."""
    B = len(tiles)
    if not 1 <= B <= GRID_MAX_TILES:
        raise ValueError(f"video_grid_u8: {B} tiles, expected 1 to {GRID_MAX_TILES}")
    bgr = [False] * B if bgr is None else [bool(b) for b in bgr]
    if len(bgr) != B:
        raise ValueError(f"video_grid_u8: {len(bgr)} bgr flags for {B} tiles")
    arr = (_lib.GridTile * B)()
    H = W = None
    for i, t in enumerate(tiles):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError(f"video_grid_u8: tile {i} is not a CUDA tensor (no CPU fallback)")
        if t.dtype not in _GRID_DTYPES:
            raise TypeError(f"video_grid_u8: tile {i} has dtype {t.dtype}; expected uint8, float16 or float32")
        if t.dtype == torch.uint8:
            if t.dim() != 4 or t.shape[3] != 3:
                raise ValueError(f"video_grid_u8: uint8 tile {i} must be [T, H, W, 3], got {tuple(t.shape)}")
            n, h, w = t.shape[:3]
            st, sh, sw, sc = t.stride()
        else:
            if t.dim() != 5 or t.shape[0] != 1 or t.shape[1] != 3:
                raise ValueError(f"video_grid_u8: video tile {i} must be [1, 3, T, H, W], got {tuple(t.shape)}")
            if bgr[i]:
                raise ValueError(f"video_grid_u8: the bgr flag applies to uint8 tiles only (tile {i})")
            n, h, w = t.shape[2:]
            _, sc, st, sh, sw = t.stride()
        if n != 1 and n < T or (n == 1 and t.dtype != torch.uint8 and T > 1):
            raise ValueError(f"video_grid_u8: tile {i} has {n} frames for a {T}-frame grid")
        if (H, W) not in ((None, None), (h, w)):
            raise ValueError(f"video_grid_u8: tile {i} is {h}x{w}, tile 0 is {H}x{W}")
        H, W = h, w
        if t.device != tiles[0].device:
            raise ValueError(f"video_grid_u8: tile {i} is on {t.device}, tile 0 on {tiles[0].device}")
        arr[i] = _lib.GridTile(t.data_ptr(), _GRID_DTYPES[t.dtype], int(bgr[i]), 0 if n == 1 else st, sh, sw, sc)
    if T < 1 or n_rows < 1:
        raise ValueError(f"video_grid_u8: T={T}, n_rows={n_rows}")
    GH, GW = grid_shape(B, n_rows, H, W)
    _ensure(tiles[0])
    if out is None:
        out = torch.empty(T, GH, GW, 3, dtype=torch.uint8, device=tiles[0].device)
    if not (out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (T, GH, GW, 3)
            and out.device == tiles[0].device):
        raise ValueError(f"video_grid_u8: out must be a contiguous uint8 {(T, GH, GW, 3)} on {tiles[0].device}")
    check(lib().ap_video_grid_u8(arr, I(B), I(n_rows), I(T), I(H), I(W), ptr(out), stream_ptr()), "ap_video_grid_u8")
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------
# Audio2Pose head-pose decoder
# --------------------------------------------------------------------------------------------------------------
POSE_VEC = 6656          # AP_POSE_VEC: per-layer fp32 vector (biases, then the three LayerNorms' weight and bias)
POSE_E, POSE_HEADS, POSE_FFN = 512, 8, 1024


def pose_decoder(layers: dict, pose_map_w: torch.Tensor, pose_map_b: torch.Tensor, pose_map_r_w: torch.Tensor,
                 pose_map_r_b: torch.Tensor, pe: torch.Tensor, mask: torch.Tensor, id_row: torch.Tensor,
                 cross: torch.Tensor, T: int, eps: float) -> torch.Tensor:
    """All T steps of the autoregressive pose decoder in one launch (ap_pose_decoder_f16) -> fp32 [T, out_dim].
    layers: w_qkv / w_out / w_ff1 / w_ff2 fp16 [L, 1536 | 512 | 1024 | 512, 512 | 512 | 512 | 1024], vec fp32 [L, POSE_VEC];
    pose_map_w fp32 [512, out_dim], pose_map_r_w [out_dim, 512]; pe fp32 [pe_len, 512]; mask fp32 [8, n, n];
    id_row fp32 [512]; cross fp32 [T, L * 512]."""
    _ensure(cross)
    w_qkv, w_out, w_ff1, w_ff2, vec = (layers[k] for k in ("w_qkv", "w_out", "w_ff1", "w_ff2", "vec"))
    L = w_qkv.shape[0]
    for t, shape in ((w_qkv, (L, 3 * POSE_E, POSE_E)), (w_out, (L, POSE_E, POSE_E)), (w_ff1, (L, POSE_FFN, POSE_E)),
                     (w_ff2, (L, POSE_E, POSE_FFN))):
        assert t.dtype == torch.float16 and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, t.shape, shape)
    od = pose_map_r_w.shape[0]
    f32s = ((vec, (L, POSE_VEC)), (pose_map_w, (POSE_E, od)), (pose_map_b, (POSE_E,)), (pose_map_r_w, (od, POSE_E)),
            (pose_map_r_b, (od,)), (id_row, (POSE_E,)), (cross, (T, L * POSE_E)))
    for t, shape in f32s:
        assert t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, t.shape, shape)
    assert pe.dtype == torch.float32 and pe.is_contiguous() and pe.dim() == 2 and pe.shape[1] == POSE_E
    assert mask.dtype == torch.float32 and mask.is_contiguous() and mask.dim() == 3 and mask.shape[1] == mask.shape[2]
    prm = _lib.PoseDecoderParams(layers=L, out_dim=od, embed_dim=POSE_E, heads=mask.shape[0], ffn_dim=POSE_FFN,
                                 mask_len=mask.shape[1], pe_len=pe.shape[0], eps=eps,
                                 w_qkv=w_qkv.data_ptr(), w_out=w_out.data_ptr(), w_ff1=w_ff1.data_ptr(),
                                 w_ff2=w_ff2.data_ptr(), vec=vec.data_ptr(), pose_map_w=pose_map_w.data_ptr(),
                                 pose_map_b=pose_map_b.data_ptr(), pose_map_r_w=pose_map_r_w.data_ptr(),
                                 pose_map_r_b=pose_map_r_b.data_ptr(), pe=pe.data_ptr(), id_row=id_row.data_ptr(),
                                 mask=mask.data_ptr(), cross=cross.data_ptr())
    kv = torch.empty(L, 2, POSE_HEADS, T, POSE_E // POSE_HEADS, dtype=torch.float16, device=cross.device)
    out = torch.empty(T, od, dtype=torch.float32, device=cross.device)
    check(lib().ap_pose_decoder_f16(_lib.ctypes.byref(prm), I(T), ptr(kv), fptr(out), stream_ptr()),
          "ap_pose_decoder_f16")
    _count()
    return out


def pose_decoder_ctas(device: int = 0) -> int:
    """CTAs of the pose decoder's cluster on `device` (16, or 8 where 16 cannot be co-scheduled), chosen once."""
    _lib.init(device)
    n = _lib.c_int(0)
    with torch.cuda.device(device):
        check(lib().ap_pose_decoder_ctas(_lib.ctypes.byref(n)), "ap_pose_decoder_ctas")
    return n.value
