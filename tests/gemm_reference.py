"""fp64 references, per-element checks and an fp32 emulation of the wgmma GEMM / implicit-GEMM conv kernel
(ap_gemm_f16, ap_conv3x3_nhwc_f16 in csrc/ap_gemm.cu), of its fused row / column statistics and of the LayerNorm
folded into it. Imported by the CPU checker tests and the GPU contract tests; not a conftest.

References
----------
Every reference is computed in float64 on the inputs' device from the fp16 operands the kernel sees, and returns a
`Ref`: the exact result `o` [M, n_valid], the per-element bound `bound`, `locate(row, col)` (which names an element by
the kernel's work decomposition) and `exact`, whether the exact-grid check applies.
  gemm_ref   [a | a2] @ w.T, then the epilogue in the kernel's order: bias row m // bias_group_rows of a table with row
             stride bias_ld (a strided torch view), then GELU, quick-GELU or GEGLU (weights interleaved in blocks of 16:
             value rows then gate rows), then the residual. locate -> (m_tile, n_tile, 32-row box, 32-column chunk).
  conv_ref   3x3 conv, zero padding 1, stride 1 or 2, over the channel concat [x | x2], as a sum of nine shifted fp64
             matmuls (one per tap; no cuDNN), then the same epilogue with M = Nf*Ho*Wo rows. locate -> (frame, y, x, ch).
  ln_fold_ref  fp64 LayerNorm(x) followed by the linear layer with the ORIGINAL fp32 W, b, gamma, beta: the contract of
             models.blocks.fold_layer_norm + ops.LNFold, not a restatement of the fold.

Exact-grid check
----------------
`grid_operands` draws a = i/4 (i in [-4, 4]), w = j 2**-e / 32 (j in [-32, 32]), bias and residual as integer multiples
of the unit u = 2**-(7+e), and asserts on the host that K max|i j| + max|bias| + max|residual| <= 2**22 units. Every
partial sum of the accumulator and of the linear epilogue is then an integer multiple of u below 2**22 u, hence exact in
fp32 whatever the summation order and whether the hardware rounds or truncates. The only correct fp16 output of a linear
epilogue is then o*.to(float16) (round to nearest even) and the only correct fp32 output is o* itself; `check_exact`
asserts exactly that, element by element. This is the check that catches indexing bugs (a wrong tap, phase, row, bias
group, k-block or chunk): they move an output by at least one unit.

Bounded check (Gaussian data at realistic scale)
------------------------------------------------
With S = sum_k |a_k w_k| (one more fp64 GEMM) the accumulator obeys
    |acc - acc*| <= (ceil(K/16) + 2) 2**-22 S                                                           (E_acc)
one fp32 accumulator rounding (2**-24 of the partial sum, <= S) per k16 wgmma step, with a 4x allowance for truncation
and the tensor core's internal alignment. The epilogue then adds, in the kernel's order:
  bias / residual adds   2**-24 (|y*| + |b|) and 2**-24 (|y*| + |r|): one fp32 rounding per add;
  GELU (the csrc/ap_ptx.cuh polynomial: gelu(y) = max(y, 0) - t, t = |y| Phi(-|y|) from 2**(-q(z) z) ~ erfc(z))
      propagated  (|gelu'(y*)| + E_y) E_y            (|gelu''| <= 2 phi(0) < 1 covers the move of the derivative)
      own error   t (2**-14 + 2**-22 + (y**2 + 8) 2**-23) + 2**-23 |gelu(y*)| + 2**-26
                  2**-14: the polynomial's relative error against erfc over [0, 4.3], evaluated in float64 on a dense
                  grid (3.99e-5 worst, at the clamp); 2**-22: ex2.approx; (y**2 + 8) 2**-23: the fp32 roundings of
                  z and q(z) z, amplified by d ln erfc / d ln z <= 2 z**2 + 2; 2**-23 |gelu|: the final product and
                  subtraction; 2**-26: the tail beyond the z = 4.3 clamp (t < 1e-8 there).
  quick-GELU y sigmoid(1.702 y) = y rcp(1 + ex2(-2.4555 y))
      propagated  (|qgelu'(y*)| + E_y) E_y            (|qgelu''| <= 0.851 < 1)
      own error   |o*| (2**-20 + 4 |y| 2**-24) + 2**-26: ex2.approx 2**-22, rcp.approx 2**-23, two roundings
                  2**-24 each; the argument's rounding and the rounded constant move the exponent by <= 4|y| 2**-24
                  (relative, times (1 - sigmoid) <= 1); 2**-26 absolute for ftz and underflow.
  GEGLU o = v gelu(g)  |gelu(g*)| E_v + (|v*| + E_v)(|gelu'(g*)| + E_g) E_g + |v*| err_gelu(g*) + 2**-24 |o*|.
All these are multiplied by (1 + 2**-10) (second-order terms); the sum is `Ref.pre`, the bound on the fp32 value the
epilogue rounds. The fp16 output then adds half an ulp: 2**-11 |o*| (normal) + 2**-25 (subnormal). The rounding term has
no margin and cannot have one: a correctly rounded value just above a power of two sits at a ratio close to 1. So the
bounded check accepts at most a correctly rounded result of a value within `pre` of o*, and a whole-ulp error fails it
except where `pre` itself is an ulp wide. The headroom of the derivation is measured on the part that has one: the
emulation's unrounded fp32 values must stay within 0.5 `pre` (`headroom`). An fp32 output adds 2**-24 |o*| + 2**-140.

Folded LayerNorm: out = rstd (x W'^T - mean cs) + (W beta + b), W' = fp16(W diag(gamma)), cs the colsum of W' split into
fp16 hi/lo, mean split likewise (ln_finalize_kernel, csrc/ap_norm.cu). With xc = x - mu*, r* = rstd*, n = K:
  T_w     r* 2**-11 (|xc| |W'|^T)                      fp16 rounding of W diag(gamma) (the mean term uses the same W')
  T_acc   (ceil((K+8)/16) + 2) 2**-22 r* (|x| |W'|^T + 2 |mu*| |cs|)     E_acc of the extended GEMM
  T_mean  r* |cs| (d_mu + 3 2**-22 |mu*| + 2**-24)     fp32 row sum of the producer's partials
                                                       (d_mu = n 2**-24 mean|x| + 2**-23 |mu*|), the dropped parts of the
                                                       two hi/lo splits and the dropped lo x lo product
  T_rstd  |o* - bias*| (d_var / (2 (var + eps)) + 2**-21)   d_var = (n 2**-24 + 2**-22)(mu*^2 + var) + 2 |mu*| d_mu
                                                       + 2**-24 var: the E[x^2] - mean^2 cancellation of
                                                       ln_finalize_kernel, which grows with (mu / sigma)^2; 2**-21 for
                                                       rsqrtf and the roundings of Q / n and the fma
  T_bias  n 2**-24 (|W| |beta| + |b|)                  the fp32 fold of beta W^T + b
then the epilogue fma (2**-24 |o*|), GEGLU as above on the de-interleaved pre-activations, and the fp16 output.

Statistics: a sum of n fp32 terms in any order is within (n - 1) 2**-24 sum|terms| of the exact sum (fmaf chains for
the sums of squares likewise, n 2**-24 sum x^2).

Emulation
---------
`emulate_gemm` / `emulate_conv` reproduce the kernel's arithmetic in fp32 torch on any device: accumulation per 64-wide
k-block in the order of its four 16-wide steps (tap-major, then source 1, then source 2, for the conv), then the
epilogue in the kernel's order and a single fp16 rounding. Their activations use torch's erfc / sigmoid, not the
kernel's polynomial. `bug=` turns them into models of specific kernel bugs, which the checks must reject.
"""
from __future__ import annotations

import math

import torch

UNITS = 1 << 22                 # exact-grid budget: every partial sum below 2**22 units is exact in fp32
ACC_STEP = 2.0 ** -22           # per-k16-step accumulator allowance
OUT_REL = 2.0 ** -11            # fp16 output: half an ulp, normal
W16_REL = 2.0 ** -11            # fp16 rounding of a weight
OUT_FLOOR = 2.0 ** -25          # fp16 output: half an ulp, subnormal
E24 = 2.0 ** -24
GELU_POLY_REL = 2.0 ** -14
SECOND_ORDER = 1.0 + 2.0 ** -10
BM = 128


class Ref:
    def __init__(self, o, bound, locate, exact=False, out_f32=False, pre=None):
        self.o, self.bound, self.locate, self.exact, self.out_f32 = o, bound, locate, exact, out_f32
        self.pre = bound if pre is None else pre      # bound before the final fp16 rounding


def _fmt(ref, out, r, c):
    return (f"element (row {r}, col {c}) = {ref.locate(r, c)}: out {out[r, c].item():.8g}, "
            f"ref {ref.o[r, c].item():.8g}, bound {ref.bound[r, c].item():.3g}")


def worst(out: torch.Tensor, ref: Ref):
    """(largest |out - o*| / bound, (row, col) of that element); NaN / inf outputs count as inf."""
    assert out.shape == ref.o.shape, (tuple(out.shape), tuple(ref.o.shape))
    ratio = (out.double() - ref.o).abs() / ref.bound
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    i = int(ratio.argmax())
    r, c = divmod(i, ratio.shape[1])
    return ratio.reshape(-1)[i].item(), (r, c)


def check(out: torch.Tensor, ref: Ref, what: str = "") -> float:
    """Bounded check: every element within its bound. Returns the worst ratio of error to bound."""
    ratio, (r, c) = worst(out, ref)
    if not ratio <= 1.0:
        raise AssertionError(f"{what}: ratio {ratio:.3g} at {_fmt(ref, out, r, c)}")
    return ratio


def check_exact(out: torch.Tensor, ref: Ref, what: str = ""):
    """Exact-grid check: out must equal o* rounded once to the output type (fp32: o* itself)."""
    assert ref.exact, f"{what}: the exact-grid check does not apply to this case"
    want = ref.o.to(torch.float32 if ref.out_f32 else torch.float16).double()
    bad = out.double() != want
    n = int(bad.sum())
    if n:
        i = int(bad.reshape(-1).nonzero()[0])
        r, c = divmod(i, out.shape[1])
        raise AssertionError(f"{what}: {n} of {out.numel()} elements differ from the exactly rounded result; first "
                             f"{_fmt(ref, out, r, c)}, expected {want[r, c].item():.8g}")


def headroom(y32: torch.Tensor, ref: Ref) -> float:
    """Largest |y - o*| / pre over the UNROUNDED fp32 values of an emulation: how much of the derived bound, before the
    output rounding, a correct implementation uses."""
    r = (y32.double() - ref.o).abs() / ref.pre
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf).max().item()


def check_both(out, ref, what=""):
    if ref.exact:
        check_exact(out, ref, what)
    return check(out, ref, what)


# ---------------------------------------------------------------------------------------------------- operands
def grid_operands(K: int, e: int = 0, bias_units: int = 1 << 12, res_units: int = 1 << 10, i_max: int = 4,
                  j_max: int = 32):
    """Generators of exact-grid operands for a K-deep product; asserts the 2**22-unit budget first. Returns
    (make_a(shape, g), make_w(shape, g), make_bias(shape, g), make_res(shape, g)); a and w are fp16 on the CPU, bias fp32."""
    need = K * i_max * j_max + bias_units + res_units
    assert need <= UNITS, f"exact grid: K max|i j| + |bias| + |residual| = {need} units > 2**22: sums may round"
    u = 2.0 ** -(7 + e)
    # every grid value must be an fp16 number: w down to 2**-(e+5) and the residual's r u (|r| <= 2**11) down to u
    assert 7 + e <= 24 and res_units <= 1 << 11 and j_max <= 1 << 11 and i_max <= 1 << 11, \
        "exact grid: operands not representable in fp16"

    def ints(shape, lim, g):
        return torch.randint(-lim, lim + 1, shape, generator=g).double()

    return (lambda shape, g: (ints(shape, i_max, g) / 4).half(),
            lambda shape, g: (ints(shape, j_max, g) * 2.0 ** -e / 32).half(),
            lambda shape, g: (ints(shape, bias_units, g) * u).float(),
            lambda shape, g: (ints(shape, res_units, g) * u).half())


def gauss_operands(K: int):
    """Gaussian operands at realistic scale: a ~ N(0, 1), w ~ N(0, 1/K), bias / residual ~ N(0, 1)."""
    return (lambda shape, g: torch.randn(shape, generator=g).half(),
            lambda shape, g: (torch.randn(shape, generator=g) * K ** -0.5).half(),
            lambda shape, g: torch.randn(shape, generator=g).float(),
            lambda shape, g: torch.randn(shape, generator=g).half())


# ---------------------------------------------------------------------------------------------------- epilogue
_SQRT1_2 = 1.0 / math.sqrt(2.0)


def _phi(y):
    return torch.exp(-0.5 * y * y) / math.sqrt(2 * math.pi)


def _Phi(y):
    return 0.5 * torch.erfc(-y * _SQRT1_2)


def _gelu(y):
    return y * _Phi(y)


def _gelu_d(y):
    return _Phi(y) + y * _phi(y)


def _gelu_err(y):
    t = y.abs() * _Phi(-y.abs())
    return t * (GELU_POLY_REL + 2.0 ** -22 + (y * y + 8) * 2.0 ** -23) + 2.0 ** -23 * _gelu(y).abs() + 2.0 ** -26


def _qgelu(y):
    return y * torch.sigmoid(1.702 * y)


def _qgelu_d(y):
    s = torch.sigmoid(1.702 * y)
    return s + 1.702 * y * s * (1 - s)


def geglu_index(n_acc: int, device):
    """Accumulator columns of the value / gate of each GEGLU output (ops.interleave_geglu: blocks of 16)."""
    j = torch.arange(n_acc // 2, device=device)
    v = (j // 16) * 32 + j % 16
    return v, v + 16


def _bias_rows(bias, M, group, device):
    if bias is None:
        return None
    if bias.dim() == 1:
        return bias.double()[None, :].expand(M, -1)
    g = group if group and group > 0 else M
    return bias.double()[torch.arange(M, device=device) // g]


def _epilogue(acc, e_acc, b, res, act, n_valid, out_f32):
    """fp64 epilogue on the exact accumulator acc with its error bound e_acc; returns (o*, bound, pre-rounding bound)."""
    if b is not None:
        y = acc + b
        e_y = e_acc + E24 * (acc.abs() + b.abs())
    else:
        y, e_y = acc, e_acc
    if act is None:
        o, e = y, e_y
        if res is not None:
            o = y + res
            e = e_y + E24 * (y.abs() + res.abs())
    elif act == "gelu":
        o = _gelu(y)
        e = (_gelu_d(y).abs() + e_y) * e_y + _gelu_err(y)
    elif act == "quick_gelu":
        o = _qgelu(y)
        e = (_qgelu_d(y).abs() + e_y) * e_y + o.abs() * (2.0 ** -20 + 4 * y.abs() * E24) + 2.0 ** -26
    elif act == "geglu":
        vi, gi = geglu_index(y.shape[1], y.device)
        v, g, ev, eg = y[:, vi], y[:, gi], e_y[:, vi], e_y[:, gi]
        o = v * _gelu(g)
        e = (_gelu(g).abs() * ev + (v.abs() + ev) * (_gelu_d(g).abs() + eg) * eg + v.abs() * _gelu_err(g)
             + E24 * o.abs())
    else:
        raise ValueError(act)
    if n_valid:
        o, e = o[:, :n_valid], e[:, :n_valid]
    e = e * SECOND_ORDER
    if out_f32:
        e = e + E24 * o.abs() + 2.0 ** -140
        return o, e, e
    return o, e + OUT_REL * o.abs() + OUT_FLOOR, e


def _acc_bound(K, sabs):
    return (math.ceil(K / 16) + 2) * ACC_STEP * sabs


def gemm_locate(bn, geglu=False):
    w = bn // 2 if geglu else bn

    def loc(r, c):
        return dict(m_tile=r // BM, n_tile=c // w, box=(r % BM) // 32, chunk=(c % w) // 32)
    return loc


def gemm_ref(a, w, a2=None, bias=None, bias_group_rows=0, residual=None, act=None, n_valid=0, out_f32=False, bn=0,
             exact=False) -> Ref:
    """ap_gemm_f16's contract (see the module docstring). bias: fp32 [N] or a [groups, N] view (any row stride);
    residual: fp16 [M, >= n] view. exact: the operands are on the exact grid (linear epilogues only)."""
    A = a.double() if a2 is None else torch.cat([a.double(), a2.double()], 1)
    W = w.double()
    M, K = A.shape
    acc = A @ W.t()
    e_acc = _acc_bound(K, A.abs() @ W.abs().t())
    b = _bias_rows(bias, M, bias_group_rows, A.device)
    nout = w.shape[0] // 2 if act == "geglu" else w.shape[0]
    n = n_valid or nout
    res = residual[:, :n].double() if residual is not None else None
    if res is not None and n < nout:
        res = torch.cat([res, res.new_zeros(M, nout - n)], 1)
    o, bound, pre = _epilogue(acc, e_acc, b, res, act, n, out_f32)
    return Ref(o, bound, gemm_locate(bn or 128, act == "geglu"), exact=exact and act is None, out_f32=out_f32, pre=pre)


def conv_taps(x, stride):
    """The nine shifted views of x [Nf, H, W, C] (fp64, zero padded by 1) that tap (ky, kx) multiplies, each
    [Nf*Ho*Wo, C]."""
    nf, h, wd, c = x.shape
    ho, wo = h // stride, wd // stride
    xp = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))
    taps = []
    for ky in range(3):
        for kx in range(3):
            v = xp[:, ky:ky + stride * (ho - 1) + 1:stride, kx:kx + stride * (wo - 1) + 1:stride, :]
            taps.append(v.reshape(nf * ho * wo, c))
    return taps


def conv_locate(ho, wo):
    def loc(r, c):
        return dict(frame=r // (ho * wo), y=(r // wo) % ho, x=r % wo, channel=c)
    return loc


def conv_ref(x, w_packed, cout, x2=None, stride=1, bias=None, bias_group_rows=0, residual=None, exact=False) -> Ref:
    """ap_conv3x3_nhwc_f16's contract: sum over the nine taps of shifted([x | x2]) @ w_tap.T, then the GEMM epilogue.
    w_packed [Cout_p, 9 (C1 + C2)] tap-major / channel-minor (ops.pack_conv3x3_weight); out / residual [Nf, Ho, Wo, cout]."""
    nf, h, wd, c1 = x.shape
    c2 = x2.shape[3] if x2 is not None else 0
    ct = c1 + c2
    ho, wo = h // stride, wd // stride
    W = w_packed.double()
    t1 = conv_taps(x, stride)
    t2 = conv_taps(x2, stride) if x2 is not None else None
    M = nf * ho * wo
    acc = torch.zeros(M, W.shape[0], dtype=torch.float64, device=x.device)
    sabs = torch.zeros_like(acc)
    for t in range(9):
        wt = W[:, t * ct:(t + 1) * ct]
        a = t1[t] if t2 is None else torch.cat([t1[t], t2[t]], 1)
        acc += a @ wt.t()
        sabs += a.abs() @ wt.abs().t()
    e_acc = _acc_bound(9 * ct, sabs)
    b = _bias_rows(bias, M, bias_group_rows, x.device)
    res = residual.reshape(M, cout).double() if residual is not None else None
    if res is not None and cout < W.shape[0]:
        res = torch.cat([res, res.new_zeros(M, W.shape[0] - cout)], 1)
    o, bound, pre = _epilogue(acc, e_acc, b, res, None, cout, False)
    return Ref(o, bound, conv_locate(ho, wo), exact=exact, pre=pre)


def ln_fold_ref(x, w, b, gamma, beta, eps, wg, act=None, bn=0, bias_group_rows=0) -> Ref:
    """LayerNorm(x) (fp64, biased variance) followed by x_n W^T + b with the original fp32 W [N, K], b, gamma, beta;
    act None or 'geglu' (then W, b are in the interleaved layout of ops.interleave_geglu). wg: the folded fp16 weights
    actually used ([N, K + 8]), for the size of the fp16 rounding of W diag(gamma). b may be a [groups, N] table
    (row m uses b[m // bias_group_rows]: the temporal blocks' per-frame positional-encoding bias)."""
    X = x.double()
    M, K = X.shape
    W, g64, be = w.double(), gamma.double(), beta.double()
    b64 = _bias_rows(b, M, bias_group_rows, X.device) if b is not None else None
    mu = X.mean(1, keepdim=True)
    var = ((X - mu) ** 2).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    xc = X - mu
    bias = (W @ be)[None, :] + (b64 if b64 is not None else 0.0)
    acc = r * (xc @ (W * g64[None, :]).t())
    y = acc + bias
    Wp = wg[:, :K].double().abs()
    cs = wg[:, :K].double().sum(1).abs()[None, :]
    n = K
    d_mu = n * E24 * X.abs().mean(1, keepdim=True) + 2.0 ** -23 * mu.abs()
    d_var = (n * E24 + 2.0 ** -22) * (mu * mu + var) + 2 * mu.abs() * d_mu + E24 * var
    t_w = r * W16_REL * (xc.abs() @ Wp.t())
    t_acc = (math.ceil((K + 8) / 16) + 2) * ACC_STEP * r * (X.abs() @ Wp.t() + 2 * mu.abs() * cs)
    t_mean = r * cs * (d_mu + 3 * 2.0 ** -22 * mu.abs() + E24)
    t_rstd = acc.abs() * (d_var / (2 * (var + eps)) + 2.0 ** -21)
    t_bias = n * E24 * ((W.abs() @ be.abs())[None, :] + (b64.abs() if b64 is not None else 0.0))
    e_y = t_w + t_acc + t_mean + t_rstd + t_bias + E24 * (acc.abs() + bias.abs())
    o, bound, pre = _epilogue(y, e_y, None, None, act, 0, False)
    return Ref(o, bound, gemm_locate(bn or 128, act == "geglu"), pre=pre)


# ---------------------------------------------------------------------------------------------------- statistics
def row_stat_parts(out: torch.Tensor, bn: int) -> torch.Tensor:
    """Which row-statistics part covers each output column: part = 2 * n_tile + (32-column chunk parity)."""
    c = torch.arange(out.shape[1], device=out.device)
    return 2 * (c // bn) + (c % bn) // 32 % 2


def row_stats_ref(out: torch.Tensor, bn: int, parts: int):
    """fp64 {sum, sumsq} of the STORED fp16 output per (part, row) and their fp32 summation bounds: [parts, M, 2] each."""
    o = out.double()
    M, N = o.shape
    pidx = row_stat_parts(out, bn)
    s = torch.zeros(parts, M, 2, dtype=torch.float64, device=o.device)
    bnd = torch.zeros_like(s)
    for p in range(parts):
        cols = (pidx == p).nonzero().flatten()
        if cols.numel() == 0:
            continue
        v = o[:, cols]
        n = cols.numel()
        s[p, :, 0] = v.sum(1)
        s[p, :, 1] = (v * v).sum(1)
        bnd[p, :, 0] = n * E24 * v.abs().sum(1)
        bnd[p, :, 1] = n * E24 * (v * v).sum(1)
    return s, bnd


def gemm_box_rows(M: int, m_tiles: int, device):
    """Output rows of every 32-row box of a plain GEMM, [4 * m_tiles, 32] (-1 past M)."""
    r = torch.arange(4 * m_tiles * 32, device=device).view(-1, 32)
    return torch.where(r < M, r, torch.full_like(r, -1))


def _pow2_div(v, cap):
    d = 1
    while d * 2 <= cap and v % (d * 2) == 0:
        d *= 2
    return d


def conv_box_rows(nf: int, ho: int, wo: int, device):
    """Output rows (n Ho + y) Wo + x of every 32-row sub-box of the conv's tiles, [4 * m_tiles, 32] (-1 outside the
    grid): the tile box is bw x bh x bn output pixels (bw | Wo, bh | Ho powers of two, 128 pixels), row r of the tile at
    (frame r / (bh bw), y (r / bw) % bh, x r % bw) from its origin, as the kernel's epilogue addresses it."""
    bw = _pow2_div(wo, 128)
    bh = _pow2_div(ho, 128 // bw)
    bnf = 128 // (bw * bh)
    tx, ty = wo // bw, ho // bh
    mt = ((nf + bnf - 1) // bnf) * tx * ty
    t = torch.arange(mt, device=device)[:, None]
    r = torch.arange(128, device=device)[None, :]
    tn, rem = t // (tx * ty), t % (tx * ty)
    n = tn * bnf + r // (bh * bw)
    y = (rem // tx) * bh + (r // bw) % bh
    x = (rem % tx) * bw + r % bw
    ok = (n < nf) & (y < ho) & (x < wo)
    rows = torch.where(ok, (n * ho + y) * wo + x, torch.full_like(n, -1))
    return rows.view(4 * mt, 32)


def col_stats_ref(out: torch.Tensor, box_rows: torch.Tensor):
    """fp64 {sum, sumsq} per (32-row box, column) of the stored output and their bounds: [boxes, N, 2] each."""
    o = torch.cat([out.double(), out.new_zeros(1, out.shape[1]).double()], 0)      # row -1 -> zeros
    v = o[box_rows]                                                                  # [boxes, 32, N]
    s = torch.stack([v.sum(1), (v * v).sum(1)], -1)
    bnd = torch.stack([32 * E24 * v.abs().sum(1), 32 * E24 * (v * v).sum(1)], -1)
    return s, bnd


def check_stats(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """Per-entry check of statistics partials; entries whose exact value is 0 with no terms must be exactly 0."""
    err = (got.double() - want).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    i = int(ratio.argmax())
    worst_r = ratio.reshape(-1)[i].item()
    if not worst_r <= 1.0:
        idx = list(torch.unravel_index(torch.tensor(i), ratio.shape))
        raise AssertionError(f"{what}: statistics entry {[int(t) for t in idx]}: got {got.reshape(-1)[i].item():.8g}, "
                             f"want {want.reshape(-1)[i].item():.8g}, bound {bound.reshape(-1)[i].item():.3g}")
    return worst_r


def group_norm_ref(x: torch.Tensor, gamma, beta, groups: int, eps: float, silu: bool, stat_terms: int = 32) -> Ref:
    """fp64 GroupNorm (+ SiLU) of channels-last x [Nf, HW, C] against ops.group_norm fed with column statistics.
    Bound: the partials are fp32 sums of stat_terms values (d_S <= stat_terms 2**-24 sum|x|, same for sum x^2); the
    per-group combination is in double; mean and rstd are rounded to fp32 (2**-24 each); the apply computes
    a = rstd gamma, b = beta - mean a, v = x a + b in fp32 (two roundings per product / sum, relative to the terms'
    magnitudes: 4 2**-24 (|x a| + |mean a| + |beta|)); SiLU by ex2 / rcp (2**-20 relative, derivative <= 1.1);
    the fp16 output."""
    nf, hw, c = x.shape
    X = x.double().view(nf, hw, groups, c // groups)
    n = hw * (c // groups)
    mu = X.mean((1, 3), keepdim=True)
    var = ((X - mu) ** 2).mean((1, 3), keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    d_mu = stat_terms * E24 * X.abs().mean((1, 3), keepdim=True) + E24 * mu.abs()
    d_var = stat_terms * E24 * (X * X).mean((1, 3), keepdim=True) + 2 * mu.abs() * d_mu
    d_r = r * (d_var / (2 * (var + eps)) + 2 * E24)
    g = gamma.double().view(1, 1, groups, -1)
    be = beta.double().view(1, 1, groups, -1)
    xc = X - mu
    v = xc * r * g + be
    e_v = (xc.abs() * d_r + r * d_mu) * g.abs() + 4 * E24 * ((X * r * g).abs() + (mu * r * g).abs() + be.abs())
    if silu:
        o = v * torch.sigmoid(v)
        e = 1.1 * e_v + o.abs() * 2.0 ** -20 + 2.0 ** -26
    else:
        o, e = v, e_v
    o, e = o.reshape(nf * hw, c), e.reshape(nf * hw, c) * SECOND_ORDER
    return Ref(o, e + OUT_REL * o.abs() + OUT_FLOOR, lambda rr, cc: dict(frame=rr // hw, row=rr % hw, channel=cc), pre=e)


# ---------------------------------------------------------------------------------------------------- emulation
def _mm_steps(A32: torch.Tensor, W32: torch.Tensor) -> torch.Tensor:
    """fp32 accumulation in the kernel's order: 64-wide k-blocks, each as four 16-wide steps."""
    acc = torch.zeros(A32.shape[0], W32.shape[0], dtype=torch.float32, device=A32.device)
    for k in range(0, A32.shape[1], 16):
        acc = acc + A32[:, k:k + 16] @ W32[:, k:k + 16].t()
    return acc


def _pad64(t: torch.Tensor) -> torch.Tensor:
    k = t.shape[1]
    kp = (k + 63) // 64 * 64
    return t if kp == k else torch.cat([t, t.new_zeros(t.shape[0], kp - k)], 1)


def _gelu32(y):
    """GELU in the kernel's form, max(y, 0) - |y| Phi(-|y|): no cancellation for y << 0 (torch's 1 + erf(y / sqrt 2)
    loses every digit there)."""
    return y.clamp_min(0) - y.abs() * (0.5 * torch.erfc(y.abs() * _SQRT1_2))


def _epi32(acc, bias_rows, res, act, ln_rstd=None):
    y = acc if ln_rstd is None else acc * ln_rstd[:, None]
    if bias_rows is not None:
        y = y + bias_rows
    if act == "gelu":
        return _gelu32(y)
    if act == "quick_gelu":
        return y * torch.sigmoid(1.702 * y)
    if act == "geglu":
        vi, gi = geglu_index(y.shape[1], y.device)
        return y[:, vi] * _gelu32(y[:, gi])
    if res is not None:
        y = y + res
    return y


def emulate_gemm(a, w, a2=None, bias=None, bias_group_rows=0, residual=None, act=None, n_valid=0, out_f32=False,
                 bn=128, ln_rstd=None, bug=None, out=None, unrounded=False):
    """The kernel in fp32 (module docstring), writing into `out` (a [M, n_valid] view of a guarded buffer) when given.
    Bugs: 'm_tail' (the last partial 128-row tile is not written), 'res_box' (residual read one 32-row box down),
    'bias_tile' (bias group from the tile's first row), 'bias_ld' (bias rows read with stride N instead of the table's),
    'src2_kb' (source-2 k-blocks read one block later), 'bn160_chunk' (the 5th 32-column chunk of each 160-wide tile is
    not written), 'geglu_swap' (value and gate swapped), 'ln_row' (folded-LN rstd of the next row), 'n_valid' (columns
    >= n_valid written too), 'stats_clipped' (row statistics include the clipped columns: see emulate_row_stats).
    unrounded: return the fp32 values the epilogue rounds, [M, n_valid], instead of writing the output."""
    M = a.shape[0]
    k1 = a.shape[1]
    A = _pad64(a.float())
    if a2 is not None:
        a2f = a2.float()
        if bug == "src2_kb":
            a2f = torch.cat([a2f[:, 64:], a2f.new_zeros(M, min(64, a2f.shape[1]))], 1)
        A = torch.cat([A, _pad64(a2f)], 1)
    Wf = w.float()
    Wp = torch.zeros(Wf.shape[0], A.shape[1], device=w.device)
    kp1 = (k1 + 63) // 64 * 64
    Wp[:, :k1] = Wf[:, :k1]
    if a2 is not None:
        Wp[:, kp1:kp1 + a2.shape[1]] = Wf[:, k1:]
    acc = _mm_steps(A, Wp)
    N = w.shape[0]
    brows = None
    if bias is not None:
        if bias.dim() == 1:
            brows = bias.float()[None, :].expand(M, -1)
        else:
            tab = bias
            if bug == "bias_ld":
                tab = torch.as_strided(bias, bias.shape, (N, 1))
            g = bias_group_rows if bias_group_rows > 0 else M
            m = torch.arange(M, device=a.device)
            if bug == "bias_tile":
                m = m // BM * BM
            brows = tab.float()[m // g]
    res = None
    nout = N // 2 if act == "geglu" else N
    nv = n_valid or nout
    if residual is not None:
        rsrc = residual
        if bug == "res_box":
            rsrc = torch.cat([residual[32:], residual[:32]], 0)
        res = torch.zeros(M, N, device=a.device)
        res[:, :nv] = rsrc[:, :nv].float()
    rstd = None
    if ln_rstd is not None:
        rstd = ln_rstd.float()
        if bug == "ln_row":
            rstd = torch.cat([rstd[1:], rstd[-1:]])
    if bug == "geglu_swap":
        vi, gi = geglu_index(N, w.device)
        perm = torch.arange(N, device=w.device)
        perm[vi], perm[gi] = gi, vi
        acc = acc[:, perm]
        if brows is not None:
            brows = brows[:, perm]
    y = _epi32(acc, brows, res, act, rstd)
    if unrounded:
        return y[:, :nv]
    y = y if out_f32 else y.half()
    ncols = nout if bug == "n_valid" else nv
    rows = M
    if bug == "m_tail" and M % BM:
        rows = M // BM * BM
    if out is None:
        out = torch.zeros(M, nv, dtype=y.dtype, device=a.device)
    if bug == "n_valid":
        wide = torch.as_strided(out, (M, ncols), out.stride())
        wide[:rows] = y[:rows, :ncols]
    else:
        out[:rows] = y[:rows, :nv]
    if bug == "bn160_chunk" and bn == 160:
        c = torch.arange(nv, device=a.device)
        drop = (c % 160) // 32 == 4
        out[:, drop] = 0
    return out


def emulate_row_stats(out_full: torch.Tensor, bn: int, parts: int, nv: int, bug=None) -> torch.Tensor:
    """fp32 row partials [parts, M, 2] as the epilogue forms them from the fp16 values it rounds. `out_full` holds every
    computed column (including any past n_valid); bug='stats_clipped' keeps the clipped columns in the sums."""
    o = out_full.float() if bug == "stats_clipped" else out_full[:, :nv].float()
    pidx = row_stat_parts(o, bn)
    st = torch.zeros(parts, o.shape[0], 2, device=o.device)
    for p in range(parts):
        cols = (pidx == p).nonzero().flatten()
        if cols.numel():
            v = o[:, cols]
            st[p, :, 0] = v.sum(1)
            st[p, :, 1] = (v * v).sum(1)
    return st


def emulate_conv(x, w_packed, cout, x2=None, stride=1, bias=None, bias_group_rows=0, residual=None, bug=None,
                 unrounded=False):
    """The conv kernel in fp32: an im2col operand assembled in the kernel's K order (tap-major, then source 1, then
    source 2), stride-2 taps read through the (phase_x * C + c, W/2, phase_y, H/2, Nf) view of each source. bug='phase_c1'
    addresses source 2's odd x-phase at C1 + c instead of C2 + c (the defect this suite was written against)."""
    nf, h, wd, c1 = x.shape
    c2 = x2.shape[3] if x2 is not None else 0
    ho, wo = h // stride, wd // stride
    M = nf * ho * wo

    def gather(src, c_phase, ky, kx):
        C = src.shape[3]
        if stride == 1:
            return conv_taps(src, 1)[3 * ky + kx].float()
        # input pixel 2 o + k - 1: k = 0 -> (o - 1, phase 1), k = 1 -> (o, phase 0), k = 2 -> (o, phase 1)
        px, dx = (0, 0) if kx == 1 else (1, -1 if kx == 0 else 0)
        py, dy = (0, 0) if ky == 1 else (1, -1 if ky == 0 else 0)
        merged = src.float().view(nf, h // 2, 2, wd // 2, 2 * C)            # (n, y/2, phase_y, x/2, phase_x C + c)
        pad = torch.zeros(nf, h // 2 + 1, 2, wd // 2 + 1, 2 * C + 64, device=src.device)
        pad[:, 1:, :, 1:, :2 * C] = merged
        v = pad[:, 1 + dy:1 + dy + ho, py, 1 + dx:1 + dx + wo, px * c_phase:px * c_phase + C]
        return v.reshape(M, C)

    cols = []
    for ky in range(3):
        for kx in range(3):
            cols.append(gather(x, c1, ky, kx))
            if x2 is not None:
                cols.append(gather(x2, c1 if bug == "phase_c1" else c2, ky, kx))
    A = torch.cat(cols, 1)
    acc = _mm_steps(A, w_packed.float())
    brows = None
    if bias is not None:
        brows = _bias_rows(bias, M, bias_group_rows, x.device).float()
    res = None
    if residual is not None:
        res = torch.zeros(M, w_packed.shape[0], device=x.device)
        res[:, :cout] = residual.reshape(M, cout).float()
    y = _epi32(acc, brows, res, None)[:, :cout]
    return y if unrounded else y.half()


# ---------------------------------------------------------------------------------------------------- guard band
F16_SENTINEL = -2049       # int16 bits 0xF7FF: -32752 in fp16 (no kernel output of these tests reaches it)
F32_SENTINEL = -1048577    # int32 bits 0xFFEFFFFF: a negative NaN payload


class Guarded:
    """An output view [rows, cols] with row stride ld inside a flat allocation that starts `pre` elements before it and
    ends `post_rows` rows after it; every element outside the view holds a sentinel bit pattern."""

    def __init__(self, rows, cols, ld, dtype, device, pre=64, post_rows=3):
        self.rows, self.cols, self.ld, self.pre = rows, cols, ld, pre
        total = pre + (rows + post_rows) * ld
        it = torch.int16 if dtype == torch.float16 else torch.int32
        self.bits = torch.full((total,), F16_SENTINEL if dtype == torch.float16 else F32_SENTINEL, dtype=it,
                               device=device)
        self.flat = self.bits.view(dtype)
        self.view = torch.as_strided(self.flat, (rows, cols), (ld, 1), pre)
        self.mask = torch.zeros(total, dtype=torch.bool, device=device)
        torch.as_strided(self.mask, (rows, cols), (ld, 1), pre).fill_(True)
        self.sentinel = self.bits[0].item()

    def check(self, what=""):
        bad = (~self.mask) & (self.bits != self.sentinel)
        n = int(bad.sum())
        if n:
            i = int(bad.nonzero()[0]) - self.pre
            raise AssertionError(f"{what}: {n} elements outside the output were written; first at offset {i} "
                                 f"(row {i // self.ld}, column {i % self.ld}; output is {self.rows} x {self.cols}, "
                                 f"ld {self.ld})")


# ---------------------------------------------------------------------------------------------------- case table
def gemm_case(name, M, N, K1, K2=0, bn=0, bias=None, gr=0, res=False, lda_pad=0, ldo_pad=0, ldr_pad=0, act=None,
              out_f32=False, n_valid=0, pre=64, res_off=0):
    """One ap_gemm_f16 call shape. bias: None | 'row' | 'group' (gr rows per bias row) | 'slice' (a column slice
    [groups, N] at column N of a [groups, 3N] table, gr rows per group). pre: elements of guard band before the output
    (64 keeps it 16-byte aligned; an odd value makes every output row start off the 16-byte grid). res_off: the residual's
    base sits res_off elements past the 16-byte grid."""
    return dict(name=name, M=M, N=N, K1=K1, K2=K2, bn=bn, bias=bias, gr=gr, res=res, lda_pad=lda_pad, ldo_pad=ldo_pad,
                ldr_pad=ldr_pad, act=act, out_f32=out_f32, n_valid=n_valid, pre=pre, res_off=res_off)


# The variant matrix: every tile width of the linear epilogue, GEGLU at BN 64 and 128, M and K edges, and each epilogue
# feature alone. Names say what the case exercises.
GEMM_CASES = [
    *[gemm_case(f"bn{bn}_bias_res_m129", 129, 1280, 200, bn=bn, bias="row", res=True) for bn in (32, 64, 128, 160, 256)],
    *[gemm_case(f"bn{bn}_m4101", 4101, 1280, 320, bn=bn, bias="row") for bn in (32, 160, 256)],
    *[gemm_case(f"m{m}", m, 192, 72, bn=64, bias="row", res=True) for m in (1, 31, 33, 127, 129, 514)],
    *[gemm_case(f"k{k}", 257, 320, k, bias="row") for k in (8, 40, 72, 200, 320, 5120)],
    gemm_case("k1280_plus8_src2", 300, 640, 1280, 8, bias="row"),
    gemm_case("two_source_640_320", 514, 640, 640, 320, res=True),
    gemm_case("bias_group_100", 1000, 320, 320, bias="group", gr=100),
    gemm_case("bias_group_72_bn32", 1000, 320, 320, bn=32, bias="group", gr=72, res=True),
    gemm_case("bias_table_slice", 514, 320, 320, bias="slice", gr=100),
    gemm_case("strided_a", 257, 320, 320, lda_pad=24, bias="row"),
    gemm_case("strided_out", 257, 320, 320, ldo_pad=40, bias="row", res=True),
    gemm_case("strided_res_ldr_ne_ldo", 257, 320, 320, ldo_pad=8, ldr_pad=24, res=True),
    gemm_case("gelu", 257, 1024, 320, bias="row", act="gelu"),
    gemm_case("quick_gelu", 257, 1024, 320, bias="row", act="quick_gelu"),
    gemm_case("out_f32", 257, 320, 320, bias="row", out_f32=True),
    gemm_case("out_f32_nvalid", 129, 1408, 1024, bias="row", out_f32=True, n_valid=1404),
    gemm_case("n_valid_301", 257, 320, 320, bias="row", res=True, n_valid=301),
    gemm_case("n_valid_296", 257, 320, 320, bias="row", n_valid=296),
    gemm_case("geglu_bn64", 129, 640, 320, bn=64, bias="row", act="geglu"),
    gemm_case("geglu_bn128_m4101", 4101, 1280, 320, bn=128, bias="row", act="geglu"),
    gemm_case("geglu_nvalid", 257, 640, 320, bias="row", act="geglu", n_valid=300),
    # outputs and residuals that TMA cannot address: the direct-store epilogue with unaligned bases
    gemm_case("direct_out_unaligned", 257, 320, 320, bias="row", res=True, pre=65, ldo_pad=8),
    gemm_case("direct_out_unaligned_gelu", 129, 320, 200, bias="row", act="gelu", pre=67, ldo_pad=8),
    gemm_case("direct_out_unaligned_geglu", 129, 640, 320, bias="row", act="geglu", pre=65, ldo_pad=8),
    gemm_case("direct_res_unaligned", 257, 320, 320, bias="row", res=True, ldr_pad=8, res_off=1),
]
GEMM_LINEAR_NAMES = [c["name"] for c in GEMM_CASES if c["act"] is None]


def build_gemm_case(case, device, grid, seed=0, M=None):
    """Tensors of one case on `device`: returns (call kwargs for ops.gemm without `out`, Guarded output, ref kwargs).
    grid: exact-grid operands (linear cases) or Gaussian ones. Padding columns of A / residual hold NaN."""
    c = dict(case)
    M = M or c["M"]
    N, K1, K2 = c["N"], c["K1"], c["K2"]
    K = K1 + K2
    g = torch.Generator().manual_seed(seed)
    mk_a, mk_w, mk_b, mk_r = grid_operands(K) if grid else gauss_operands(K)
    abig = torch.full((M, K1 + c["lda_pad"]), float("nan"), dtype=torch.float16)
    abig[:, :K1] = mk_a((M, K1), g)
    a = abig.to(device)[:, :K1]
    a2 = mk_a((M, K2), g).to(device) if K2 else None
    w = mk_w((N, K), g).to(device)
    nout = N // 2 if c["act"] == "geglu" else N
    nv = c["n_valid"] or nout
    bias = None
    if c["bias"] == "row":
        bias = mk_b((N,), g).to(device)
    elif c["bias"] in ("group", "slice"):
        groups = (M + c["gr"] - 1) // c["gr"]
        if c["bias"] == "group":
            bias = mk_b((groups, N), g).to(device)
        else:
            bias = mk_b((groups, 3 * N), g).to(device)[:, N:2 * N]
    residual = None
    if c["res"]:
        rbig = torch.full((M, nout + c["ldr_pad"]), float("nan"), dtype=torch.float16)
        rbig[:, :nout] = mk_r((M, nout), g)
        off = c["res_off"]
        flat = torch.full((rbig.numel() + 8,), float("nan"), dtype=torch.float16)
        flat[off:off + rbig.numel()] = rbig.reshape(-1)
        residual = flat.to(device)[off:off + rbig.numel()].view(M, -1)[:, :nout]
    dtype = torch.float32 if c["out_f32"] else torch.float16
    out = Guarded(M, nv, nv + c["ldo_pad"], dtype, device, pre=c["pre"])
    call = dict(bias=bias, residual=residual, a2=a2, bias_group_rows=c["gr"], n_valid=c["n_valid"],
                block_n=c["bn"], out_f32=c["out_f32"], geglu=c["act"] == "geglu", gelu=c["act"] == "gelu",
                quick_gelu=c["act"] == "quick_gelu")
    ref = dict(a2=a2, bias=bias, bias_group_rows=c["gr"], residual=residual, act=c["act"], n_valid=c["n_valid"],
               out_f32=c["out_f32"], bn=c["bn"] or 128, exact=grid)
    return a, w, call, out, ref
