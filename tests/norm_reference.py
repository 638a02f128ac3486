"""fp64 references, per-element bounds and fp32 emulations of the normalisation, small-convolution and elementwise kernels
(csrc/ap_norm.cu, ap_stem.cu, ap_audio.cu, ap_misc.cu). Imported by the CPU checker tests and the GPU contract tests; not
a conftest. The checks themselves (`check`, `check_exact`, `headroom`, `Guarded`) and the GELU error terms are those of
gemm_reference.py; every reference here returns its `Ref` (o*, bound, pre-rounding bound `pre`, `locate`).

Every bound ends with the fp16 output rounding, OUT_REL |o*| + OUT_FLOOR (half an ulp), and multiplies the fp32 part by
SECOND_ORDER (1 + 2**-10) for the products of first-order terms. Below, u = 2**-24 (one fp32 rounding), and a chain of
n fp32 additions in any order is within n u sum|terms| of the exact sum.

GroupNorm, statistics pass (ap_groupnorm_nhwc_f16)
-------------------------------------------------
gn_stats_kernel: a thread adds ceil(rpb / k) rows of its 8 channels, the block adds its k row-lanes in a fixed order,
one thread adds the cpg channels of a group; gn_finalize_kernel adds the chunks in double. Each fp32 partial is thus a
chain of at most stat_terms = ceil(rpb / k) + k + cpg roundings (x**2 of an fp16 value is exact in fp32), and
GR.group_norm_ref(stat_terms=...) bounds the rest (double combine, fp32 mean / rstd, the fp32 apply, SiLU). rpb and k
come from `gn_geometry`, a restatement of gn_launch_geometry; with two sources the larger chain counts. The one-pass
E[x^2] - mean^2 makes d_var grow with (mean / sigma)**2: the bound says how much.

LayerNorm (ap_layernorm_f16: layernormv_kernel<8/16/32>, layernorm_kernel<5/10/20/32>)
-------------------------------------------------------------------------------------
Two-pass fp32 statistics over n = C values. With mu, var the exact mean and biased variance, xc = x - mu:
  d_mu   = n u mean|x| + u |mu|                      the n-term sum and the division by C
  d_var  = (n + 5) u var + 2 d_mu**2                 sum (x - m)**2 with m = mu + delta: sum = n (var + delta**2); each
                                                     term has the rounding of x - m, of its square, and its place in an
                                                     n-term sum, then / C
  d_r    = r (d_var / (2 (var + eps)) + 2**-22 + u)  rsqrtf (<= 2 ulp) and the + eps
  e_v    = |g| (r d_mu + |xc| d_r) + 6 u (|xc r g| + |b| + |pe|)   the five roundings of (x - m) r g + b + pe
A constant row has var = 0, its fp32 mean is exact (n copies of an fp16 value sum exactly) and every x - m is 0: the
output must be exactly fp16(fp32(beta + pe)) (`ln_constant_rows`).

BatchNorm, batch statistics (ap_batchnorm_train_nhwc_f16)
-------------------------------------------------------
bn_stats_kernel is gn_stats_kernel without the group sum: stat_terms = ceil(rpb / k) + k, rpb / k from `bn_geometry`.
bn_finalize_kernel works in double and rounds a = gamma rstd and b = beta - mean a to fp32 once each; bn_apply_kernel
does v = fmaf(x, a, b). With r, d_mu, d_var as for GroupNorm (d_r = r (d_var / (2 (var + eps)) + u)):
  e_v = |a| (|xc| d_r / r + d_mu) + u (|x a| + |beta| + |mu a| + |v|)      (the two fp32 roundings and the fmaf)
then ReLU (1-Lipschitz, exact) or GELU (the csrc/ap_ptx.cuh polynomial: GR's propagated and own-error terms).
Channels with gamma = beta = 0 (the PoseGuider's padding) must be exactly 0.

Direct convolution (ap_conv2d_direct_nhwc_f16)
---------------------------------------------
An fp64 sum of the K*K shifted taps (no cuDNN). The kernel starts from the bias and runs one sequential fmaf chain of
K*K*Cin terms (fp16 x fp16 products are exact in fp32): within (K*K*Cin + 1) u S of o*, S = sum |x w| + |bias|.
Exact-grid operands (GR.grid_operands) keep every partial sum exact, so the only correct output is fp16(o*).

wav2vec2 stem (ap_conv1d_stem_f32)
---------------------------------
out[t, c] = sum_k w[c, k] wave[5 t + k], k < 10: one 10-term fmaf chain, 10 u S. Exact-grid variant as above.

Positional convolution (ap_pos_conv1d_gelu_f16)
----------------------------------------------
out = x + GELU(conv + bias), conv the grouped Conv1d(K, padding K/2) without its last output (SamePad). The mma.sync
accumulator takes 3K k16 steps over 48 channels per tap: (3K + 2) 2**-22 S (GR's per-step allowance), then the bias
add, the GR GELU terms and the residual add (u (|x| + |gelu|)).

Resample (ap_resample_rows_linear_f16)
-------------------------------------
fp64 align_corners=True interpolation at src* = i (T_in - 1) / (T_out - 1). Every fp32 operation of the kernel is
allowed a full ulp (2**-23, twice the rounding), so that the bound keeps a factor 2 of headroom where one rounding
dominates: the fp32 scale and src are within d_s = 2**-22 src* of src*, and the interpolant is continuous and piecewise
linear in src (an i0 that flips at an integer src changes nothing): d_s D, D the larger slope of the two segments around
src*. lambda = src - i0 is exact; 1 - lambda, the two products and the sum add 2**-23 (|a| + |a l0| + |b l1| + |o|). `emulate_resample`
restates the kernel's formula with separate round-to-nearest fp32 operations, as the kernel's __fmul_rn / __fadd_rn do:
on the GPU the kernel must equal it bit for bit. (torch's fp32 F.interpolate is a different formula in the last bit.)

Timestep embedding (ap_timestep_embedding_f16)
---------------------------------------------
o* = [cos(t w_i), sin(t w_i)], w_i = 10000**(-i / half). The exponent -ln(1e4) i / half is formed from the fp32
constant in two roundings (3 u relative), expf is within 2 ulp (2**-22): w has relative error e_w = 3 u e* + 2**-22,
e* = ln(1e4) i / half; the product t w adds u; cosf / sinf are within 2 ulp of the result and 1-Lipschitz:
  pre = |t| w_i (e_w + u) + 2**-22 |o*|.

SiLU (ap_silu_f16)
-----------------
y = v / (1 + __expf(-v)). __expf is documented within 2 + floor(1.173 |v|) ulp; that relative error reaches the
denominator scaled by e / (1 + e) = sigmoid(-v); the + 1 and the IEEE division are allowed a full ulp each (2**-23,
as for the resample: one rounding dominates, and this keeps a factor 2 of headroom); 2**-26 absolute covers the
flush to zero of ex2.approx.ftz. Values whose exp overflows give -0 where |o*| < 2**-100.

Add (ap_add_f16, ap_add_bcast_f16)
---------------------------------
One fp32 add of two fp16 values and one rounding: bit-identical to torch's fp16 a + b (b tiled over the leading dup
dimension for add_bcast).

Emulations
----------
`emulate_*` reproduce each kernel's arithmetic in fp32 torch in the kernel's order. `bug=` turns them into models of
plausible kernel mistakes, which the checks must reject.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import gemm_reference as GR
from gemm_reference import E24, OUT_FLOOR, OUT_REL, SECOND_ORDER, Ref

GN_MAX_BLOCKS = 2368      # AP_GN_MAX_BLOCKS in include/aniportrait_b200.h
BN_MAX_BLOCKS = 2048      # AP_BN_MAX_BLOCKS
LN_WIDE_MAX = 1536        # layernormv_kernel: C % 8 == 0 and C / 8 <= 6 * 32
LN10K = 9.210340371976184  # ln(10000), as the kernel's fp32 constant is written


def _out16(o, pre):
    pre = pre * SECOND_ORDER
    return pre + OUT_REL * o.abs() + OUT_FLOOR, pre


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------- GroupNorm
def gn_geometry(HW: int, C: int, Nf: int, max_blocks: int = GN_MAX_BLOCKS):
    """gn_launch_geometry (csrc/ap_norm.cu): (k row-lanes, rows per block, chunks) of one source of C channels."""
    vecs = C // 8
    k = max(256 // vecs, 1)
    rpb = 8 * k
    while _cdiv(HW, rpb) * Nf > max_blocks and rpb < HW:
        rpb *= 2
    return k, rpb, _cdiv(HW, rpb)


def gn_refused(HW, cs, Nf, max_blocks=GN_MAX_BLOCKS) -> bool:
    """ap_groupnorm_nhwc_f16 refuses when a source's Nf * chunks exceeds the partial-sum workspace."""
    return any(gn_geometry(HW, c, Nf, max_blocks)[2] * Nf > max_blocks for c in cs if c)


def gn_stat_terms(HW, cs, cpg, Nf, max_blocks=GN_MAX_BLOCKS) -> int:
    t = 0
    for c in cs:
        if c:
            k, rpb, _ = gn_geometry(HW, c, Nf, max_blocks)
            t = max(t, _cdiv(rpb, k) + k + cpg)
    return t


def gn_ref(x, x2, gamma, beta, groups, eps, silu, max_blocks=GN_MAX_BLOCKS) -> Ref:
    """x [Nf, HW, C1], x2 [Nf, HW, C2] or None; output [Nf * HW, C1 + C2]."""
    nf, hw, c1 = x.shape
    c2 = x2.shape[2] if x2 is not None else 0
    cpg = (c1 + c2) // groups
    cat = x if x2 is None else torch.cat([x, x2], -1)
    ref = GR.group_norm_ref(cat, gamma, beta, groups, eps, silu,
                            stat_terms=gn_stat_terms(hw, (c1, c2), cpg, nf, max_blocks))
    rpb = [gn_geometry(hw, c, nf, max_blocks)[1] if c else 1 for c in (c1, c2)]

    def loc(r, c):
        s = 0 if c < c1 else 1
        return dict(frame=r // hw, chunk=(r % hw) // rpb[s], row=r % hw, group=c // cpg, source=s, channel=c)
    ref.locate = loc
    return ref


def _chunk_totals(x32, k, rpb, chunks):
    """Per-chunk channel totals {sum, sumsq} in the stats kernels' order: x32 [Nf, HW, C] -> two [Nf, chunks, C]."""
    nf, hw, c = x32.shape
    xp = F.pad(x32, (0, 0, 0, chunks * rpb - hw)).view(nf, chunks, rpb // k, k, c)
    s = torch.zeros(nf, chunks, k, c, dtype=torch.float32, device=x32.device)
    q = torch.zeros_like(s)
    for j in range(rpb // k):            # a thread's rows r0 + rl, r0 + rl + k, ...
        v = xp[:, :, j]
        s = s + v
        q = q + v * v
    ts = torch.zeros(nf, chunks, c, dtype=torch.float32, device=x32.device)
    tq = torch.zeros_like(ts)
    for r in range(k):                   # the fixed-order sum over the block's row-lanes
        ts = ts + s[:, :, r]
        tq = tq + q[:, :, r]
    return ts, tq


def emulate_gn(x, x2, gamma, beta, groups, eps, silu, bug=None, unrounded=False, max_blocks=GN_MAX_BLOCKS):
    """ap_groupnorm_nhwc_f16 in fp32. Bugs: 'drop_last_chunk' (each frame's last chunk of partials is not added),
    'straddle_one_source' (a group that straddles the two sources takes its statistics from source 1 only)."""
    nf, hw, c1 = x.shape
    c2 = x2.shape[2] if x2 is not None else 0
    C = c1 + c2
    cpg = C // groups
    S = torch.zeros(nf, groups, dtype=torch.float64, device=x.device)
    Q = torch.zeros_like(S)
    for src, c_off, cs in ((x, 0, c1), (x2, c1, c2)):
        if not cs:
            continue
        k, rpb, chunks = gn_geometry(hw, cs, nf, max_blocks)
        ts, tq = _chunk_totals(src.float(), k, rpb, chunks)
        if bug == "drop_last_chunk" and chunks > 1:
            ts, tq = ts[:, :-1], tq[:, :-1]
        for g in range(c_off // cpg, (c_off + cs - 1) // cpg + 1):
            lo, hi = max(g * cpg, c_off) - c_off, min((g + 1) * cpg, c_off + cs) - c_off
            if bug == "straddle_one_source" and c_off > 0 and g * cpg < c_off:
                continue
            ps = torch.zeros(nf, ts.shape[1], dtype=torch.float32, device=x.device)
            pq = torch.zeros_like(ps)
            for c in range(lo, hi):
                ps = ps + ts[:, :, c]
                pq = pq + tq[:, :, c]
            S[:, g] += ps.double().sum(1)
            Q[:, g] += pq.double().sum(1)
    n = hw * cpg
    mean = S / n
    var = (Q / n - mean * mean).clamp_min(0)
    m32 = mean.float().repeat_interleave(cpg, 1)[:, None, :]
    r32 = (1.0 / torch.sqrt(var + eps)).float().repeat_interleave(cpg, 1)[:, None, :]
    a = r32 * gamma.float()
    b = beta.float() - m32 * a
    cat = (x if x2 is None else torch.cat([x, x2], -1)).float()
    v = cat * a + b
    if silu:
        v = v * torch.sigmoid(v)
    v = v.reshape(nf * hw, C)
    return v if unrounded else v.half()


# ---------------------------------------------------------------------------------------------------- LayerNorm
def ln_kernel(C: int, narrow: bool = False):
    """('wide', LPR) for layernormv_kernel, ('narrow', MAXV) for layernorm_kernel, as ap_layernorm_f16 dispatches
    (narrow: AP_LAYERNORM_NARROW set)."""
    if C % 8 == 0 and C <= LN_WIDE_MAX and not narrow:
        nvec = C // 8
        return "wide", 8 if nvec <= 48 else (16 if nvec <= 96 else 32)
    maxv = (C // 2 + 31) // 32
    return "narrow", 5 if maxv <= 5 else 10 if maxv <= 10 else 20 if maxv <= 20 else 32


def _pe_rows(rows, pe, rows_per_pe, pe_period, device, bug=None):
    r = torch.arange(rows, device=device)
    idx = r % pe_period if bug == "pe_row" else (r // rows_per_pe) % pe_period
    return pe[idx]


def ln_ref(x, gamma, beta, eps, pe=None, rows_per_pe=1, pe_period=1, narrow=False) -> Ref:
    X = x.double()
    rows, n = X.shape
    mu = X.mean(1, keepdim=True)
    xc = X - mu
    var = (xc * xc).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    g, b = gamma.double()[None], beta.double()[None]
    p = _pe_rows(rows, pe.double(), rows_per_pe, pe_period, x.device) if pe is not None else torch.zeros_like(b)
    o = xc * r * g + b + p
    d_mu = n * E24 * X.abs().mean(1, keepdim=True) + E24 * mu.abs()
    d_var = (n + 5) * E24 * var + 2 * d_mu * d_mu
    d_r = r * (d_var / (2 * (var + eps)) + 2.0 ** -22 + E24)
    e = g.abs() * (r * d_mu + xc.abs() * d_r) + 6 * E24 * ((xc * r * g).abs() + b.abs() + p.abs())
    bound, pre = _out16(o, e)
    kind, par = ln_kernel(n, narrow)

    def loc(rr, cc):
        if kind == "wide":
            return dict(kernel=f"layernormv<{par}>", row=rr, warp_row=rr % (32 // par), lane=(cc // 8) % par,
                        vector=cc // 8, channel=cc)
        return dict(kernel=f"layernorm<{par}>", row=rr, lane=(cc // 2) % 32, half2=cc // 2, channel=cc)
    return Ref(o, bound, loc, pre=pre)


def ln_constant_rows(gamma, beta, pe=None, rows=None, rows_per_pe=1, pe_period=1):
    """The exact output of constant rows: fp16(fp32(beta) + fp32(pe row))."""
    y = beta.float()[None].expand(rows, -1)
    if pe is not None:
        y = y + _pe_rows(rows, pe.float(), rows_per_pe, pe_period, beta.device)
    return y.half()


def _lane_sums(vals, lanes):
    """vals [rows, U, P] fp32: lane l adds units l, l + lanes, ... (P values each, in order), then the xor-shuffle tree."""
    rows, U, P = vals.shape
    s = torch.zeros(rows, lanes, dtype=torch.float32, device=vals.device)
    lane = torch.arange(lanes, device=vals.device)
    for i in range(_cdiv(U, lanes)):
        u = lane + lanes * i
        ok = u < U
        uc = u.clamp(max=U - 1)
        for t in range(P):
            s = s + torch.where(ok[None], vals[:, uc, t], torch.zeros((), device=vals.device))
    o = lanes // 2
    while o:
        s = s + s[:, lane ^ o]
        o //= 2
    return s[:, 0]


def emulate_ln(x, gamma, beta, eps, pe=None, rows_per_pe=1, pe_period=1, narrow=False, bug=None, unrounded=False,
               out=None):
    """ap_layernorm_f16 in fp32, in the order of the kernel it dispatches to. Bugs: 'pe_row' (pe row r % period instead
    of (r // rows_per_pe) % period), 'last_vec' (the row's last 8 channels are neither in the statistics nor stored)."""
    rows, C = x.shape
    kind, par = ln_kernel(C, narrow)
    xf = x.float()
    keep = C - 8 if bug == "last_vec" else C
    xs = xf[:, :keep]

    def sums(pairs):         # per-half2 values -> the row total in the kernel's lane / shuffle order
        if kind == "wide":
            return _lane_sums(pairs.reshape(rows, -1, 4), par)
        return _lane_sums(pairs.reshape(rows, -1, 1), 32)
    mean = sums(xs[:, 0::2] + xs[:, 1::2]) / C
    d = xs - mean[:, None]
    sq = sums(d[:, 0::2] * d[:, 0::2] + d[:, 1::2] * d[:, 1::2])
    rstd = torch.rsqrt(sq / C + eps)
    y = (xf - mean[:, None]) * rstd[:, None] * gamma.float() + beta.float()
    if pe is not None:
        y = y + _pe_rows(rows, pe.float(), rows_per_pe, pe_period, x.device, bug)
    if unrounded:
        return y
    if out is None:
        out = torch.zeros(rows, C, dtype=torch.float16, device=x.device)
    out[:, :keep] = y[:, :keep].half()
    return out


# ---------------------------------------------------------------------------------------------------- BatchNorm
def bn_geometry(rows: int, C: int, max_blocks: int = BN_MAX_BLOCKS):
    """ap_batchnorm_train_nhwc_f16's (k, rows per block, chunks)."""
    k = max(256 // (C // 8), 1)
    rpb = 8 * k
    min_rpb = _cdiv(rows, max_blocks)
    if rpb < min_rpb:
        rpb = _cdiv(min_rpb, k) * k
    return k, rpb, _cdiv(rows, rpb)


def _act_bound(v, e_v, act):
    if act == "gelu":
        return GR._gelu(v), (GR._gelu_d(v).abs() + e_v) * e_v + GR._gelu_err(v)
    if act == "relu":
        return v.clamp_min(0), e_v
    return v, e_v


def bn_ref(x, gamma, beta, eps, act="none") -> Ref:
    """x [rows, C] fp16: per-channel batch statistics over every row (biased variance), then act."""
    X = x.double()
    rows, C = X.shape
    k, rpb, chunks = bn_geometry(rows, C)
    terms = _cdiv(rpb, k) + k
    mu = X.mean(0, keepdim=True)
    xc = X - mu
    var = (xc * xc).mean(0, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    a = gamma.double()[None] * r
    be = beta.double()[None]
    v = xc * a + be
    d_mu = terms * E24 * X.abs().mean(0, keepdim=True) + E24 * mu.abs()
    d_var = terms * E24 * (X * X).mean(0, keepdim=True) + 2 * mu.abs() * d_mu
    d_rr = d_var / (2 * (var + eps)) + E24
    e_v = a.abs() * (xc.abs() * d_rr + d_mu) + E24 * ((X * a).abs() + be.abs() + (mu * a).abs() + v.abs())
    o, e = _act_bound(v, e_v, act)
    bound, pre = _out16(o, e)

    def loc(rr, cc):
        return dict(chunk=rr // rpb, row_lane=(rr % rpb) % k, row=rr, channel=cc, channel_vector=cc // 8)
    return Ref(o, bound, loc, pre=pre)


def emulate_bn(x, gamma, beta, eps, act="none", bug=None, unrounded=False, max_blocks=BN_MAX_BLOCKS):
    """Bugs: 'unbiased' (variance divided by rows - 1), 'drop_last_chunk' (the last chunk's partials are not added)."""
    rows, C = x.shape
    k, rpb, chunks = bn_geometry(rows, C, max_blocks)
    ts, tq = _chunk_totals(x.float()[None], k, rpb, chunks)
    if bug == "drop_last_chunk" and chunks > 1:
        ts, tq = ts[:, :-1], tq[:, :-1]
    s, q = ts[0].double().sum(0), tq[0].double().sum(0)
    mean = s / rows
    var = (q / rows - mean * mean).clamp_min(0)
    if bug == "unbiased":
        var = var * rows / (rows - 1)
    a = gamma.double() / torch.sqrt(var + eps)
    a32, b32 = a.float(), (beta.double() - mean * a).float()
    v = (x.double() * a32.double() + b32.double()).float()            # fmaf: fp16 x fp32 is exact in double
    if act == "relu":
        v = v.clamp_min(0)
    elif act == "gelu":
        v = GR._gelu32(v)
    return v if unrounded else v.half()


# ---------------------------------------------------------------------------------------------------- direct conv
DIRECT_CONV_VARIANTS = [(8, 3, 1, 8), (8, 4, 2, 16), (16, 3, 1, 16), (16, 4, 2, 16), (32, 3, 1, 16), (32, 4, 2, 16)]


def _taps(x, K, stride, pad, ho, wo, shift=0):
    """[(ky, kx, [Nf*Ho*Wo, Cin] view of the input pixel (oy S - pad + ky - shift, ox S - pad + kx - shift))]."""
    P = pad + 1
    xp = F.pad(x, (0, 0, P, P + K, P, P + K))
    out = []
    for ky in range(K):
        for kx in range(K):
            y0, x0 = P - pad - shift + ky, P - pad - shift + kx
            v = xp[:, y0:y0 + stride * (ho - 1) + 1:stride, x0:x0 + stride * (wo - 1) + 1:stride, :]
            out.append((ky, kx, v.reshape(-1, x.shape[3])))
    return out


def direct_out_hw(H, W, K, stride, pad):
    return (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1


def direct_conv_ref(x, w, bias, stride, pad, exact=False) -> Ref:
    """x [Nf, H, W, Cin] fp16, w [Cout, K, K, Cin] fp16, bias fp32 [Cout] or None -> [Nf*Ho*Wo, Cout]."""
    nf, H, W, cin = x.shape
    cout, K = w.shape[0], w.shape[1]
    ho, wo = direct_out_hw(H, W, K, stride, pad)
    acc = torch.zeros(nf * ho * wo, cout, dtype=torch.float64, device=x.device)
    sabs = torch.zeros_like(acc)
    W64 = w.double()
    for ky, kx, v in _taps(x.double(), K, stride, pad, ho, wo):
        acc += v @ W64[:, ky, kx, :].t()
        sabs += v.abs() @ W64[:, ky, kx, :].abs().t()
    if bias is not None:
        acc += bias.double()[None]
        sabs += bias.double().abs()[None]
    bound, pre = _out16(acc, (K * K * cin + 1) * E24 * sabs)
    ct = 8 if (cin, K) == (8, 3) else 16

    def loc(r, c):
        return dict(frame=r // (ho * wo), y=(r // wo) % ho, x=r % wo, block=r // 128, cout_tile=c // ct, channel=c)
    return Ref(acc, bound, loc, exact=exact, pre=pre)


def emulate_direct_conv(x, w, bias, stride, pad, bug=None, unrounded=False):
    """The kernel's sequential fp32 chain (bias, then taps row-major, channels in order). Bugs: 'flip_tap' (the kernel
    rows read bottom-up), 'pad_off' (input pixel oy S - pad - 1 + ky: padding off by one)."""
    nf, H, W, cin = x.shape
    cout, K = w.shape[0], w.shape[1]
    ho, wo = direct_out_hw(H, W, K, stride, pad)
    acc = torch.zeros(nf * ho * wo, cout, dtype=torch.float32, device=x.device)
    if bias is not None:
        acc = acc + bias.float()[None]
    wf = w.float()
    for ky, kx, v in _taps(x.float(), K, stride, pad, ho, wo, shift=1 if bug == "pad_off" else 0):
        wk = wf[:, K - 1 - ky if bug == "flip_tap" else ky, kx, :]
        for ci in range(cin):
            acc = acc + v[:, ci:ci + 1] * wk[None, :, ci]
    return acc if unrounded else acc.half()


# ---------------------------------------------------------------------------------------------------- audio
def stem_frames(samples):
    return (samples - 10) // 5 + 1


def stem_ref(wave, w, exact=False) -> Ref:
    """wave fp32 [S], w fp32 [Cout, 10] -> [T0, Cout]."""
    X = wave.double().unfold(0, 10, 5)
    W = w.double()
    o = X @ W.t()
    bound, pre = _out16(o, 10 * E24 * (X.abs() @ W.abs().t()))
    cout = w.shape[0]
    return Ref(o, bound, lambda r, c: dict(block=r // 16, frame=r, thread=(c % cout) // 2, channel=c), exact=exact,
               pre=pre)


def emulate_stem(wave, w, unrounded=False):
    X = wave.double().unfold(0, 10, 5)
    acc = torch.zeros(X.shape[0], w.shape[0], dtype=torch.float32, device=wave.device)
    for k in range(10):
        acc = (acc.double() + X[:, k:k + 1] * w.double()[None, :, k]).float()    # fmaf (the product is exact in double)
    return acc if unrounded else acc.half()


PC_CPG = 48


def _pos_shifted(x64, K, tap, shift=0):
    T, C = x64.shape
    xp = torch.zeros(T + K + 1, C, dtype=x64.dtype, device=x64.device)
    xp[K // 2 + 1:K // 2 + 1 + T] = x64
    return xp[tap + 1 + shift:tap + 1 + shift + T]


def pos_conv_ref(x, wp, bias) -> Ref:
    """x [T, C] fp16, wp [C, K, 48] fp16 (ops.pack_pos_conv_weight), bias fp32 [C] -> [T, C]."""
    T, C = x.shape
    K = wp.shape[1]
    G = C // PC_CPG
    X = x.double()
    W = wp.double().view(G, PC_CPG, K, PC_CPG)
    acc = torch.zeros(T, G, PC_CPG, dtype=torch.float64, device=x.device)
    sabs = torch.zeros_like(acc)
    for tap in range(K):
        v = _pos_shifted(X, K, tap).view(T, G, PC_CPG)
        wt = W[:, :, tap, :]
        acc += torch.einsum("tgc,goc->tgo", v, wt)
        sabs += torch.einsum("tgc,goc->tgo", v.abs(), wt.abs())
    acc, sabs = acc.reshape(T, C), sabs.reshape(T, C)
    b = bias.double()[None]
    y = acc + b
    e_y = (3 * K + 2) * GR.ACC_STEP * sabs + E24 * (acc.abs() + b.abs())
    gl = GR._gelu(y)
    e_g = (GR._gelu_d(y).abs() + e_y) * e_y + GR._gelu_err(y)
    o = X + gl
    bound, pre = _out16(o, e_g + E24 * (X.abs() + gl.abs()))

    def loc(r, c):
        return dict(t_block=r // 32, row=r, group=c // PC_CPG, warp=(r % 32) // 16 + 2 * ((c % PC_CPG) // 24),
                    channel=c)
    return Ref(o, bound, loc, pre=pre)


def emulate_pos_conv(x, wp, bias, bug=None, unrounded=False):
    """fp32 accumulation per k16 step (tap-major, three 16-channel steps per tap). Bugs: 'trim_side' (the first output
    dropped instead of the last: input row t + tap - K/2 + 1), 'group_offset' (group g reads group g + 1's channels)."""
    T, C = x.shape
    K = wp.shape[1]
    G = C // PC_CPG
    xf = x.float()
    if bug == "group_offset":
        xf = torch.roll(xf.view(T, G, PC_CPG), -1, 1).reshape(T, C)
    W = wp.float().view(G, PC_CPG, K, PC_CPG)
    acc = torch.zeros(G, T, PC_CPG, dtype=torch.float32, device=x.device)
    for tap in range(K):
        v = _pos_shifted(xf, K, tap, 1 if bug == "trim_side" else 0).view(T, G, PC_CPG).transpose(0, 1)
        for ks in range(0, PC_CPG, 16):
            acc = acc + torch.bmm(v[:, :, ks:ks + 16], W[:, :, tap, ks:ks + 16].transpose(1, 2))
    y = acc.transpose(0, 1).reshape(T, C) + bias.float()[None]
    o = x.float() + GR._gelu32(y)
    return o if unrounded else o.half()


def resample_ref(x, t_out) -> Ref:
    """F.interpolate(mode='linear', align_corners=True) along the rows of x [T_in, C] in float64."""
    t_in = x.shape[0]
    X = x.double()
    i = torch.arange(t_out, dtype=torch.float64, device=x.device)
    src = i * ((t_in - 1) / (t_out - 1)) if t_out > 1 else torch.zeros_like(i)
    i0 = src.floor().clamp(max=t_in - 1).long()
    lam = (src - i0)[:, None]
    i1 = torch.where(i0 < t_in - 1, i0 + 1, i0)
    a, b = X[i0], X[i1]
    o = (1 - lam) * a + lam * b
    d = torch.cat([X[1:] - X[:-1], X.new_zeros(1, X.shape[1])], 0).abs()       # d[j] = |x[j+1] - x[j]|
    D = torch.maximum(d[i0], d[(i0 - 1).clamp_min(0)])
    e = 2.0 ** -22 * src[:, None] * D + 2.0 ** -23 * (a.abs() + ((1 - lam) * a).abs() + (lam * b).abs() + o.abs())
    bound, pre = _out16(o, e)
    return Ref(o, bound, lambda r, c: dict(row=r, i0=int(i0[r]), vector=c // 8, channel=c), pre=pre)


def emulate_resample(x, t_out, bug=None, unrounded=False):
    """The kernel's formula in fp32 (module docstring). bug='align_false': the align_corners=False source index."""
    t_in = x.shape[0]
    i = torch.arange(t_out, device=x.device, dtype=torch.float32)
    if bug == "align_false":
        src = ((i + 0.5) * torch.tensor(t_in / t_out, dtype=torch.float32) - 0.5).clamp_min(0)
    else:
        scale = (torch.tensor(float(t_in - 1), dtype=torch.float32) / float(t_out - 1)) if t_out > 1 else \
            torch.tensor(0.0)
        src = scale.to(x.device) * i
    i0 = src.floor().clamp(max=t_in - 1)
    l1 = (src - i0).clamp(0, 1)[:, None]
    l0 = 1 - l1
    i0 = i0.long()
    i1 = torch.where(i0 < t_in - 1, i0 + 1, i0)
    xf = x.float()
    o = xf[i0] * l0 + xf[i1] * l1
    return o if unrounded else o.half()


# ---------------------------------------------------------------------------------------------------- small kernels
def timestep_ref(t, dim) -> Ref:
    half = dim // 2
    i = torch.arange(half, dtype=torch.float64, device=t.device)
    ex = LN10K * i / half
    w = torch.exp(-ex)
    arg = t.double()[:, None] * w[None]
    o = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    e_w = 3 * E24 * ex + 2.0 ** -22
    e = (t.double().abs()[:, None] * w[None] * (e_w + E24)).repeat(1, 2) + 2.0 ** -22 * o.abs() + 2.0 ** -60
    bound, pre = _out16(o, e)
    return Ref(o, bound, lambda r, c: dict(batch=r, freq=c % half, part="sin" if c >= half else "cos"), pre=pre)


def emulate_timestep(t, dim, bug=None, unrounded=False):
    """bug='swap': [sin, cos] instead of [cos, sin]."""
    half = dim // 2
    i = torch.arange(half, dtype=torch.float32, device=t.device)
    freq = torch.exp((-torch.tensor(LN10K, dtype=torch.float32) * i) / half)
    arg = t.float()[:, None] * freq[None]
    parts = [torch.cos(arg), torch.sin(arg)]
    if bug == "swap":
        parts = parts[::-1]
    o = torch.cat(parts, 1)
    return o if unrounded else o.half()


def silu_ref(x) -> Ref:
    """x fp16 [n] -> [n, 1]."""
    v = x.double()[:, None]
    o = v * torch.sigmoid(v)
    eps_exp = (2 + torch.floor(1.173 * v.abs())) * 2.0 ** -23
    e = o.abs() * (eps_exp * torch.sigmoid(-v) + 2.0 ** -22) + 2.0 ** -26
    bound, pre = _out16(o, e)
    return Ref(o, bound, lambda r, c: dict(index=r, x=x[r].item()), pre=pre)


def emulate_silu(x, unrounded=False):
    v = x.float()[:, None]
    o = v / (1 + torch.exp(-v))
    return o if unrounded else o.half()


def add_ref(a, b, dup=1):
    """torch's fp16 a + b, b tiled `dup` times over the leading dimension (add_bcast)."""
    return a + b.repeat(dup, *([1] * (b.dim() - 1)))


def emulate_add_bcast(a, b, dup, bug=None):
    """bug='interleave': each row of b repeated `dup` times in place (repeat_interleave) instead of the whole tiled."""
    if bug == "interleave":
        return (a.float() + b.float().repeat_interleave(dup, 0)).half()
    return (a.float() + b.float().repeat(dup, *([1] * (b.dim() - 1)))).half()


def all_finite_f16(device=None):
    """Every finite fp16 value (both zeros and the subnormals included), 63488 values."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(torch.float16)
    v = v[torch.isfinite(v)]
    return v.to(device) if device is not None else v
