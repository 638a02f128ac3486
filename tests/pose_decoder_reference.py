"""fp64 references, per-element bounds and an fp32 emulation of the Audio2Pose decoder kernel (pose_decoder_kernel<NC,
TRACE> in csrc/ap_pose_decoder.cu). Imported by the CPU checker tests and the GPU contract tests; not a conftest. The
checks (`check`, `headroom`) and constants are those of gemm_reference.py; every reference returns its `Ref`.

Teacher forcing
---------------
The traced entry point (ap_pose_decoder_trace_f16) writes trace [T, 5 L + 1, 512], the input of every stage: rows
(i, 5 l + k) of step i, layer l hold x (k = 0, the layer input), q, the attention output a, the LN2 output x2 and
y3 = x2 + linear2(relu(linear1(x2))) (LN3's input); row (i, 5 L) the pose head's input. Every stage is checked against fp64
evaluated on the kernel's own inputs to that stage, so errors never compound across stages, layers or steps, every bound
covers at most two matrices and two LayerNorms, and one stage is checked for all T steps in one batch:
  kv[l, :, h, i]   fp16 of the fp64 k / v rows of x                        (kv_ref)
  q                in_proj rows 0..511 of x + bias                          (q_ref)
  a                softmax(q K^T / 8 + mask[h, i, 0..i]) V over the kernel's own fp16 cache rows 0..i   (attn_ref)
  x2               LN2(LN1(x + out_proj(a)) + cross[i, l])                  (ln2_ref)
  y3               x2 + linear2(relu(linear1(x2)))                          (ffn_ref)
  next x           LN3(y3)                                                  (ln3_ref)
  out[i]           pose_map_r(pose head input)                              (head_ref)
  trace[i, 0]      token + (pe[i] + id_row), token = pose_map_b at i = 0, else pose_map(out[i - 1])   (token_ref)
`reference_run` runs the same functions autoregressively on their own outputs (unrounded fp64 cache): that is the
module's decoder in fp64 (the CPU checker compares it with kv_cached_infer).

Bounds
------
u = 2**-24. A fixed-order reduction in which every term passes through at most `depth` fp32 roundings (fmaf counts one)
is within depth u S of the exact sum, S = sum |terms|. Depths, read from the kernel:
  gemv_phase     8-term fmaf chain per uint4 + (K/256 - 1) partial adds + 5 warp_sum levels: 12 (K = 512), 16 (K = 1024);
                 then + bias and + residual, u |result| each
  scores         dot8 (a product and 7 fmaf) + 7 adds of the 8 dot8: 15; x 0.125 is exact; + mask: u |s|
  BlockReduce    5 + 4 levels (plus the per-thread pre-sum of <= 2 keys for z): 10
  P.V            ceil((i + 1) / 64)-term fmaf chain per group, then 7 + 7 adds: n_c + 14; / z: u |a|
  pose head      16-term fmaf chain + 5 warp_sum levels + bias: 21 u S + u |o|
  token          out_dim-term fmaf chain, + bias, pe + id_row, + token: 2 u (out_dim S + |t| + |pe + id| + |x|),
                 a full ulp per rounding (a factor 2 of headroom where one rounding dominates)
Softmax: expf is within 2 ulp (4 u relative) of exp of its fp32 argument s_j - m, which is itself rounded (u |s_j - m|):
eps_j = u |s_j - m| + 4 u. With p* the fp64 probabilities, own error |da_d| <= sum_j p_j |v_jd| ((n_c + 14) u + eps_j)
+ |a_d| (sum_j p_j eps_j + 11 u) (the z sum and the division). A score error ds propagates through the softmax
Jacobian diag(p) - p p^T elementwise: |da_d| <= sum_j p_j ds_j |v_jd| + (sum_k p_k ds_k) sum_j p_j |v_jd| (tighter than
its l2 norm <= 1/2, and as cheap). ds_j = 0.125 (15 u sum |q k_j| + sum |k_j| b_q) + u |s_j|, b_q the bound on q.
Two-pass LayerNorm over n = 512 (BlockReduce sums, exact / 512, rsqrtf within 2 ulp), norm_reference's derivation
with the tree depth 9 for the n-term sums:
  d_mu = 9 u mean|x|, d_var = 14 u var + 2 d_mu**2, d_r = r (d_var / (2 (var + eps)) + 2**-22 + u)
  own  = |g| (r d_mu + |xc| d_r) + 4 u (|xc r g| + |b|)
Within a stage, an error that enters before a matrix or a LayerNorm is carried as a per-element bound b and an l2 bound
B on the error vector:
  matrix W    b'_e = ||W_e||_2 B (Cauchy-Schwarz, row norms of the fp16 matrix in fp64)
  LayerNorm   the Jacobian is g / sigma (I - 1 1^T / n - xh xh^T / n): b'_e = |g_e| r (b_e + (1 + |xh_e|) B / sqrt(n)),
              B' = min(max|g| r B + ||own||, ||b'||)
  ReLU        1-Lipschitz; residual adds add both bounds
and every bound is multiplied by SECOND_ORDER for the products of first-order terms. Chaining a whole layer this way
would put every element's bound near the l2 norm of all 512 worst-case errors of the stage before, thousands of times
the kernel's error; checking each stage on its own traced inputs keeps a stage's bound within a small factor of the
worst case of its own roundings, so a change of 1e-4 relative in q, in the attention output or in a LayerNorm fails it.
The cache check is exact where it can be: kv must equal fp16(k*) unless [k* - pre, k* + pre] straddles a rounding
boundary, and then it may be either neighbour.

Emulation
---------
`emulate` reproduces the kernel in fp32 torch in the kernel's order (fmaf as one rounding of the fp64 sum, which can
differ from the hardware in rare double-rounding ties: the emulation is a model, not a bit-exact twin). `bug=` turns it
into models of plausible kernel mistakes (BUGS), which the checks must reject naming (step, layer, element).
"""
from __future__ import annotations

import math

import torch

import gemm_reference as GR
from gemm_reference import E24, OUT_FLOOR, OUT_REL, SECOND_ORDER, Ref

E, HEADS, D, FF, QKV = 512, 8, 64, 1024, 1536
VEC = 6656                                     # AP_POSE_VEC and the AP_POSE_* offsets of include/aniportrait_b200.h
B_QKV, B_OUT, B_FF1, B_FF2 = 0, 1536, 2048, 3072
LN1_G, LN1_B, LN2_G, LN2_B, LN3_G, LN3_B = 3584, 4096, 4608, 5120, 5632, 6144
THREADS, PV_GROUPS = 512, 64
STAGES = 5                    # trace rows per layer: x, q, attention output, LN2 output, linear2 + residual
DEPTH_512, DEPTH_1024, DEPTH_SCORE, DEPTH_BLOCK, DEPTH_HEAD = 12, 16, 15, 9, 21
u = E24

BUGS = ["mask_stride_T", "mask_transposed", "keys_lt_i", "keys_le_i_plus_1", "mask_next_head", "cache_next_head",
        "ln3_other_parity", "bias_other_parity", "cross_prev_layer", "cross_prev_step", "max_drops_keys_ge_512",
        "sum_drops_keys_ge_512", "pv_drops_group_7", "q_fp16", "attn_fp16", "unbiased_var", "no_eps",
        "pose_map_w_transposed", "pe_prev_row", "no_id_row"]


# ---------------------------------------------------------------------------------------------------- parameters
def layer_params(P, l):
    """fp64 views of layer l: (w_qkv, w_out, w_ff1, w_ff2, vec)."""
    return tuple(P[k][l].double() for k in ("w_qkv", "w_out", "w_ff1", "w_ff2", "vec"))


def _norms(P):
    """Per layer: spectral norms and row norms of the four fp16 matrices, in fp64, computed once per parameter set."""
    if "_norms" not in P:
        out = []
        for l in range(P["w_qkv"].shape[0]):
            ws = [P[k][l].double() for k in ("w_qkv", "w_out", "w_ff1", "w_ff2")]
            out.append([(torch.linalg.matrix_norm(w, ord=2).item(), w.norm(dim=1)) for w in ws])
        P["_norms"] = out
    return P["_norms"]


def _l2(b):
    return b.norm(dim=-1, keepdim=True)


def _ln(y, b, B, g, beta, eps):
    """fp64 LayerNorm of rows y [n, 512] whose error is bounded by b (per element) and B (l2): (value, b', B')."""
    n = y.shape[-1]
    mu = y.mean(-1, keepdim=True)
    xc = y - mu
    var = (xc * xc).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    xh = xc * r
    o = xh * g + beta
    d_mu = DEPTH_BLOCK * u * y.abs().mean(-1, keepdim=True)
    d_var = (DEPTH_BLOCK + 5) * u * var + 2 * d_mu ** 2
    d_r = r * (d_var / (2 * (var + eps)) + 2.0 ** -22 + u)
    own = g.abs() * (r * d_mu + xc.abs() * d_r) + 4 * u * ((xh * g).abs() + beta.abs())
    prop = g.abs() * r * (b + (1 + xh.abs()) * B / math.sqrt(n))
    bo = (own + prop) * SECOND_ORDER
    Bo = torch.minimum(g.abs().max() * r * B + _l2(own), _l2(bo)) * SECOND_ORDER
    return o, bo, Bo


def _gemv(x, w, bias, depth):
    """x [n, K] exact or bounded inputs, fp64 W [R, K]: (x W^T + bias, own error of the kernel's dot + bias add)."""
    o = x @ w.t()
    S = x.abs() @ w.abs().t()
    y = o + bias
    return y, depth * u * S + u * y.abs()


# ---------------------------------------------------------------------------------------------------- references
def _eps32(P):
    return float(torch.tensor(P["eps"], dtype=torch.float32))     # the kernel's fp32 epsilon


def kv_ref(P, x, l):
    """k / v of layer l for the trace rows x = trace[:, l] [T, 512] -> Ref over rows (which, head, step) [2 * 8 * T, 64]."""
    wq, _, _, _, vec = layer_params(P, l)
    x = x.double()
    T = x.shape[0]
    y, pre = _gemv(x, wq[E:], vec[B_QKV + E:B_QKV + QKV], DEPTH_512)        # [T, 1024]: k | v
    o = y.view(T, 2, HEADS, D).permute(1, 2, 0, 3).reshape(2 * HEADS * T, D)
    pre = (pre * SECOND_ORDER).view(T, 2, HEADS, D).permute(1, 2, 0, 3).reshape(2 * HEADS * T, D)

    def loc(r, c):
        which, rem = divmod(r, HEADS * T)
        h, i = divmod(rem, T)
        return dict(step=i, layer=l, cache="kv"[which], head=h, dim=c)
    return Ref(o, pre + OUT_REL * o.abs() + OUT_FLOOR, loc, pre=pre)


def _stage_ref(o, b, steps, l, stage):
    return Ref(o, b, lambda r, c: dict(step=int(steps[r]), layer=l, stage=stage, element=c), pre=b)


def q_ref(P, x, steps, l):
    """q = in_proj rows 0..511 (x) + bias for the layer inputs x [n, 512] -> Ref [n, 512] (fp32, no output rounding)."""
    wqkv, _, _, _, vec = layer_params(P, l)
    q, own = _gemv(x.double(), wqkv[:E], vec[B_QKV:B_QKV + E], DEPTH_512)
    return _stage_ref(q, own * SECOND_ORDER, steps, l, "q")


def attn_ref(P, q, steps, l, kv_l):
    """The attention output of the 8 heads for the kernel's q [n, 512] at the given steps, over its fp16 cache
    kv_l [2, 8, >= max(steps) + 1, 64] (rows j <= step) with mask[h, step, j] -> Ref [n, 512]."""
    dev = q.device
    n = q.shape[0]
    steps = steps.to(dev)
    K, V = kv_l[0].double(), kv_l[1].double()                               # [8, T, 64]
    T = K.shape[1]
    qh = q.double().view(n, HEADS, D)
    j = torch.arange(T, device=dev)
    valid = (j.view(1, 1, T) <= steps.view(n, 1, 1)).expand(n, HEADS, T)
    mrows = P["mask"][:, steps.to(P["mask"].device), :T].to(dev, torch.float64).permute(1, 0, 2)
    zero = torch.zeros((), dtype=torch.float64, device=dev)
    s = torch.einsum("nhd,htd->nht", qh, K) * 0.125 + torch.where(valid, mrows, zero)   # only j <= i is read
    s = torch.where(valid, s, torch.full((), -math.inf, dtype=torch.float64, device=dev))
    del mrows
    valid = valid & torch.isfinite(s)          # a -inf mask entry drops key j exactly (expf(-inf) = 0)
    ds = 0.125 * DEPTH_SCORE * u * torch.einsum("nhd,htd->nht", qh.abs(), K.abs())
    ds = torch.where(valid, ds + u * s.abs(), zero)
    p = torch.softmax(s, -1)
    m = s.max(-1, keepdim=True).values
    eps_j = torch.where(valid, u * (s - m).abs() + 4 * u, zero)
    del s
    Va = V.abs()
    a = torch.einsum("nht,htd->nhd", p, V)
    PV = torch.einsum("nht,htd->nhd", p, Va)
    n_c = torch.div(steps + 1 + PV_GROUPS - 1, PV_GROUPS, rounding_mode="floor").double().view(n, 1, 1)
    own = PV * (n_c + 14) * u + torch.einsum("nht,htd->nhd", p * eps_j, Va) \
        + a.abs() * ((p * eps_j).sum(-1, keepdim=True) + 11 * u)
    prop = torch.einsum("nht,htd->nhd", p * ds, Va) + (p * ds).sum(-1, keepdim=True) * PV
    b = ((own + prop) * SECOND_ORDER).reshape(n, E)
    return _stage_ref(a.reshape(n, E), b, steps.tolist(), l, "attention")


def ln2_ref(P, x, a, steps, l, cross_rows):
    """x2 = LN2(LN1(x + out_proj(a)) + cross) for the kernel's layer input x and attention output a [n, 512]."""
    _, wo, _, _, vec = layer_params(P, l)
    n_o, rn_o = _norms(P)[l][1]
    eps = _eps32(P)
    x = x.double()
    o, own = _gemv(a.double(), wo, vec[B_OUT:B_OUT + E], DEPTH_512)
    y = x + o
    b_y = (own + u * y.abs()) * SECOND_ORDER
    y, b_y, B_y = _ln(y, b_y, _l2(b_y), vec[LN1_G:LN1_G + E], vec[LN1_B:LN1_B + E], eps)
    y = y + cross_rows.double()
    b_y = b_y + u * y.abs()
    x2, b, _ = _ln(y, b_y, B_y + _l2(u * y.abs()), vec[LN2_G:LN2_G + E], vec[LN2_B:LN2_B + E], eps)
    return _stage_ref(x2, b, steps, l, "LN2")


def ffn_ref(P, x2, steps, l):
    """x2 + linear2(relu(linear1(x2))) for the kernel's LN2 output x2 [n, 512] (LN3's input)."""
    _, _, w1, w2, vec = layer_params(P, l)
    (n_1, rn_1), (n_2, rn_2) = _norms(P)[l][2:]
    x2 = x2.double()
    h, own = _gemv(x2, w1, vec[B_FF1:B_FF1 + FF], DEPTH_512)
    f = h.clamp_min(0)
    b_f = own * SECOND_ORDER                                                # ReLU is 1-Lipschitz
    o, own = _gemv(f, w2, vec[B_FF2:B_FF2 + E], DEPTH_1024)
    y = x2 + o
    b = (rn_2 * _l2(b_f) + own + u * y.abs()) * SECOND_ORDER
    return _stage_ref(y, b, steps, l, "FFN")


def ln3_ref(P, y, steps, l):
    """LN3 of the kernel's linear2 + residual y [n, 512]: the next layer's input (or the pose head's)."""
    vec = P["vec"][l].double()
    zero = torch.zeros(y.shape[0], 1, dtype=torch.float64, device=y.device)
    o, b, _ = _ln(y.double(), zero, zero, vec[LN3_G:LN3_G + E], vec[LN3_B:LN3_B + E], _eps32(P))
    return _stage_ref(o, b, steps, l, "LN3")


def head_ref(P, x):
    """out [T, out_dim] = pose_map_r(x), x = trace[:, L]."""
    y, own = _gemv(x.double(), P["pose_map_r_w"].double(), P["pose_map_r_b"].double(), DEPTH_HEAD)
    pre = own * SECOND_ORDER
    return Ref(y, pre, lambda r, c: dict(step=r, layer="pose head", element=c), pre=pre)


def token_ref(P, out, T):
    """trace[:, 0] [T, 512]: token + (pe[i] + id_row), token = pose_map_b (i = 0) or pose_map(out[i - 1])."""
    od = P["pose_map_w"].shape[1]
    pw, pb = P["pose_map_w"].double(), P["pose_map_b"].double()
    prev = out[:T - 1].double()
    t = torch.cat([pb.view(1, E), prev @ pw.t() + pb])
    # a full ulp (2 u) per rounding, as norm_reference allows where a few roundings dominate: a factor 2 of headroom
    own = torch.cat([torch.zeros(1, E, dtype=torch.float64, device=t.device),
                     2 * od * u * (prev.abs() @ pw.abs().t()) + 2 * u * t[1:].abs()])
    pi = P["pe"][:T].double() + P["id_row"].double()
    x = t + pi
    pre = (own + 2 * u * pi.abs() + 2 * u * x.abs()) * SECOND_ORDER
    return Ref(x, pre, lambda r, c: dict(step=r, layer="token", element=c), pre=pre)


def _cross_rows(P, l, T):
    return P["cross"][:T].view(T, -1, E)[:, l]


def stage(trace, l, k):
    """Trace rows of stage k of layer l for all steps (k = 0 the layer input; layer L, stage 0 the pose head input)."""
    return trace[:, STAGES * l + k]


def refs(P, T, out, kv, trace, kv_got=None):
    """(family, name, kernel values, Ref) for every checked quantity, in the order a bug shows up first: per layer the
    cache, then each stage; then the pose head and the tokens. kv fp16 [L, 2, 8, T, 64], the cache the layers read;
    trace [T, 5 L + 1, 512]; kv_got: the cache values to check (default kv; the emulation's unrounded fp32 values for
    `headroom`)."""
    L = P["w_qkv"].shape[0]
    steps = torch.arange(T, device=trace.device)
    st = steps.tolist()
    kv_got = kv if kv_got is None else kv_got
    for l in range(L):
        x, q, a, x2, y3 = (stage(trace, l, k) for k in range(STAGES))
        yield "kv", f"kv[{l}]", kv_got[l].reshape(2 * HEADS * T, D), kv_ref(P, x, l)
        yield "q", f"q[{l}]", q, q_ref(P, x, st, l)
        yield "attention", f"attention[{l}]", a, attn_ref(P, q, steps, l, kv[l])
        yield "LN2", f"LN2[{l}]", x2, ln2_ref(P, x, a, st, l, _cross_rows(P, l, T))
        yield "FFN", f"FFN[{l}]", y3, ffn_ref(P, x2, st, l)
        yield "LN3", f"LN3[{l}]", stage(trace, l + 1, 0), ln3_ref(P, y3, st, l)
    yield "pose head", "pose head", out, head_ref(P, stage(trace, L, 0))
    yield "token", "token", stage(trace, 0, 0), token_ref(P, out, T)


def check_kv_rounding(got16, ref, what):
    """got must be fp16(k*) or, where [k* - pre, k* + pre] straddles a rounding boundary, either neighbour."""
    lo = (ref.o - ref.pre).float().half().double()
    hi = (ref.o + ref.pre).float().half().double()
    g = got16.double()
    bad = ~((g >= lo) & (g <= hi))
    nb = int(bad.sum())
    if nb:
        i = int(bad.reshape(-1).nonzero()[0])
        r, c = divmod(i, got16.shape[1])
        raise AssertionError(f"{what}: {nb} cache elements are not a rounding of a value within the bound; first "
                             f"{ref.locate(r, c)}: got {g[r, c].item():.8g}, ref {ref.o[r, c].item():.8g}, allowed "
                             f"[{lo[r, c].item():.8g}, {hi[r, c].item():.8g}]")


def check(P, T, out, kv, trace, what=""):
    """Every element of out, kv and trace within its bound -> {quantity family: worst error / bound}."""
    worst = {}
    for fam, name, got, ref in refs(P, T, out, kv, trace):
        if fam == "kv":
            check_kv_rounding(got, ref, f"{what} {name}")
        r = GR.check(got, ref, f"{what} {name}")
        worst[fam] = max(worst.get(fam, 0.0), r)
    return worst


def headroom(P, T, out, kv, trace, kv32):
    """Largest |y - o*| / pre over the emulation's unrounded values (kv32: the fp32 k / v before the fp16 store)."""
    return max(GR.headroom(got, ref) for _, _, got, ref in refs(P, T, out, kv, trace, kv32))


# ---------------------------------------------------------------------------------------------------- fp64 run
def reference_run(P, T):
    """The decoder in fp64, each function above fed its own outputs: (out [T, od], kv fp64 [L, 2, 8, T, 64],
    trace [T, 5 L + 1, 512])."""
    L = P["w_qkv"].shape[0]
    od = P["pose_map_r_w"].shape[0]
    dev = P["vec"].device
    kv = torch.zeros(L, 2, HEADS, T, D, dtype=torch.float64, device=dev)
    trace = torch.zeros(T, STAGES * L + 1, E, dtype=torch.float64, device=dev)
    out = torch.zeros(T, od, dtype=torch.float64, device=dev)
    for i in range(T):
        trace[i, 0] = token_ref(P, out[:i + 1], i + 1).o[i]
        st = torch.tensor([i], device=dev)
        for l in range(L):
            r = trace[i:i + 1, STAGES * l:STAGES * l + STAGES + 1]           # this layer's stages and the next input
            kv[l, :, :, i] = kv_ref(P, r[:, 0], l).o.view(2, HEADS, D)
            r[:, 1] = q_ref(P, r[:, 0], [i], l).o
            r[:, 2] = attn_ref(P, r[:, 1], st, l, kv[l]).o
            r[:, 3] = ln2_ref(P, r[:, 0], r[:, 2], [i], l, _cross_rows(P, l, T)[i:i + 1]).o
            r[:, 4] = ffn_ref(P, r[:, 3], [i], l).o
            r[:, 5] = ln3_ref(P, r[:, 4], [i], l).o
        out[i] = head_ref(P, trace[i:i + 1, STAGES * L]).o[0]
    return out, kv, trace


# ---------------------------------------------------------------------------------------------------- emulation
def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _warp_sum(v):
    """warp_sum over the last dim (32 lanes): xor butterfly 16, 8, 4, 2, 1; every lane ends with the same bits."""
    idx = torch.arange(32, device=v.device)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v[..., 0]


def _block_sum(v):
    """BlockReduce::sum of one value per thread, v [..., 512]: warp sums, then a butterfly over the 16 partials."""
    w = _warp_sum(v.view(*v.shape[:-1], 16, 32))
    idx = torch.arange(16, device=v.device)
    for o in (8, 4, 2, 1):
        w = w + w[..., idx ^ o]
    return w[..., 0]


def _gemv32(w16, x):
    """gemv_phase for all rows of w16 [R, K] and fp32 x [K]: lane l's uint4 u holds elements (l + 32 u) * 8 .. + 7."""
    R, K = w16.shape
    U = K // 256
    wv = w16.float().view(R, U, 32, 8)
    xv = x.view(U, 32, 8)
    d = torch.zeros(R, U, 32, dtype=torch.float32, device=x.device)
    for e in range(8):
        d = _fma(wv[..., e], xv[..., e], d)
    s = d[:, 0]
    for k in range(1, U):
        s = s + d[:, k]
    return _warp_sum(s)


def _ln32(v, g, b, eps, bug):
    mean = _block_sum(v) * (1.0 / E)
    c = v - mean
    ss = _block_sum(c * c)
    var = ss / (E - 1) if bug == "unbiased_var" else ss * (1.0 / E)
    r = (1.0 / torch.sqrt((var if bug == "no_eps" else var + eps).double())).float()
    return c * r * g + b


def _attend32(q, kc, vc, P, i, T, bug):
    """Phase B for all 8 heads: q fp32 [8, 64], kc / vc fp16 [8, T, 64] -> fp32 [8, 64]."""
    dev = q.device
    ml = P["mask"].shape[1]
    n = min(i + 2, T) if bug == "keys_le_i_plus_1" else (i if bug == "keys_lt_i" else i + 1)
    heads = torch.arange(HEADS, device=dev)
    hk = (heads + 1) % HEADS if bug == "cache_next_head" else heads
    hm = (heads + 1) % HEADS if bug == "mask_next_head" else heads
    if n == 0:                                                          # no key: m = -inf, z = 0, 0 / 0
        return torch.full((HEADS, D), math.nan, device=dev)
    K, V = kc[hk, :n].float(), vc[hk, :n].float()                       # [8, n, 64]
    j = torch.arange(n, device=dev)
    mflat = P["mask"].reshape(-1)
    if bug == "mask_stride_T":
        midx = (hm.view(8, 1) * ml + i) * T + j
    elif bug == "mask_transposed":
        midx = (hm.view(8, 1) * ml + j) * ml + i
    else:
        midx = (hm.view(8, 1) * ml + i) * ml + j
    mrow = mflat[midx].float()
    s = torch.zeros(HEADS, n, dtype=torch.float32, device=dev)
    for uu in range(8):                                                 # s += dot8(k[u], q[u])
        kk, qq = K[..., uu * 8:uu * 8 + 8], q[:, None, uu * 8:uu * 8 + 8].expand(HEADS, n, 8)
        t = kk[..., 0] * qq[..., 0]
        for e in range(1, 8):
            t = _fma(kk[..., e], qq[..., e], t)
        s = s + t
    s = s * 0.125 + mrow
    m = (s[:, :min(n, THREADS)] if bug == "max_drops_keys_ge_512" else s).max(-1, keepdim=True).values
    e = torch.exp(s - m)
    ez = e[:, :THREADS] if bug == "sum_drops_keys_ge_512" else e
    zt = torch.zeros(HEADS, 2 * THREADS, dtype=torch.float32, device=dev)
    zt[:, :ez.shape[1]] = ez
    z = _block_sum(zt[:, :THREADS] + zt[:, THREADS:])                  # <= 2 keys per thread, then BlockReduce
    nc = -(-n // PV_GROUPS)
    ep = torch.zeros(HEADS, nc * PV_GROUPS, dtype=torch.float32, device=dev)
    ep[:, :n] = e
    vp = torch.zeros(HEADS, nc * PV_GROUPS, D, dtype=torch.float32, device=dev)
    vp[:, :n] = V
    ep, vp = ep.view(HEADS, nc, PV_GROUPS), vp.view(HEADS, nc, PV_GROUPS, D)
    acc = torch.zeros(HEADS, PV_GROUPS, D, dtype=torch.float32, device=dev)
    for k in range(nc):
        acc = _fma(ep[:, k, :, None], vp[:, k], acc)
    acc = acc.view(HEADS, 8, 8, D)
    s1 = acc[:, :, 0]
    for k in range(1, 7 if bug == "pv_drops_group_7" else 8):
        s1 = s1 + acc[:, :, k]
    a = s1[:, 0]
    for k in range(1, 8):
        a = a + s1[:, k]
    a = a / z[:, None]
    return a.half().float() if bug == "attn_fp16" else a


def emulate(P, T, bug=None):
    """The kernel in fp32 -> (out fp32 [T, od], kv fp16 [L, 2, 8, T, 64], trace fp32 [T, 5 L + 1, 512], kv32 fp32)."""
    assert bug is None or bug in BUGS, bug
    L = P["w_qkv"].shape[0]
    od = P["pose_map_r_w"].shape[0]
    dev = P["vec"].device
    vec = P["vec"].float()
    eps = torch.tensor(P["eps"], dtype=torch.float32)
    cross = P["cross"][:T].reshape(T * L, E).float()
    kv32 = torch.zeros(L, 2, HEADS, T, D, dtype=torch.float32, device=dev)
    kv = torch.zeros(L, 2, HEADS, T, D, dtype=torch.float16, device=dev)
    trace = torch.zeros(T, STAGES * L + 1, E, dtype=torch.float32, device=dev)
    out = torch.zeros(T, od, dtype=torch.float32, device=dev)
    pmw = P["pose_map_w"].float().reshape(-1)
    if bug == "pose_map_w_transposed":
        pmw = pmw.view(od, E).t().reshape(-1)
    pmw = pmw.view(E, od)
    tok = P["pose_map_b"].float()
    # LN3 of layer l - 1 runs at the start of layer l (and before the pose head) from the parameter block of global
    # layer g - 1; the other parity buffer holds block g, i.e. layer l (layer 0 of the next step before the pose head)
    ln3 = (lambda l: l % L) if bug == "ln3_other_parity" else (lambda l: l - 1)    # noqa: E731
    for i in range(T):
        pe = P["pe"][max(i - 1, 0) if bug == "pe_prev_row" else i].float()
        idr = torch.zeros(E, device=dev) if bug == "no_id_row" else P["id_row"].float()
        xs = tok + (pe + idr)
        hs = None
        for l in range(L):
            g = i * L + l
            if l > 0:
                lv = vec[ln3(l)]
                xs = _ln32(hs, lv[LN3_G:LN3_G + E], lv[LN3_B:LN3_B + E], eps, bug)
            r = trace[i, STAGES * l:STAGES * l + STAGES]
            r[0] = xs
            v = vec[(l - 1) % L] if bug == "bias_other_parity" else vec[l]
            lnv = vec[l]
            cg = {"cross_prev_layer": max(g - 1, 0), "cross_prev_step": g - L if g >= L else g}.get(bug, g)
            qkv = _gemv32(P["w_qkv"][l], xs) + v[B_QKV:B_QKV + QKV]
            kv32[l, :, :, i] = qkv[E:].view(2, HEADS, D)
            kv[l, :, :, i] = kv32[l, :, :, i].half()
            q = qkv[:E].half().float() if bug == "q_fp16" else qkv[:E]
            a = _attend32(q.view(HEADS, D), kv[l, 0], kv[l, 1], P, i, T, bug).reshape(E)
            hs = xs + (_gemv32(P["w_out"][l], a) + v[B_OUT:B_OUT + E])
            y = _ln32(hs, lnv[LN1_G:LN1_G + E], lnv[LN1_B:LN1_B + E], eps, bug) + cross[cg]
            xs = _ln32(y, lnv[LN2_G:LN2_G + E], lnv[LN2_B:LN2_B + E], eps, bug)
            f = (_gemv32(P["w_ff1"][l], xs) + v[B_FF1:B_FF1 + FF]).clamp_min(0)
            hs = xs + (_gemv32(P["w_ff2"][l], f) + v[B_FF2:B_FF2 + E])
            r[1], r[2], r[3], r[4] = q, a, xs, hs
        lv = vec[ln3(L)]
        xs = _ln32(hs, lv[LN3_G:LN3_G + E], lv[LN3_B:LN3_B + E], eps, bug)
        trace[i, STAGES * L] = xs
        rw = P["pose_map_r_w"].float().view(od, 16, 32)
        s = torch.zeros(od, 32, dtype=torch.float32, device=dev)
        for k in range(16):
            s = _fma(rw[:, k], xs.view(16, 32)[k], s)
        pose = _warp_sum(s) + P["pose_map_r_b"].float()
        out[i] = pose
        t = torch.zeros(E, dtype=torch.float32, device=dev)
        for o in range(od):
            t = _fma(pmw[:, o], pose[o].expand(E), t)
        tok = t + P["pose_map_b"].float()
    return out, kv, trace, kv32


# ---------------------------------------------------------------------------------------------------- operands
def synthetic_params(L, od, T, mask_len, pe_len, seed=0, eps=1e-5, device="cpu", mask="alibi_finite"):
    """Seeded decoder parameters at the scales of the module's initialisation (xavier in_proj, kaiming-uniform linears,
    LayerNorm weights near 1). mask: 'alibi_finite' (ALiBi below the diagonal, finite noise above it, so a read past
    the diagonal moves the result), 'alibi' (-inf above)."""
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape, s=1.0):
        return torch.randn(*shape, generator=g) * s

    vec = torch.zeros(L, VEC)
    vec[:, :LN1_G] = rnd(L, LN1_G, s=0.02)
    for gg, bb in ((LN1_G, LN1_B), (LN2_G, LN2_B), (LN3_G, LN3_B)):
        vec[:, gg:gg + E] = 1 + rnd(L, E, s=0.1)
        vec[:, bb:bb + E] = rnd(L, E, s=0.1)
    from pose_decoder_helpers import alibi_causal_mask
    m = alibi_causal_mask(HEADS, mask_len)
    if mask == "alibi_finite":
        up = torch.triu(torch.ones(mask_len, mask_len, dtype=torch.bool), 1)
        m = torch.where(up, rnd(HEADS, mask_len, mask_len, s=1.0), m)
    i = torch.arange(pe_len).float().unsqueeze(1)
    div = torch.exp(torch.arange(0, E, 2).float() * (-math.log(10000.0) / E))
    pe = torch.zeros(pe_len, E)
    pe[:, 0::2], pe[:, 1::2] = torch.sin(i * div), torch.cos(i * div)
    P = dict(w_qkv=rnd(L, QKV, E, s=0.054).half(), w_out=rnd(L, E, E, s=0.044).half(),
             w_ff1=rnd(L, FF, E, s=0.044).half(), w_ff2=rnd(L, E, FF, s=0.031).half(), vec=vec,
             pose_map_w=rnd(E, od, s=0.5), pose_map_b=rnd(E, s=0.1), pose_map_r_w=rnd(od, E, s=0.044),
             pose_map_r_b=rnd(od, s=0.02), pe=pe, id_row=rnd(E, s=0.5), mask=m.contiguous(),
             cross=rnd(T, L * E, s=0.5), eps=eps)
    return {k: (v.to(device).contiguous() if torch.is_tensor(v) else v) for k, v in P.items()}
