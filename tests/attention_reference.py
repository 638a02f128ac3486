"""fp64 references, a per-element error bound and fp32 emulations of the three attention kernels:
ap_attention_f16 (spatial / reference attention), ap_temporal_attention_f16 (motion module) and ap_softmax_rows_f16
(VAE mid-block). Imported by the CPU checker tests and the GPU contract tests; not a conftest.

References
----------
`spatial_ref`, `temporal_ref` and `softmax_ref` compute the op in float64 from the fp16 inputs the kernel sees, on
whatever device the inputs live on, one (frame, head) block at a time (query rows chunked further so that no
score matrix exceeds 2**24 elements). Each returns a `Ref`: the exact output `o`, the per-element error bound `bound`
and `locate(row, col)`, which names an element of the kernel's output matrix as (frame, head, row, column).

Per-element bound for the attention kernels
-------------------------------------------
For an output element o* = sum_j P*_j V_jc, with P* the fp64 softmax weights over the n keys of its row:

    |o - o*| <= TAU * (P* . |V|)_c + ALPHA_PER_KEY * n * max_j |V_jc| + OUT_FLOOR,     TAU = 4 * 2**-11

where (P* . |V|)_c = sum_j P*_j |V_jc| is the absolute-weighted mean the element averages. One 2**-11 each for:
  1. P rounded to fp16 before the P.V product (the fused kernels round it once: spatial the unnormalised
     p = exp2(s*c - m) <= 1, temporal mma.sync path the normalised P). A normal fp16 value carries a relative error
     <= 2**-11 (half an ulp), so the numerator sum_j p_j V_jc moves by <= 2**-11 sum_j p_j |V_jc|; l is summed from the
     unrounded fp32 p, so dividing by it gives 2**-11 (P* . |V|)_c.
  2. O / l rounded to fp16 once: 2**-11 |o| <= 2**-11 (P* . |V|)_c.
  3. fp32 accumulation of S, l and O: the products of fp16 operands are exact in fp32, the sums run over at most
     dpad = 192 terms (S) or over key tiles (O, l), each step rounding by 2**-24: far below 2**-11 for the key counts
     used here (<= 8192 keys), so a whole unit also covers the tensor cores' accumulation, whose rounding is not
     documented.
  4. Error of the weights themselves: an absolute error e in the exponent (S in fp32 times the fp32 scale, ex2.approx
     with relative error ~2**-22, the fma with -m) changes every P_j by a factor (1 + e ln 2); after normalisation the
     output moves by <= 2 |e| ln2 (P* . |V|)_c. The worst case of a d-term fp32 sum is
     |e| <= d 2**-24 sum_i |q_i k_i| scale log2(e), which keeps 2 |e| ln2 <= 2**-11 while
     sum_i |q_i k_i| scale <= 2**12.5 / d (90 at d = 64, 30 at d = 192); every case in the suite stays inside it.
P values below 2**-14 are fp16 subnormals: their rounding error is absolute, <= 2**-25 (half the subnormal spacing
2**-24), not relative. Over n keys that is at most n * 2**-25 * max_j |V_jc| / l with l >= 1 (the key at the running
maximum contributes exp2(0) = 1, and later rescaling only shrinks earlier errors): ALPHA_PER_KEY = 2**-25. OUT_FLOOR =
2**-25 is the same half-ulp for an output that is itself subnormal. The fp16 inputs are exact in float64, so the
reference adds no error of its own. None of these constants is fitted to a kernel's output.

Softmax rows: |y - y*| <= 2**-10 |y*| + 2**-24: 2**-11 for rounding y to fp16, 2**-11 for __expf (argument error
|x - max| * 2**-24 relative) and the fp32 row sum (a tree over 256 threads); 2**-24 covers outputs in fp16's subnormal
range (half-ulp 2**-25) and values that underflow.

Emulations
----------
`spatial_emulate`, `temporal_emulate` and `softmax_emulate` reproduce each kernel's rounding points in fp32 torch on any
device, so the bound can be calibrated without a GPU: spatial: fp32 S, an online softmax over the kernel's BN-key tiles
(BN = 128, or 64 for dpad = 192; own keys and bank keys are tiled separately), P rounded to fp16, fp32 O and l, O / l
rounded to fp16; temporal: the mma.sync path rounds the normalised P to fp16, the scalar path keeps it in fp32; softmax:
fp32 throughout. They do not model ex2.approx / __expf (torch's exp2 / exp are used) or the kernels' summation order.
The `bug=` argument turns an emulation into a model of a specific kernel bug, which the checker must reject.
"""
from __future__ import annotations

import math

import torch

TAU = 4 * 2.0 ** -11
ALPHA_PER_KEY = 2.0 ** -25
OUT_FLOOR = 2.0 ** -25
SOFTMAX_REL = 2.0 ** -10
SOFTMAX_ABS = 2.0 ** -24
_CHUNK = 1 << 24          # score-matrix elements per fp64 chunk
LOG2E = 1.4426950408889634


class Ref:
    def __init__(self, o: torch.Tensor, bound: torch.Tensor, locate):
        self.o, self.bound, self.locate = o, bound, locate


def worst(out: torch.Tensor, ref: Ref):
    """(largest |out - o*| / bound over all elements, location of that element). NaN / inf outputs count as inf."""
    assert out.shape == ref.o.shape, (tuple(out.shape), tuple(ref.o.shape))
    ratio = (out.double() - ref.o).abs() / ref.bound
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    i = int(ratio.argmax())
    r, c = divmod(i, ratio.shape[1])
    return ratio.view(-1)[i].item(), ref.locate(r, c), (r, c)


def check(out: torch.Tensor, ref: Ref, what: str = "") -> float:
    """Asserts every element of `out` is within its bound; returns the worst ratio of error to bound."""
    ratio, loc, (r, c) = worst(out, ref)
    if not ratio <= 1.0:
        raise AssertionError(f"{what}: worst element {loc} ratio {ratio:.3g}: out {out[r, c].item():.6g}, "
                             f"ref {ref.o[r, c].item():.6g}, bound {ref.bound[r, c].item():.3g}")
    return ratio


def _attend(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float):
    """fp64 softmax(scale q k^T) v and its bound for q [B, n, d], k/v [B, m, d]; chunked over B and query rows."""
    B, n, _ = q.shape
    m = k.shape[1]
    o = torch.empty(B, n, v.shape[2], dtype=torch.float64, device=q.device)
    bound = torch.empty_like(o)
    vabs = v.abs()
    floor = ALPHA_PER_KEY * m * vabs.amax(1, keepdim=True) + OUT_FLOOR           # [B, 1, d]
    rows = max(1, _CHUNK // m)
    bstep = max(1, rows // n)
    for b0 in range(0, B, bstep):
        b1 = min(B, b0 + bstep)
        for r0 in range(0, n, rows):
            r1 = min(n, r0 + rows)
            p = torch.softmax((q[b0:b1, r0:r1] @ k[b0:b1].transpose(1, 2)) * scale, dim=-1)
            o[b0:b1, r0:r1] = p @ v[b0:b1]
            bound[b0:b1, r0:r1] = TAU * (p @ vabs[b0:b1]) + floor[b0:b1]
    return o, bound


def _heads(x: torch.Tensor, heads: int, width: int, d: int) -> torch.Tensor:
    """[rows, >= heads*width] (head h at columns [h*width, h*width + d)) -> fp64 [heads, rows, d]."""
    rows = x.shape[0]
    return x[:, :heads * width].reshape(rows, heads, width)[..., :d].permute(1, 0, 2).double()


def spatial_ref(q, k, v, n_frames, tokens, heads, d, dpad, bank_k=None, bank_v=None, bank_tokens=0, n_banks=0,
                first_bank_frame=0, frames_per_bank=1, scale=None) -> Ref:
    """ap_attention_f16's contract, in the reference's formulation (mutual_self_attention.py:147-186): a frame's keys
    are its own tokens, concatenated (torch.cat(..., dim=1)) with its bank entry when it reads the bank. The bank list is
    built as the reference builds `bank_fea`: every bank repeated for the frames_per_bank frames that read it
    ("b t l c -> (b t) l c"); frames from first_bank_frame on take its entries in order, earlier frames (the
    unconditional CFG half, recomputed without the bank at :166-186) attend to their own tokens only."""
    scale = d ** -0.5 if scale is None else scale
    has_bank = bank_k is not None and bank_tokens > 0
    bank_fea = [b for b in range(n_banks) for _ in range(frames_per_bank)] if has_bank else []
    o = torch.empty(n_frames * tokens, heads * d, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(o)
    for f in range(n_frames):
        sl = slice(f * tokens, (f + 1) * tokens)
        qf, kf, vf = (_heads(t[sl], heads, dpad, d) for t in (q, k, v))
        if has_bank and f >= first_bank_frame:
            b = bank_fea[f - first_bank_frame]    # IndexError: the call would read past the last bank
            bs = slice(b * bank_tokens, (b + 1) * bank_tokens)
            kf = torch.cat([kf, _heads(bank_k[bs], heads, dpad, d)], dim=1)
            vf = torch.cat([vf, _heads(bank_v[bs], heads, dpad, d)], dim=1)
        of, bf = _attend(qf, kf, vf, scale)
        o[sl] = of.permute(1, 0, 2).reshape(tokens, heads * d)
        bound[sl] = bf.permute(1, 0, 2).reshape(tokens, heads * d)
    return Ref(o, bound, lambda r, c: dict(frame=r // tokens, head=c // d, row=r % tokens, col=c % d))


def temporal_ref(qkv, B, F, N, C, heads, scale=None) -> Ref:
    """The motion module's attention (motion_module.py:351-388): rows (b f n) -> (b n) f, softmax over the F frames of
    each (batch, position, head). qkv: [B*F*N, >= 3C] = [q | k | v]."""
    d = C // heads
    scale = d ** -0.5 if scale is None else scale
    o = torch.empty(B * F * N, C, dtype=torch.float64, device=qkv.device)
    bound = torch.empty_like(o)
    for b in range(B):
        sl = slice(b * F * N, (b + 1) * F * N)
        # [F*N, C] -> [N*heads, F, d]
        q, k, v = (qkv[sl, i * C:(i + 1) * C].double().reshape(F, N, heads, d).permute(1, 2, 0, 3)
                   .reshape(N * heads, F, d) for i in range(3))
        ob, bb = _attend(q, k, v, scale)
        o[sl] = ob.reshape(N, heads, F, d).permute(2, 0, 1, 3).reshape(F * N, C)
        bound[sl] = bb.reshape(N, heads, F, d).permute(2, 0, 1, 3).reshape(F * N, C)
    return Ref(o, bound, lambda r, c: dict(frame=r // N, head=c // d, row=r % N, col=c % d))


def softmax_ref(x: torch.Tensor, cols: int) -> Ref:
    """Row softmax of the first `cols` columns of x [rows, ld]."""
    y = torch.softmax(x[:, :cols].double(), dim=-1)
    return Ref(y, SOFTMAX_REL * y.abs() + SOFTMAX_ABS, lambda r, c: dict(frame=0, head=0, row=r, col=c))


# ------------------------------------------------------------------------------------------------------ emulations
def _tile_rows(x: torch.Tensor, start: int, count: int) -> torch.Tensor:
    """Rows [start, start + count) of x as a TMA box reads them: rows past the end of the tensor are zeros."""
    out = torch.zeros(count, x.shape[1], dtype=x.dtype, device=x.device)
    n = max(0, min(count, x.shape[0] - start))
    if n:
        out[:n] = x[start:start + n]
    return out


def spatial_emulate(q, k, v, n_frames, tokens, heads, d, dpad, bank_k=None, bank_v=None, bank_tokens=0, n_banks=0,
                    first_bank_frame=0, frames_per_bank=1, scale=None, bug=None) -> torch.Tensor:
    """ap_attention_f16's rounding points in fp32 (see the module docstring). Bugs modelled by `bug`:
    'bank_index' (bank index + 1), 'first_bank_frame' (the bank starts one frame early), 'tail_next' (the ragged last
    key tile is not masked: its extra keys are the next frame's / bank's rows), 'tail_zero' (same, read as zero keys),
    'scale_dpad' (scale from dpad instead of d), 'lazy_rescale' (a new running max does not rescale O and l),
    'row' (one output token row 1 % off)."""
    scale = d ** -0.5 if scale is None else scale
    if bug == "scale_dpad":
        scale = dpad ** -0.5
    bn = 64 if dpad == 192 else 128
    c2 = torch.tensor(scale * LOG2E, dtype=torch.float32).item()
    has_bank = bank_k is not None and bank_tokens > 0
    first = first_bank_frame - (bug == "first_bank_frame")
    cols = heads * dpad
    qf32, kf, vf = (t[:, :cols].float() for t in (q, k, v))
    bkf = bank_k[:, :cols].float() if has_bank else None
    bvf = bank_v[:, :cols].float() if has_bank else None
    out = torch.empty(n_frames * tokens, heads * d, dtype=torch.float16, device=q.device)
    for f in range(n_frames):
        tiles = [(kf, vf, f * tokens + j, min(bn, tokens - j)) for j in range(0, tokens, bn)]
        if has_bank and f >= first:
            b = (f - first) // frames_per_bank + (bug == "bank_index")
            tiles += [(bkf, bvf, b * bank_tokens + j, min(bn, bank_tokens - j)) for j in range(0, bank_tokens, bn)]
        Q = qf32[f * tokens:(f + 1) * tokens].view(tokens, heads, dpad).transpose(0, 1)      # [h, n, dpad]
        O = torch.zeros(heads, tokens, dpad, device=q.device)
        m = torch.full((heads, tokens, 1), -math.inf, device=q.device)
        l = torch.zeros(heads, tokens, 1, device=q.device)
        for K_, V_, row, valid in tiles:
            Kt = _tile_rows(K_, row, bn).view(bn, heads, dpad).transpose(0, 1)
            Vt = _tile_rows(V_, row, bn).view(bn, heads, dpad).transpose(0, 1)
            if bug == "tail_zero" and valid < bn:
                Kt[:, valid:] = 0
                Vt[:, valid:] = 0
            S = Q @ Kt.transpose(1, 2)
            if valid < bn and bug not in ("tail_next", "tail_zero"):
                S[..., valid:] = -math.inf
            m_new = torch.maximum(m, S.amax(-1, keepdim=True) * c2)
            alpha = torch.exp2(m - m_new)
            if bug == "lazy_rescale":
                alpha = torch.ones_like(alpha)
            m = m_new
            p = torch.exp2(S * c2 - m)
            l = l * alpha + p.sum(-1, keepdim=True)
            O = O * alpha + p.half().float() @ Vt
        o = (O * (1.0 / l)).half()[..., :d]                                                   # [h, n, d]
        out[f * tokens:(f + 1) * tokens] = o.transpose(0, 1).reshape(tokens, heads * d)
    if bug == "row":
        r = (n_frames - 1) * tokens + tokens // 2
        out[r] = (out[r].float() * 1.01).half()
    return out


def temporal_mma_path(F, C, heads) -> bool:
    """Whether ap_temporal_attention_f16 takes its mma.sync kernel (else the scalar one)."""
    d = C // heads
    return F <= 16 and C % 320 == 0 and d in (40, 80, 160)


def temporal_emulate(qkv, B, F, N, C, heads, scale=None, bug=None) -> torch.Tensor:
    """ap_temporal_attention_f16's rounding points in fp32. The mma.sync path pads the window to 16 key frames with zero
    rows and rounds the normalised P to fp16; the scalar path keeps P in fp32. bug='frames' stops masking the padded
    key frames (zero keys and values at frames F.. of the padded window: 16 on the mma.sync path, the next power of two
    on the scalar path)."""
    d = C // heads
    scale = d ** -0.5 if scale is None else scale
    mma = temporal_mma_path(F, C, heads)
    fp = 16 if mma else max(4, 1 << (F - 1).bit_length())
    q, k, v = (qkv[:, i * C:(i + 1) * C].float().reshape(B, F, N, heads, d).permute(0, 2, 3, 1, 4) for i in range(3))
    pad = lambda t: torch.cat([t, t.new_zeros(*t.shape[:3], fp - F, d)], dim=3)  # noqa: E731
    k, v = pad(k), pad(v)
    S = q @ k.transpose(-1, -2)                                                   # [B, N, h, F, fp]
    if bug != "frames":
        S[..., F:] = -math.inf
    if mma:
        sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32).item()
        p = torch.exp2((S - S.amax(-1, keepdim=True)) * sl2)
        P = (p * (1.0 / p.sum(-1, keepdim=True))).half().float()
    else:
        Ss = S * scale
        p = torch.exp(Ss - Ss.amax(-1, keepdim=True))
        P = p * (1.0 / p.sum(-1, keepdim=True))
    o = (P @ v).half()                                                            # [B, N, h, F, d]
    return o.permute(0, 3, 1, 2, 4).reshape(B * F * N, C)


def softmax_emulate(x: torch.Tensor, cols: int, bug=None) -> torch.Tensor:
    """ap_softmax_rows_f16 in fp32. bug='pad' adds the first padding column (x[:, cols], ld > cols) to the row sum."""
    xf = x[:, :cols].float()
    mx = xf.amax(-1, keepdim=True)
    e = torch.exp(xf - mx)
    s = e.sum(-1, keepdim=True)
    if bug == "pad":
        s = s + torch.exp(x[:, cols:cols + 1].float() - mx)
    return (e * (1.0 / s)).half()
