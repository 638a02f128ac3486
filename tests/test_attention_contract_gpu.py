"""The call contract of the three attention kernels, element by element against float64 (attention_reference.py), at
the layouts every caller uses and at the edges of the C ABI:

  ap_attention_f16           UNet reference attention (the four bank layouts of BasicTransformerBlock.run in
                             models/blocks.py), PoseGuider, CLIP ViT-L/14, wav2vec2; dpad / bank / stride edges
  ap_temporal_attention_f16  motion module: mma.sync path (F <= 16, d in {40, 80, 160}) and scalar path
  ap_softmax_rows_f16        VAE mid-block attention

Every case runs through ops.* on fp16 inputs, checks every output element against its bound, and checks that a second
call gives the same bits. The worst ratio of error to bound is printed per case (run with -s to see it).
"""
import pytest
import torch

import attention_reference as AR

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _heads_buf(rows, heads, d, dpad, n, g, dev, sigma=1.5, extra=0):
    """n fp16 column blocks [rows, heads*dpad] of one buffer [rows, n*heads*dpad + extra] (head h: N(0, sigma^2) values
    at columns [h*dpad, h*dpad + d), zeros up to dpad); the `extra` columns after them hold NaN, which must never be
    read."""
    hp = heads * dpad
    t = torch.zeros(rows, n, heads, dpad)
    t[..., :d] = torch.randn(rows, n, heads, d, generator=g) * sigma
    buf = torch.full((rows, n * hp + extra), float("nan"), dtype=torch.float16)
    buf[:, :n * hp] = t.to(torch.float16).reshape(rows, n * hp)
    buf = buf.to(dev)
    return [buf[:, i * hp:(i + 1) * hp] for i in range(n)]


def _report(kernel, name, ratio):
    print(f"\n[{kernel}] {name}: worst error / bound = {ratio:.3f}")


def _spatial(dev, name, frames, tokens, heads, d, n_banks=0, bank_tokens=None, first=0, fpb=1, scale=None, sigma=1.5,
             ld_extra=0, seed=0, shape_keys=None, out=None):
    """Runs ops.attention twice on a seeded case and checks it; returns (output, kwargs of the call)."""
    from aniportrait_b200 import ops
    dpad = ops.head_pad(d)
    g = _gen(seed)
    q, k, v = _heads_buf(frames * tokens, heads, d, dpad, 3, g, dev, sigma, ld_extra)
    kw = dict(n_frames=frames, tokens=tokens, heads=heads, d=d, dpad=dpad, scale=scale)
    bank_tokens = tokens if bank_tokens is None else bank_tokens
    if n_banks:
        bk, bv = _heads_buf(n_banks * bank_tokens, heads, d, dpad, 2, g, dev, sigma)
        if shape_keys is not None:
            shape_keys(bk)
        kw.update(bank_k=bk, bank_v=bv, bank_tokens=bank_tokens, n_banks=n_banks, first_bank_frame=first,
                  frames_per_bank=fpb)
    call = dict(kw, head_dim=d)
    del call["d"]
    o1 = ops.attention(q, k, v, out=out, **call).clone()
    o2 = ops.attention(q, k, v, out=out, **call)
    assert torch.equal(o1, o2), f"{name}: two calls differ"
    ratio = AR.check(o1, AR.spatial_ref(q, k, v, **kw), name)
    _report("ap_attention_f16", name, ratio)
    return o1, (q, k, v), call


# ----------------------------------------------------------------------------------- spatial: one case per caller layout
# BasicTransformerBlock.run (models/blocks.py:358-388), F = 4 frames per window
F_WIN = 4
UNET_LAYOUTS = {
    # grouped windows of one video: n_uncond units own-only, then n_cond units reading one conditional bank
    "unet_grouped_u1_c2": dict(frames=3 * F_WIN, n_banks=1, first=1 * F_WIN, fpb=2 * F_WIN),
    "unet_grouped_u2_c2": dict(frames=4 * F_WIN, n_banks=1, first=2 * F_WIN, fpb=2 * F_WIN),
    "unet_grouped_u0_c4": dict(frames=4 * F_WIN, n_banks=1, first=0, fpb=4 * F_WIN),
    "unet_grouped_u3_c0": dict(frames=3 * F_WIN),                 # n_cond = 0: the block makes an own-only call
    # single conditional branch of a CFG reader: nb = 4 banks, the conditional half (2) read by batches of F frames
    "unet_cond_branch": dict(frames=2 * F_WIN, n_banks=2, first=0, fpb=F_WIN),
    # CFG batch B = 4: frames of the first half own-only, frame f of the second half reads bank (f - 2F) // F
    "unet_cfg_batch_b4": dict(frames=4 * F_WIN, n_banks=2, first=2 * F_WIN, fpb=F_WIN),
    "unet_cfg_batch_b2": dict(frames=2 * F_WIN, n_banks=1, first=F_WIN, fpb=F_WIN),
    # no CFG: every frame reads bank f // F
    "unet_no_cfg_b3": dict(frames=3 * F_WIN, n_banks=3, first=0, fpb=F_WIN),
}


@pytest.mark.parametrize("name", list(UNET_LAYOUTS))
@pytest.mark.parametrize("tokens,d", [(256, 40), (64, 160)])
def test_unet_reference_attention_layouts(cuda_dev, name, tokens, d):
    _spatial(cuda_dev, f"{name} N={tokens} d={d}", tokens=tokens, heads=8, d=d, seed=1, **UNET_LAYOUTS[name])


def test_pose_guider_attention(cuda_dev):
    _spatial(cuda_dev, "pose_guider 16 heads d=88", frames=2, tokens=1024, heads=16, d=88, seed=2)


def test_clip_attention(cuda_dev):
    # 257 tokens: the last query tile and the last key tile hold one row each; d = dpad = 64
    _spatial(cuda_dev, "clip B=2 T=257", frames=2, tokens=257, heads=16, d=64, seed=3)


@pytest.mark.parametrize("seq_len", [1, 2, 49, 129, 1499])
def test_wav2vec2_attention(cuda_dev, seq_len):
    _spatial(cuda_dev, f"wav2vec2 T={seq_len}", frames=1, tokens=seq_len, heads=12, d=64, seed=4)


# ------------------------------------------------------------------------------------------------------ spatial edges
@pytest.mark.parametrize("d", [40, 64, 80, 128, 160, 192])
def test_head_dims(cuda_dev, d):
    _spatial(cuda_dev, f"d={d}", frames=3, tokens=200, heads=4, d=d, n_banks=1, bank_tokens=150, first=1, fpb=2,
             sigma=1.2, seed=5)


@pytest.mark.parametrize("bank_tokens", [256, 77, 333])
def test_bank_tokens(cuda_dev, bank_tokens):
    _spatial(cuda_dev, f"bank_tokens={bank_tokens} tokens=256", frames=4, tokens=256, heads=8, d=40, n_banks=2,
             bank_tokens=bank_tokens, first=2, fpb=1, seed=6)


def test_first_bank_frame_past_the_end_is_own_only(cuda_dev):
    from aniportrait_b200 import ops
    for first in (4, 9):
        o, (q, k, v), call = _spatial(cuda_dev, f"first_bank_frame={first} n_frames=4", frames=4, tokens=200, heads=4,
                                      d=80, n_banks=1, first=first, fpb=1, seed=7)
        plain = {key: call[key] for key in ("n_frames", "tokens", "heads", "head_dim", "dpad")}
        assert torch.equal(o, ops.attention(q, k, v, **plain))


def test_more_units_than_sms_mixed_tile_counts(cuda_dev):
    # 8 frames x 8 heads x 3 query tiles = 192 units on 132 SMs; own-only units have 3 key tiles, bank units 5 (ragged)
    _spatial(cuda_dev, "192 units, 3/5 key tiles", frames=8, tokens=300, heads=8, d=40, n_banks=2, bank_tokens=200,
             first=3, fpb=3, seed=8)


def test_wide_qkv_stride(cuda_dev):
    # ld_qkv = 3*heads*dpad + 136; the extra columns hold NaN
    _spatial(cuda_dev, "ld_qkv > 3*heads*dpad", frames=2, tokens=300, heads=4, d=80, n_banks=1, first=1, fpb=1,
             ld_extra=136, seed=9)


def test_out_column_slice_keeps_sentinels(cuda_dev):
    frames, tokens, heads, d = 3, 150, 4, 40
    rows, width = frames * tokens, heads * d
    buf = torch.full((rows + 5, width + 24), -7.25, dtype=torch.float16, device=cuda_dev)
    out = buf[:rows, 8:8 + width]
    _spatial(cuda_dev, "out column slice", frames=frames, tokens=tokens, heads=heads, d=d, n_banks=1, first=1,
             fpb=2, seed=10, out=out)
    assert (buf[:, :8] == -7.25).all() and (buf[:, 8 + width:] == -7.25).all() and (buf[rows:] == -7.25).all()


@pytest.mark.parametrize("scale", [0.05, 0.3])
def test_scale_not_head_dim(cuda_dev, scale):
    _spatial(cuda_dev, f"scale={scale}", frames=2, tokens=200, heads=4, d=64, n_banks=1, first=1, fpb=1,
             scale=scale, sigma=1.0, seed=11)


def test_row_max_first_in_late_bank_tile(cuda_dev):
    # the last 128-key bank tile has keys 5x larger than all others: the running maximum jumps there
    def grow(bk):
        bk[256:] *= 5
    _spatial(cuda_dev, "max in last bank tile", frames=2, tokens=256, heads=4, d=40, n_banks=1, bank_tokens=300,
             first=0, fpb=2, sigma=1.0, seed=12, shape_keys=grow)


def test_attention_refuses_misaligned_out(cuda_dev):
    from aniportrait_b200 import _lib, ops
    frames, tokens, heads, d = 1, 64, 2, 64
    q, k, v = _heads_buf(frames * tokens, heads, d, 64, 3, _gen(13), cuda_dev)
    flat = torch.zeros(tokens * heads * d + 8, dtype=torch.float16, device=cuda_dev)
    out = flat[1:1 + tokens * heads * d].view(tokens, heads * d)   # 2-byte offset
    with pytest.raises(_lib.ApError, match="4-byte aligned"):
        ops.attention(q, k, v, frames, tokens, heads, d, 64, out=out)


# ----------------------------------------------------------------------------------------------------------- temporal
def _temporal(dev, name, B, Fr, N, C, heads, sigma=1.0, seed=0, wide=False):
    from aniportrait_b200 import ops
    g = _gen(seed)
    rows = B * Fr * N
    qkv_v = (torch.randn(rows, 3 * C, generator=g) * sigma).to(torch.float16)
    out = None
    if wide:   # 16-byte aligned slices of wider buffers (column offset 8, 24 spare columns), sentinels around them
        qb = torch.full((rows, 3 * C + 32), 1234.0, dtype=torch.float16, device=dev)
        qb[:, 8:8 + 3 * C] = qkv_v.to(dev)
        qkv = qb[:, 8:8 + 3 * C]
        ob = torch.full((rows, C + 16), -3.5, dtype=torch.float16, device=dev)
        out = ob[:, 8:8 + C]
    else:
        qkv = qkv_v.to(dev)
    o1 = ops.temporal_attention(qkv, B, Fr, N, C, heads, out=out).clone()
    o2 = ops.temporal_attention(qkv, B, Fr, N, C, heads, out=out)
    assert torch.equal(o1, o2), f"{name}: two calls differ"
    path = "mma.sync" if AR.temporal_mma_path(Fr, C, heads) else "scalar"
    ratio = AR.check(o1, AR.temporal_ref(qkv, B, Fr, N, C, heads), name)
    _report("ap_temporal_attention_f16", f"{path} {name}", ratio)
    if wide:
        assert (ob[:, :8] == -3.5).all() and (ob[:, 8 + C:] == -3.5).all()
        assert torch.equal(qb[:, 8:8 + 3 * C].cpu(), qkv_v)


# every F and every d on both paths; N = 1 and N = 333 on each path
TEMPORAL_CASES = [
    # mma.sync path (F <= 16)
    (1, 1, 333, 320), (2, 2, 64, 640), (4, 8, 1, 1280), (2, 9, 64, 320), (1, 15, 333, 640), (2, 16, 64, 1280),
    (1, 16, 1, 320),
    # scalar path (F > 16)
    (2, 17, 64, 320), (1, 20, 333, 640), (4, 24, 1, 1280), (2, 31, 1, 320), (1, 32, 64, 640), (1, 20, 64, 1280),
    (1, 17, 333, 1280),
]


@pytest.mark.parametrize("B,Fr,N,C", TEMPORAL_CASES)
def test_temporal_windows(cuda_dev, B, Fr, N, C):
    _temporal(cuda_dev, f"B={B} F={Fr} N={N} C={C}", B, Fr, N, C, 8, sigma=1.5, seed=20 + Fr)


@pytest.mark.parametrize("heads,Fr", [(1, 16), (2, 12), (4, 20), (5, 8)])
def test_temporal_head_counts(cuda_dev, heads, Fr):
    _temporal(cuda_dev, f"heads={heads} F={Fr} C=320", 2, Fr, 37, 320, heads, sigma=1.5, seed=40 + heads)


@pytest.mark.parametrize("Fr,C", [(16, 640), (24, 320)])
def test_temporal_strided_views(cuda_dev, Fr, C):
    _temporal(cuda_dev, f"strided qkv/out F={Fr} C={C}", 2, Fr, 50, C, 8, sigma=1.5, seed=50, wide=True)


@pytest.mark.parametrize("Fr,C", [(16, 1280), (32, 640)])
def test_temporal_large_logits(cuda_dev, Fr, C):
    _temporal(cuda_dev, f"large logits F={Fr} C={C}", 1, Fr, 64, C, 8, sigma=2.0, seed=60)


def test_temporal_refuses_misaligned(cuda_dev):
    from aniportrait_b200 import _lib, ops
    B, Fr, N, C = 1, 16, 4, 320
    rows = B * Fr * N
    flat = torch.zeros(rows * 3 * C + 16, dtype=torch.float16, device=cuda_dev)
    good = flat[:rows * 3 * C].view(rows, 3 * C)
    bad = flat[4:4 + rows * 3 * C].view(rows, 3 * C)                # 8-byte offset
    out_flat = torch.zeros(rows * C + 16, dtype=torch.float16, device=cuda_dev)
    bad_out = out_flat[4:4 + rows * C].view(rows, C)
    for qkv, out in ((bad, None), (good, bad_out)):
        with pytest.raises(_lib.ApError, match="16-byte aligned"):
            ops.temporal_attention(qkv, B, Fr, N, C, 8, out=out)


# ------------------------------------------------------------------------------------------------------------ softmax
def _softmax_abi(x, out, rows, cols, ld):
    from aniportrait_b200 import _lib, ops
    ops._ensure(x)
    _lib.check(_lib.lib().ap_softmax_rows_f16(_lib.ptr(x), _lib.ptr(out), _lib.LL(rows), _lib.I(cols), _lib.LL(ld),
                                              _lib.stream_ptr()), "ap_softmax_rows_f16")


def _softmax_case(dev, name, x):
    from aniportrait_b200 import ops
    ref = AR.softmax_ref(x, x.shape[1])
    y1 = ops.softmax_rows(x.clone())
    y2 = ops.softmax_rows(x.clone())
    assert torch.equal(y1, y2), f"{name}: two calls differ"
    ratio = AR.check(y1, ref, name)
    _report("ap_softmax_rows_f16", name, ratio)


@pytest.mark.parametrize("rows", [1, 7, 4096])
@pytest.mark.parametrize("cols", [2, 128, 1000, 4096, 6144])
def test_softmax_shapes(cuda_dev, rows, cols):
    x = (torch.randn(rows, cols, generator=_gen(70 + cols)) * 3).to(torch.float16).to(cuda_dev)
    _softmax_case(cuda_dev, f"rows={rows} cols={cols}", x)


def test_softmax_special_rows(cuda_dev):
    cols = 1000
    x = torch.randn(6, cols, generator=_gen(80)).to(torch.float16)
    x[0] = 2.5                                     # constant row
    x[1] = -30.0
    x[1, 417] = 0.0                                # one-hot after softmax
    x[2, 3] = 65504.0                              # +max fp16 beside ordinary values
    x[3] = -65504.0
    x[3, 999] = 65504.0
    x[4, ::3] = -65504.0                           # a third of the row at -max
    x[5] = 65504.0                                 # every entry at +max
    _softmax_case(cuda_dev, "constant / one-hot / +-65504 rows", x.to(cuda_dev))


def test_softmax_padded_rows_keep_padding(cuda_dev):
    rows, cols, ld = 33, 1000, 1032
    buf = (torch.randn(rows, ld, generator=_gen(81)) * 2).to(torch.float16).to(cuda_dev)
    buf[:, cols:] = 9.0                            # padding: a large value the row must not see
    x = buf.clone()
    out = torch.full_like(buf, -1.0)
    _softmax_abi(x, out, rows, cols, ld)
    ratio = AR.check(out[:, :cols], AR.softmax_ref(buf, cols), "ld > cols")
    _report("ap_softmax_rows_f16", "ld > cols (out of place)", ratio)
    assert (out[:, cols:] == -1.0).all() and torch.equal(x, buf)
    _softmax_abi(x, x, rows, cols, ld)             # in place
    assert torch.equal(x[:, :cols], out[:, :cols]) and (x[:, cols:] == 9.0).all()


def test_softmax_refuses_misaligned(cuda_dev):
    from aniportrait_b200 import _lib, ops
    flat = torch.zeros(4 * 128 + 8, dtype=torch.float16, device=cuda_dev)
    good = flat[:4 * 128]
    bad = flat[1:1 + 4 * 128]                      # 2-byte offset
    with pytest.raises(_lib.ApError, match="4-byte aligned"):
        ops.softmax_rows(bad.view(4, 128))
    with pytest.raises(_lib.ApError, match="4-byte aligned"):
        _softmax_abi(good, bad, 4, 128, 128)


def test_vae_mid_block_attention(cuda_dev):
    """models/vae.py::_mid_attn_run (GroupNorm -> q/k/v GEMMs -> ap_softmax_rows_f16 -> P.V GEMM -> out GEMM +
    residual) against float64 on the fp16 weights. The chain rounds to fp16 six times before the output (normalised x,
    q, k, the [n, n] scores, P, P.V); the score rounding is the largest: 2**-11 |s| in the logit, ~1e-2 relative in P at
    |s| ~ 20. So the attention branch b = (P.V).Wo^T is held to 2**-5 of its absolute-weighted sum
    (|P*| . |V*|) . |Wo|^T, and the output rounding to 2**-11 |o*|."""
    from aniportrait_b200.models.vae import _Attn, _mid_attn_run, _pack_attn
    torch.manual_seed(90)
    c, groups, nf, h, w = 512, 32, 2, 16, 16
    a = _Attn(c, groups)
    with torch.no_grad():
        for lin, std in ((a.to_q, 0.08), (a.to_k, 0.08), (a.to_v, 0.05), (a.to_out[0], 0.05)):
            lin.weight.normal_(0, std)
            lin.bias.normal_(0, 0.1)
        a.group_norm.weight.normal_(1, 0.2)
        a.group_norm.bias.normal_(0, 0.2)
    a = a.to(cuda_dev, torch.float16)
    x = (torch.randn(nf, h, w, c, generator=_gen(91)) * 1.5 + 0.3).to(torch.float16).to(cuda_dev)
    pk = _pack_attn(a)
    o1 = _mid_attn_run(x, pk, groups).clone()
    o2 = _mid_attn_run(x, pk, groups)
    assert torch.equal(o1, o2)

    P = {n: p.double() for n, p in a.named_parameters()}
    xd = x.double().view(nf, h * w, c)
    hn = torch.nn.functional.group_norm(xd.transpose(1, 2), groups, P["group_norm.weight"], P["group_norm.bias"],
                                        1e-6).transpose(1, 2)
    q = hn @ P["to_q.weight"].T + P["to_q.bias"]
    k = hn @ P["to_k.weight"].T + P["to_k.bias"]
    v = hn @ P["to_v.weight"].T + P["to_v.bias"]
    p = torch.softmax(q @ k.transpose(1, 2) * c ** -0.5, dim=-1)
    wo = P["to_out.0.weight"]
    ref = ((p @ v) @ wo.T + P["to_out.0.bias"] + xd).view(nf, h, w, c)
    branch_abs = ((p @ v.abs()) @ wo.abs().T).view(nf, h, w, c)
    bound = 2.0 ** -5 * branch_abs + 2.0 ** -11 * ref.abs() + 2.0 ** -24
    ratio = AR.check(o1.view(-1, c), AR.Ref(ref.view(-1, c), bound.view(-1, c),
                                            lambda r, col: dict(frame=r // (h * w), head=0, row=r % (h * w), col=col)),
                     "vae mid attention")
    _report("VAE _mid_attn_run (ap_softmax_rows_f16)", "2 frames 16x16 c=512", ratio)
