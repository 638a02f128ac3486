"""CPU checks of the per-element attention checker in attention_reference.py: the fp32 emulations of the three
attention kernels pass it with room to spare, modelled kernel bugs fail it, and the fp64 spatial reference agrees with
the reference project's own formulation (torch.cat of own keys and bank, then SDPA)."""
import pytest
import torch
import torch.nn.functional as F

import attention_reference as AR


def _heads_buf(rows, heads, d, dpad, n, g, sigma=1.5):
    """n fp16 [rows, heads*dpad] matrices of N(0, sigma^2) values with each head zero padded from d to dpad."""
    t = torch.zeros(rows, n, heads, dpad)
    t[..., :d] = torch.randn(rows, n, heads, d, generator=g) * sigma
    t = t.to(torch.float16).reshape(rows, n * heads * dpad)
    return [t[:, i * heads * dpad:(i + 1) * heads * dpad] for i in range(n)]


def _spatial_case(frames=4, tokens=200, heads=2, d=40, n_banks=2, bank_tokens=150, first=2, fpb=1, sigma=1.5,
                  seed=0):
    dpad = (d + 63) // 64 * 64
    g = torch.Generator().manual_seed(seed)
    q, k, v = _heads_buf(frames * tokens, heads, d, dpad, 3, g, sigma)
    kw = dict(n_frames=frames, tokens=tokens, heads=heads, d=d, dpad=dpad)
    if n_banks:
        bk, bv = _heads_buf(n_banks * bank_tokens, heads, d, dpad, 2, g, sigma)
        kw.update(bank_k=bk, bank_v=bv, bank_tokens=bank_tokens, n_banks=n_banks, first_bank_frame=first,
                  frames_per_bank=fpb)
    return (q, k, v), kw


SPATIAL_CASES = {
    "cfg_two_banks": dict(),
    "d64_one_row_tiles": dict(frames=2, tokens=257, heads=2, d=64, n_banks=0),
    "dpad192_bank": dict(frames=3, tokens=100, heads=1, d=160, n_banks=1, bank_tokens=70, first=1, fpb=2),
    "d88_grouped": dict(frames=4, tokens=130, heads=2, d=88, n_banks=1, bank_tokens=130, first=2, fpb=2),
}


@pytest.mark.parametrize("name", list(SPATIAL_CASES))
def test_spatial_emulation_within_bound(name):
    args, kw = _spatial_case(**SPATIAL_CASES[name])
    ref = AR.spatial_ref(*args, **kw)
    ratio = AR.check(AR.spatial_emulate(*args, **kw), ref, name)
    print(f"spatial emulation {name}: worst error / bound = {ratio:.3f}")
    assert ratio <= 0.5


@pytest.mark.parametrize("B,Fr,N,C,heads", [(2, 9, 5, 320, 8), (1, 16, 3, 640, 8), (1, 20, 4, 640, 8),
                                             (2, 32, 2, 320, 5)])
def test_temporal_emulation_within_bound(B, Fr, N, C, heads):
    g = torch.Generator().manual_seed(1)
    qkv = (torch.randn(B * Fr * N, 3 * C, generator=g) * 1.5).to(torch.float16)
    ratio = AR.check(AR.temporal_emulate(qkv, B, Fr, N, C, heads), AR.temporal_ref(qkv, B, Fr, N, C, heads))
    path = "mma.sync" if AR.temporal_mma_path(Fr, C, heads) else "scalar"
    print(f"temporal emulation ({path}) B={B} F={Fr} N={N} C={C} heads={heads}: worst error / bound = {ratio:.3f}")
    assert ratio <= 0.5


def test_softmax_emulation_within_bound():
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(64, 1000, generator=g) * 4).to(torch.float16)
    x[3] = 65504.0
    x[4, ::2] = -65504.0
    ratio = AR.check(AR.softmax_emulate(x, 1000), AR.softmax_ref(x, 1000))
    print(f"softmax emulation: worst error / bound = {ratio:.3f}")
    assert ratio <= 0.5


# each modelled bug: (emulation bug name, case overrides). Ragged-tail bugs need a key count that is not a multiple of
# the 128-key tile; the dropped-rescale bug needs several key tiles; the one-row bug needs peaked attention (sigma 2),
# so that rows exist whose output is close to the absolute-weighted mean the bound scales with.
SPATIAL_BUGS = {
    "bank_index": ("bank_index", dict()),
    "first_bank_frame": ("first_bank_frame", dict()),
    "own_tail_next": ("tail_next", dict(n_banks=0, sigma=1.0)),
    "own_tail_zero": ("tail_zero", dict(frames=2, n_banks=0, sigma=1.0)),
    "bank_tail_next": ("tail_next", dict(tokens=256, sigma=1.0)),
    "bank_tail_zero": ("tail_zero", dict(tokens=256, n_banks=1, fpb=2, sigma=1.0)),
    "scale_dpad": ("scale_dpad", dict()),
    "lazy_rescale": ("lazy_rescale", dict(tokens=300, n_banks=0)),
    "row_1pct": ("row", dict(sigma=2.0)),
}


@pytest.mark.parametrize("name", list(SPATIAL_BUGS))
def test_checker_rejects_spatial_bug(name):
    bug, over = SPATIAL_BUGS[name]
    args, kw = _spatial_case(**over)
    ref = AR.spatial_ref(*args, **kw)
    ratio, loc, _ = AR.worst(AR.spatial_emulate(*args, **kw, bug=bug), ref)
    print(f"modelled bug {name}: rejected, worst ratio {ratio:.3g} at {loc}")
    assert ratio > 1.0
    if bug == "row":
        assert loc["frame"] == kw["n_frames"] - 1 and loc["row"] == kw["tokens"] // 2


def test_checker_rejects_temporal_unmasked_frames():
    g = torch.Generator().manual_seed(3)
    for B, Fr, N, C in [(1, 9, 4, 320), (1, 20, 4, 640)]:
        qkv = torch.randn(B * Fr * N, 3 * C, generator=g).to(torch.float16)
        ref = AR.temporal_ref(qkv, B, Fr, N, C, 8)
        AR.check(AR.temporal_emulate(qkv, B, Fr, N, C, 8), ref)
        ratio, loc, _ = AR.worst(AR.temporal_emulate(qkv, B, Fr, N, C, 8, bug="frames"), ref)
        print(f"modelled bug unmasked key frames (F={Fr}): rejected, worst ratio {ratio:.3g} at {loc}")
        assert ratio > 1.0


def test_checker_rejects_softmax_padded_column():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(16, 136, generator=g).to(torch.float16)   # cols = 128, ld = 136: the padding holds data too
    ref = AR.softmax_ref(x, 128)
    AR.check(AR.softmax_emulate(x, 128), ref)
    ratio, loc, _ = AR.worst(AR.softmax_emulate(x, 128, bug="pad"), ref)
    print(f"modelled bug softmax sums a padded column: rejected, worst ratio {ratio:.3g} at {loc}")
    assert ratio > 1.0


def test_checker_reports_location_and_rejects_nan():
    args, kw = _spatial_case(n_banks=0)
    ref = AR.spatial_ref(*args, **kw)
    out = AR.spatial_emulate(*args, **kw)
    out[kw["tokens"] + 7, 1 * kw["d"] + 5] = float("nan")
    with pytest.raises(AssertionError, match=r"'frame': 1, 'head': 1, 'row': 7, 'col': 5"):
        AR.check(out, ref, "nan")


@pytest.mark.parametrize("cfg", [True, False])
def test_spatial_ref_matches_reference_formulation(cfg):
    """The reference's read-mode block (mutual_self_attention.py:147-188) in float64: own tokens concatenated with the
    bank repeated per frame, SDPA, and under CFG the first half of the batch redone on its own tokens only. The kernel
    call for the same layout passes only the conditional half of the banks (models/blocks.py)."""
    b, video_length, tokens, heads, d = 2, 3, 24, 2, 16
    batch = 2 * b if cfg else b
    g = torch.Generator().manual_seed(5)
    x = torch.randn(batch * video_length, tokens, 3, heads, d, generator=g).to(torch.float16)
    bank = torch.randn(batch, tokens, 2, heads, d, generator=g).to(torch.float16)   # one bank per batch element

    def sdpa(qh, kh, vh):   # [frames, n, heads, d] -> same
        return F.scaled_dot_product_attention(qh.transpose(1, 2), kh.transpose(1, 2), vh.transpose(1, 2)).transpose(1, 2)

    xd, bd = x.double(), bank.double()
    bank_fea = [t.unsqueeze(1).repeat(1, video_length, 1, 1, 1).reshape(-1, tokens, heads, d)
                for t in (bd[:, :, 0], bd[:, :, 1])]
    k_all = torch.cat([xd[:, :, 1], bank_fea[0]], dim=1)
    v_all = torch.cat([xd[:, :, 2], bank_fea[1]], dim=1)
    want = sdpa(xd[:, :, 0], k_all, v_all)
    first = 0
    if cfg:
        half = batch * video_length // 2
        want[:half] = sdpa(xd[:half, :, 0], xd[:half, :, 1], xd[:half, :, 2])
        first = half
    rows = batch * video_length * tokens
    flat = x.reshape(rows, 3 * heads * d)
    hp = heads * d
    nb0 = batch // 2 if cfg else 0
    bflat = bank[nb0:].reshape(-1, 2 * hp)
    ref = AR.spatial_ref(flat[:, :hp], flat[:, hp:2 * hp], flat[:, 2 * hp:], batch * video_length, tokens, heads, d, d,
                         bank_k=bflat[:, :hp], bank_v=bflat[:, hp:], bank_tokens=tokens, n_banks=batch - nb0,
                         first_bank_frame=first, frames_per_bank=video_length)
    err = (ref.o - want.reshape(rows, hp)).abs().max().item()
    assert err < 1e-12, err
