"""The call contract of the denoising-loop, layout and patchify kernels, element by element against float64
(denoise_reference.py), at the shapes their callers use:

  gather       ap_gather_window_f16: _window_step (dup 2, or 1 without CFG), _group_step (up to 4 windows in one call),
               _unit_step (one branch) of pipeline_pose2vid_long.py:297-343
  scatter      ap_scatter_accumulate_f16: the same callers, ld = the UNet output's width (4) and a padded 32 whose pad
               lanes hold NaN, group slices into one acc plane
  step         ap_cfg_ddim_step_f16: every step of 25 of inference_v2.yaml (v-prediction, zero terminal SNR, trailing:
               alpha_t = 0 at the first step), inference_v1.yaml (epsilon, leading, clip_sample) and `sample`, guidance
               1.0 / 3.5 / 7.5, weights 1, 1/2 and 1/3, |x0| on both sides of the clip range
  loop         gather -> stand-in denoiser -> scatter over every window -> step, every step, with and without CFG,
               against the reference loop (pipeline_pose2vid_long.py:459-559, which divides by the window count only
               under CFG), fed the kernel's latents each step
  layouts      ap_ncfhw_to_nhwc_f16 / ap_nhwc_to_ncfhw_f16 at every caller geometry; ap_patchify_nchw_f16 at ViT-L/14
  refusals     misaligned pointers and empty or too narrow sizes return AP_ERR_INVALID and write nothing

Geometries: the benchmark's L = 16 at 64x64 latents, pipeline_small's L = 20 at 16x16, a long video (L = 120 at 64x64),
HW = 13 x 17 (not a multiple of 256) with stride-2 windows that wrap around and repeat frames. Every C-ABI call writes
into a buffer with a guard band that must stay untouched, the inputs must be unchanged, and a call repeated on a second
copy of its in-place operands must give the same bits. The worst ratio of error to bound is printed per case (-s).
"""
import math

import pytest
import torch

import denoise_reference as DR
import gemm_reference as GR
from test_gemm_contract_gpu import _snapshot, _twice, _unchanged
from test_norm_contract_gpu import _abi, _f, _off

pytestmark = pytest.mark.gpu


def _report(family, name, ratio):
    print(f"\n[{family}] {name}: worst error / bound = {ratio:.3f}")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


GEOMS = {
    "bench_L16_64x64": dict(L=16, h=64, w=64, stride=1),
    "small_L20_16x16": dict(L=20, h=16, w=16, stride=1),
    "long_L120_64x64": dict(L=120, h=64, w=64, stride=1),
    "odd_L24_13x17_stride2": dict(L=24, h=13, w=17, stride=2),
}


def _windows(geom):
    from aniportrait_b200.pipelines.sharding import plan_windows
    g = GEOMS[geom]
    windows, inv = plan_windows(g["L"], 25, "uniform", 16, g["stride"], 4)
    return windows, inv


def test_geometries_cover_wrap_and_repeats():
    windows, inv = _windows("odd_L24_13x17_stride2")
    assert any(len(set(w)) < len(w) for w in windows), "a window with a repeated frame"
    assert any(w != sorted(w) for w in windows), "a window that wraps around"
    assert (inv < 1).any() and (inv == 1).any()
    assert (13 * 17) % 256 and len(_windows("long_L120_64x64")[0]) >= 8


def _idx(window, dev):
    return torch.tensor(window, dtype=torch.int32, device=dev)


def gather_call(lat_p, idx, out_p, dup, F, HW, cpad):
    from aniportrait_b200._lib import I, ptr
    _abi("ap_gather_window_f16", lat_p, ptr(idx), out_p, I(dup), I(F), I(HW), I(cpad))


def scatter_call(pred_p, ld, idx, acc_p, B, F, L, HW):
    from aniportrait_b200._lib import I, ptr
    _abi("ap_scatter_accumulate_f16", pred_p, I(ld), ptr(idx), acc_p, I(B), I(F), I(L), I(HW))


def step_call(acc_p, inv, cfg, g, a_t, a_p, pred, clip, lat_p, L, HW):
    from aniportrait_b200._lib import I, fptr
    _abi("ap_cfg_ddim_step_f16", acc_p, fptr(inv), I(1 if cfg else 0), _f(g), _f(a_t), _f(a_p), I(DR.PRED[pred]),
         _f(clip), lat_p, I(L), I(HW))


def _lat(L, HW, dev, seed, scale=1.0):
    return (scale * torch.randn(L, HW, 4, generator=_gen(seed))).half().to(dev)


# ---------------------------------------------------------------------------------------------------- gather
MODES = ["window", "window_no_cfg", "group", "unit"]


def _gather_plan(geom, mode):
    """(index list, dup) of each gather call the caller makes in one step."""
    windows, _ = _windows(geom)
    if mode == "group":       # _plan_groups: elements (window, branch), at most 4 per call, dup 1
        elems = [w for w in windows for _ in range(2)]
        return [(sum(elems[i:i + 4], []), 1) for i in range(0, len(elems), 4)]
    dup = 2 if mode == "window" else 1
    return [(w, dup) for w in windows]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_gather_window(cuda_dev, geom, mode):
    from aniportrait_b200._lib import ptr
    g = GEOMS[geom]
    L, HW, cpad = g["L"], g["h"] * g["w"], 64
    lat = _lat(L, HW, cuda_dev, 1)
    plan = _gather_plan(geom, mode)
    if len(plan) > 4:
        plan = plan[:2] + plan[-2:]
    for k, (window, dup) in enumerate(plan):
        idx = _idx(window, cuda_dev)
        F = len(window)
        out = GR.Guarded(dup * F * HW, cpad, cpad, torch.float16, cuda_dev)
        snap = _snapshot(lat, idx)
        _twice(lambda: gather_call(ptr(lat), idx, ptr(out.view), dup, F, HW, cpad), out, f"{geom} {mode} call {k}")
        _unchanged(snap, f"{geom} {mode}")
        GR.check_exact(out.view.cpu(), DR.gather_ref(lat.cpu(), window, dup, cpad), f"{geom} {mode} call {k}")
    _report("gather", f"{geom} {mode} ({len(plan)} calls)", 0.0)


# ---------------------------------------------------------------------------------------------------- scatter
def _scatter_plan(geom, mode, dev, seed=3):
    """[(pred tensor, window, first acc plane)] of one step's scatter calls, ld 4 (the UNet's conv_out width) or 32
    with NaN pad lanes ('unit')."""
    windows, _ = _windows(geom)
    g = GEOMS[geom]
    HW = g["h"] * g["w"]
    gen = _gen(seed)

    def pred(rows, ld):
        p = torch.randn(rows, HW, ld, generator=gen)
        p[..., 4:] = math.nan
        return p.half().to(dev)
    if mode in ("window", "window_no_cfg"):
        dup = 2 if mode == "window" else 1
        return [(pred(dup * len(w), 4), w, 0) for w in windows]
    if mode == "unit":
        return [(pred(len(w), 32), w, b) for w in windows for b in (0, 1)]
    calls = []
    elems = [(w, b) for w in windows for b in (0, 1)]
    for i in range(0, len(elems), 4):
        grp = sorted(elems[i:i + 4], key=lambda e: e[1])
        F = len(grp[0][0])
        p = pred(len(grp) * F, 4)
        calls += [(p[e * F:(e + 1) * F], w, b) for e, (w, b) in enumerate(grp)]
    return calls


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_scatter_accumulate(cuda_dev, geom, mode):
    from aniportrait_b200._lib import fptr, ptr
    g = GEOMS[geom]
    L, HW = g["L"], g["h"] * g["w"]
    P = 1 if mode == "window_no_cfg" else 2
    calls = _scatter_plan(geom, mode, cuda_dev)
    acc0 = 0.25 * torch.randn(P, L, HW, 4, generator=_gen(4))     # what earlier windows left
    bufs = []
    for _ in range(2):
        a = GR.Guarded(P * L * HW, 4, 4, torch.float32, cuda_dev)
        a.view.copy_(acc0.view(-1, 4))
        bufs.append(a)
    for k, (pred, window, p0) in enumerate(calls):
        idx = _idx(window, cuda_dev)
        B = pred.shape[0] // len(window)
        snap = _snapshot(pred, idx)
        for a in bufs:
            plane = a.view[p0 * L * HW:]
            scatter_call(ptr(pred), pred.shape[-1], idx, fptr(plane), B, len(window), L, HW)
        torch.cuda.synchronize()
        _unchanged(snap, f"{geom} {mode} call {k}")
    for a in bufs:
        a.check(f"{geom} {mode}")
    assert torch.equal(bufs[0].bits, bufs[1].bits), f"{geom} {mode}: two runs differ"
    cpu_calls = [(p.cpu(), w, p0) for p, w, p0 in calls]
    got = bufs[0].view.cpu()
    GR.check_exact(got, DR.exact_f32(DR.scatter_replay(acc0, cpu_calls), DR.locate_rows(L, HW, P)),
                   f"{geom} {mode}: fp32 replay")
    ratio = GR.check(got, DR.scatter_ref(acc0, cpu_calls), f"{geom} {mode}: fp64 sum")
    _report("scatter", f"{geom} {mode} ({len(calls)} calls)", ratio)


# ---------------------------------------------------------------------------------------------------- step
STEP_CASES = [(s, gs, geom) for s in DR.SCHEDULES for gs in (1.0, 3.5, 7.5)
              for geom in ("small_L20_16x16", "odd_L24_13x17_stride2")]


def _step_operands(L, HW, cfg, seed):
    """acc as the sum of `count` predictions, weights cycling 1, 1/2, 1/3."""
    cnt = torch.tensor([1.0, 2.0, 3.0]).repeat(L // 3 + 1)[:L]
    acc = torch.randn(2 if cfg else 1, L, HW, 4, generator=_gen(seed)) * cnt.view(1, -1, 1, 1)
    return acc.float(), (1.0 / cnt).float()


@pytest.mark.parametrize("sched,guidance,geom", STEP_CASES, ids=[f"{s}-g{g}-{m}" for s, g, m in STEP_CASES])
def test_cfg_ddim_step_every_step(cuda_dev, sched, guidance, geom):
    from aniportrait_b200._lib import fptr, ptr
    gm = GEOMS[geom]
    L, HW = gm["L"], gm["h"] * gm["w"]
    cfg = guidance > 1.0
    P = 2 if cfg else 1
    sch = DR.scheduler(sched)
    pred, clip = sch.config.prediction_type, DR.clip_of(sch)
    lat = _lat(L, HW, "cpu", 7, scale=1.5)
    worst, first, last = 0.0, None, None
    clipped = unclipped = 0
    for i, t in enumerate(int(x) for x in sch.timesteps):
        a_t, a_p = sch.alpha_pair(t)
        acc, inv = _step_operands(L, HW, cfg, 100 + i)
        inv_d = inv.to(cuda_dev)
        runs = []
        for _ in range(2):
            la = GR.Guarded(L * HW, 4, 4, torch.float16, cuda_dev)
            ac = GR.Guarded(P * L * HW, 4, 4, torch.float32, cuda_dev)
            la.view.copy_(lat.view(-1, 4))
            ac.view.copy_(acc.view(-1, 4))
            snap = _snapshot(inv_d)
            step_call(fptr(ac.view), inv_d, cfg, guidance, a_t, a_p, pred, clip, ptr(la.view), L, HW)
            torch.cuda.synchronize()
            _unchanged(snap, f"{sched} t={t}")
            la.check(f"{sched} t={t}: latents")
            ac.check(f"{sched} t={t}: acc")
            assert bool((ac.view == 0).all()), f"{sched} t={t}: acc not zeroed"
            runs.append(la)
        assert torch.equal(runs[0].bits, runs[1].bits), f"{sched} t={t}: two runs differ"
        ref = DR.step_ref(acc, inv, lat, guidance, a_t, a_p, pred, clip)
        out = runs[0].view.cpu()
        r = GR.check(out, ref, f"{sched} g={guidance} {geom} step {i} (t={t}, alpha_t={a_t:.6g}, alpha_prev={a_p:.6g})")
        worst = max(worst, r)
        first = r if first is None else first
        last = r
        if clip:
            x0 = DR.step_ref(acc, inv, lat, guidance, a_t, 1.0, pred, 0.0).o
            clipped += int((x0.abs() > clip).sum())
            unclipped += int((x0.abs() < clip).sum())
        lat = out.view(L, HW, 4)            # the kernel's latents feed the next step
    assert sch.alpha_pair(int(sch.timesteps[-1]))[1] == 1.0
    if sched == "v2_vpred_zero_snr":
        assert sch.alpha_pair(int(sch.timesteps[0]))[0] == 0.0
    if clip:
        assert clipped and unclipped, "x0 must fall on both sides of the clip range"
    assert worst > 0.0
    _report("cfg_ddim_step", f"{sched} g={guidance} {geom} (first step {first:.3f}, last step {last:.3f})", worst)


# ---------------------------------------------------------------------------------------------------- loop
def _denoiser(x, dup, F, HW, ld=4):
    """Stand-in for the UNet: a fixed fp16 function of the gathered window (per branch, with a window mean)."""
    xv = x[..., :4].float().view(dup, F, HW, 4)
    k = torch.tensor([1.3, 0.7], device=x.device)[:dup].view(dup, 1, 1, 1)
    p = torch.sin(xv * k) + 0.3 * xv.mean(dim=1, keepdim=True) - 0.2 * xv
    out = torch.empty(dup * F, HW, ld, dtype=torch.float16, device=x.device)
    out[..., :4] = p.reshape(dup * F, HW, 4).half()
    return out


LOOP_CASES = [("bench_L16_64x64", "v2_vpred_zero_snr"), ("small_L20_16x16", "v2_vpred_zero_snr"),
              ("small_L20_16x16", "v1_epsilon_clip"), ("long_L120_64x64", "v2_vpred_zero_snr"),
              ("odd_L24_13x17_stride2", "v2_vpred_zero_snr")]


@pytest.mark.parametrize("guidance", [1.0, 3.5])
@pytest.mark.parametrize("geom,sched", LOOP_CASES, ids=[f"{g}-{s}" for g, s in LOOP_CASES])
def test_denoising_loop_against_reference_loop(cuda_dev, geom, sched, guidance):
    from aniportrait_b200 import ops
    from aniportrait_b200.pipelines.sharding import step_weights
    gm = GEOMS[geom]
    L, h, w = gm["L"], gm["h"], gm["w"]
    HW = h * w
    windows, inv = _windows(geom)
    cfg = guidance > 1.0
    dup = 2 if cfg else 1
    sch = DR.scheduler(sched)
    pred_type, clip = sch.config.prediction_type, DR.clip_of(sch)
    lat = torch.randn(L, h, w, 4, generator=_gen(21)).half().to(cuda_dev)
    acc = torch.zeros(dup, L, h, w, 4, dtype=torch.float32, device=cuda_dev)
    weights = step_weights(inv, cfg).to(cuda_dev, torch.float32)
    idxs = [_idx(wd, cuda_dev) for wd in windows]
    worst = 0.0
    for i, t in enumerate(int(x) for x in sch.timesteps):
        lat_in = lat.cpu().view(L, HW, 4)
        preds = []
        for wd, idx in zip(windows, idxs):
            x = ops.gather_window(lat, idx, dup, 64)
            assert torch.equal(x.view(dup, len(wd), h, w, 64)[..., :4], lat[wd].unsqueeze(0).expand(dup, -1, -1, -1, -1))
            p = _denoiser(x, dup, len(wd), HW).view(dup * len(wd), h, w, 4)
            ops.scatter_accumulate(p, idx, acc)
            preds.append(p.view(-1, HW, 4).cpu())
        a_t, a_p = sch.alpha_pair(t)
        ops.cfg_ddim_step(acc, weights, guidance, a_t, a_p, lat, pred_type, clip)
        ref = DR.reference_loop_step(preds, windows, lat_in, guidance, a_t, a_p, pred_type, clip)
        worst = max(worst, GR.check(lat.cpu().view(-1, 4), ref, f"{geom} {sched} g={guidance} step {i} (t={t})"))
        assert bool((acc == 0).all())
    assert worst > 0.0
    _report("loop", f"{geom} {sched} g={guidance} ({len(windows)} windows, 25 steps)", worst)


# ---------------------------------------------------------------------------------------------------- layouts
TO_NHWC = [  # (name, B, C, F, H, W, cpad)
    ("unet_conv_in_F16_64x64", 2, 4, 16, 64, 64, 64),          # unet_3d.py:304
    ("reference_net_64x64", 2, 4, 1, 64, 64, 64),              # unet_2d_condition.py:136
    ("vae_encode_512", 2, 3, 1, 512, 512, 64),                 # vae.py:307
    ("vae_decode_64x64", 4, 4, 1, 64, 64, 64),                 # vae.py:318
    ("pose_guider_512", 4, 3, 1, 512, 512, 8),                 # pose_guider.py:148
    ("odd_13x17", 2, 4, 3, 13, 17, 64),
]
TO_NCFHW = [  # (name, B, C, F, H, W, ld)
    ("unet_out_F16_64x64", 2, 4, 16, 64, 64, 4),               # unet_3d.py:313
    ("vae_encode_moments_64x64", 2, 8, 1, 64, 64, 8),          # vae.py:310
    ("vae_decode_512", 2, 3, 1, 512, 512, 3),                  # vae.py:322
    ("ld_32_over_4_odd_13x17", 2, 4, 3, 13, 17, 32),
]


@pytest.mark.parametrize("case", TO_NHWC, ids=[c[0] for c in TO_NHWC])
def test_ncfhw_to_nhwc(cuda_dev, case):
    from aniportrait_b200._lib import I, ptr
    name, B, C, F, H, W, cpad = case
    x = torch.randn(B, C, F, H, W, generator=_gen(31)).half().to(cuda_dev)
    out = GR.Guarded(B * F * H * W, cpad, cpad, torch.float16, cuda_dev)
    snap = _snapshot(x)
    _twice(lambda: _abi("ap_ncfhw_to_nhwc_f16", ptr(x), ptr(out.view), I(B), I(C), I(F), I(H * W), I(cpad)), out, name)
    _unchanged(snap, name)
    GR.check_exact(out.view.cpu(), DR.ncfhw_to_nhwc_ref(x.cpu(), cpad), name)
    _report("ncfhw_to_nhwc", name, 0.0)


@pytest.mark.parametrize("case", TO_NCFHW, ids=[c[0] for c in TO_NCFHW])
def test_nhwc_to_ncfhw(cuda_dev, case):
    from aniportrait_b200._lib import I, ptr
    name, B, C, F, H, W, ld = case
    x = torch.randn(B * F, H, W, ld, generator=_gen(32))
    x[..., C:] = math.nan                  # channels past C must not be read
    x = x.half().to(cuda_dev)
    out = GR.Guarded(B * C * F * H, W, W, torch.float16, cuda_dev)
    snap = _snapshot(x)
    _twice(lambda: _abi("ap_nhwc_to_ncfhw_f16", ptr(x), ptr(out.view), I(B), I(C), I(F), I(H * W), I(ld)), out, name)
    _unchanged(snap, name)
    GR.check_exact(out.view.cpu(), DR.nhwc_to_ncfhw_ref(x.cpu(), B, C, F), name)
    _report("nhwc_to_ncfhw", name, 0.0)


@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_patchify_vit_l14(cuda_dev, dtype, B):
    """ViT-L/14 at 224 x 224 (kpad 640). B = 16 needs more threads than the grid's num_sms * 8 blocks of 256: the
    grid-stride loop wraps."""
    from aniportrait_b200 import ops
    from aniportrait_b200._lib import I, ptr
    P, S = 14, 224
    kpad = ops.patch_kpad(P)
    tokens = 1 + (S // P) ** 2
    assert kpad == 640
    if B == 16:
        sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
        assert B * tokens * kpad // 8 > sms * 8 * 256
    px = (2.0 * torch.randn(B, 3, S, S, generator=_gen(40 + B))).to(cuda_dev, dtype)
    out = GR.Guarded(B * tokens, kpad, kpad, torch.float16, cuda_dev)
    name = f"vit_l14_{str(dtype)[6:]}_B{B}"
    snap = _snapshot(px)
    _twice(lambda: _abi("ap_patchify_nchw_f16", ptr(px), I(1 if dtype == torch.float32 else 0), I(B), I(S), I(S), I(P),
                        ptr(out.view), I(kpad)), out, name)
    _unchanged(snap, name)
    GR.check_exact(out.view.cpu(), DR.patchify_ref(px.cpu(), P, kpad), name)
    _report("patchify", name, 0.0)


# ---------------------------------------------------------------------------------------------------- refusals
def _refusal(dev, name, off):
    """(Guarded buffer that must stay untouched, call) for one refused argument of a denoising-loop entry point."""
    from aniportrait_b200._lib import fptr, ptr
    L, HW, F = 6, 64, 4
    lat = _lat(L, HW, dev, 50)
    idx = _idx([0, 1, 2, 3], dev)
    entry, arg = name.split(":")
    if entry == "gather":
        out = GR.Guarded(2 * F * HW, 64, 64, torch.float16, dev, pre=64 + (off if arg == "out" else 0))
        src = _off(lat, off) if arg == "latents" else lat
        dup, Fc, HWc, cpad = 2, F, HW, 64
        if arg == "dup":
            dup = 0
        elif arg == "F":
            Fc = 0
        elif arg == "HW":
            HWc = 0
        elif arg == "cpad":
            cpad = 4
        return out, lambda: gather_call(ptr(src), idx, ptr(out.view), dup, Fc, HWc, cpad)
    if entry == "scatter":
        acc = GR.Guarded(2 * L * HW, 4, 4, torch.float32, dev, pre=64 + (off if arg == "acc" else 0))
        pred = torch.randn(2 * F, HW, 4, generator=_gen(51)).half().to(dev)
        B, Fc, Lc, HWc, ld = 2, F, L, HW, 4
        if arg == "ld":
            ld = 3
        elif arg == "B":
            B = 0
        elif arg == "F":
            Fc = 0
        elif arg == "L":
            Lc = 0
        elif arg == "HW":
            HWc = 0
        return acc, lambda: scatter_call(ptr(pred), ld, idx, fptr(acc.view), B, Fc, Lc, HWc)
    if entry == "step":
        la = GR.Guarded(L * HW, 4, 4, torch.float16, dev)
        acc = torch.zeros(2, L, HW, 4, device=dev)
        inv = torch.ones(L, device=dev)
        Lc, HWc, pred, a_t = L, HW, "v_prediction", 0.5
        if arg == "L":
            Lc = 0
        elif arg == "HW":
            HWc = 0
        elif arg == "epsilon_alpha0":
            pred, a_t = "epsilon", 0.0
        elif arg == "sample_alpha1":
            pred, a_t = "sample", 1.0
        return la, lambda: step_call(fptr(acc), inv, True, 3.5, a_t, 0.7, pred, 0.0, ptr(la.view), Lc, HWc)
    raise KeyError(name)


MISALIGNED = ["gather:latents", "gather:out", "scatter:acc"]
BAD_SIZES = ["gather:dup", "gather:F", "gather:HW", "gather:cpad", "scatter:ld", "scatter:B", "scatter:F", "scatter:L",
             "scatter:HW", "step:L", "step:HW", "step:epsilon_alpha0", "step:sample_alpha1"]


def _refused(dev, name, off):
    from aniportrait_b200._lib import ApError
    buf, call = _refusal(dev, name, off)
    torch.cuda.synchronize()
    with pytest.raises(ApError, match=r"rc=-1\)"):
        call()
    torch.cuda.synchronize()
    buf.check(name)
    assert bool((buf.bits == buf.sentinel).all()), f"{name}: the buffer was written"


@pytest.mark.parametrize("off", [1, 2])
@pytest.mark.parametrize("name", MISALIGNED)
def test_misaligned_refusal(cuda_dev, name, off):
    """gather loads latents as uint2 and stores uint4; scatter read-modify-writes acc as float4: a pointer one or two
    elements off that grid is refused with AP_ERR_INVALID before any launch."""
    _refused(cuda_dev, name, off)


@pytest.mark.parametrize("name", BAD_SIZES)
def test_bad_size_refusal(cuda_dev, name):
    """Empty sizes (a grid of 0 blocks), ld < 4 and the coefficient singularities are refused before any launch."""
    _refused(cuda_dev, name, 0)
