"""fp64 references, per-element bounds and fp32 emulations of the multistep-sampler kernels (csrc/ap_misc.cu:
ap_cfg_multistep_step_f16, ap_gather_window_scaled_f16), in the style of denoise_reference.py. Imported by the CPU
checker tests and the GPU tests; not a conftest. The checks and `Ref` are those of gemm_reference.py; u = 2**-24.

Multistep step (bounded)
------------------------
With the fp64 coefficients of pipelines/scheduler.py::multistep_coefficients (the kernel receives each rounded once to
fp32: relative error u), the fp32 acc and weights, the fp16 latents x and the fp32 history h the kernel read:
  v* as in denoise_reference (CFG: u* + g (c* - u*), else acc w), with its error bound e_v
  m* = c_xx x + c_xv v*                  e_m = u (|c_xx x| + |c_xv v*|) + |c_xv| e_v + u (|c_xx x| + |c_xv v*| + |m*|)
  y* = k_x x + k_0 m* + k_1 h            T = |k_x x| + |k_0 m*| + |k_1 h|
                                         e_y = u T + |k_0| e_m + |k_1| e_h + u (2 T + |y*|)
(coefficient roundings, the error carried in, then three products and two sums, each one rounding whether or not nvcc
contracts them into FMAs), times SECOND_ORDER; latents: then the fp16 output rounding OUT_REL |y*| + OUT_FLOOR. The
stored history is m in fp32: bound e_m. Where k_1 = 0 the history is not an input at all: a NaN there must not reach the
output.

Scaled gather (bounded)
-----------------------
out = fp16_rn(fp32(x) * fp32(s)): |out - x s| <= 2 u |x s| + OUT_REL |x s| + OUT_FLOOR, lanes 4..Cpad exactly 0.

Emulations
----------
`emulate_step` / `emulate_gather_scaled` reproduce the kernels in fp32 numpy; `bug=` turns them into models of kernel
mistakes ('hist_not_updated', 'hist_read_at_k1_zero', 'scale_missing'), and `planted_table` turns a correct coefficient
table into models of host mistakes ('order2_first_step', 'r0_inverted'). The checks must reject every one.
"""
from __future__ import annotations

import copy

import numpy as np
import torch

from denoise_reference import _exact_v, locate_rows
from gemm_reference import E24, OUT_FLOOR, OUT_REL, SECOND_ORDER, Ref

# The two families in the configurations the pipeline goldens use, and the variants the CPU table test sweeps
BASE = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", steps_offset=1)


def make_scheduler(cls_name, steps, **kw):
    from aniportrait_b200.pipelines import scheduler as S
    s = getattr(S, cls_name)(**dict(BASE, **kw))
    s.set_timesteps(steps)
    return s


def _f32(c) -> float:
    return float(np.float32(c))


def step_ref(acc, w, lat, hist, guidance, coef, cfg=None, hist_err=None):
    """fp64 reference of ap_cfg_multistep_step_f16 on its own inputs. acc [B, L, HW, 4] fp32, w [L] fp32, lat [L, HW, 4]
    fp16, hist [L, HW, 4] fp32 (the values the kernel read; None when k_1 = 0), hist_err: an absolute error bound carried
    in with hist. Returns (Ref of the latents, Ref of the stored history m)."""
    acc = acc.double().cpu()
    B, L, HW, _ = acc.shape
    cfg = (B == 2) if cfg is None else cfg
    w = w.double().cpu().reshape(-1)
    x = lat.double().cpu().reshape(-1, 4)
    g = float(guidance)
    v, _, _, acu = _exact_v(acc, w, g, cfg)
    e_br = E24 * (acc * w.view(1, -1, 1, 1)).abs().reshape(B, -1, 4)
    if cfg:
        e_v = e_br[0] + abs(g) * (e_br[0] + e_br[1]) + 2 * E24 * abs(g) * acu + E24 * v.abs()
    else:
        e_v = e_br[0]
    cxx, cxv, kx, k0, k1 = coef.c_xx, coef.c_xv, coef.k_x, coef.k_0, coef.k_1
    m = cxx * x + cxv * v
    tm = abs(cxx) * x.abs() + abs(cxv) * v.abs()
    e_m = E24 * tm + abs(cxv) * e_v + E24 * (tm + m.abs())
    h = torch.zeros_like(x) if k1 == 0 else hist.double().cpu().reshape(-1, 4)
    eh = torch.zeros_like(x) if (hist_err is None or k1 == 0) else hist_err.double().cpu().reshape(-1, 4)
    y = kx * x + k0 * m + k1 * h
    T = abs(kx) * x.abs() + abs(k0) * m.abs() + abs(k1) * h.abs()
    pre = (E24 * T + abs(k0) * e_m + abs(k1) * eh + E24 * (2 * T + y.abs())) * SECOND_ORDER
    loc = locate_rows(L, HW)
    return (Ref(y, pre + OUT_REL * y.abs() + OUT_FLOOR, loc, pre=pre),
            Ref(m, e_m * SECOND_ORDER + 1e-300, loc, out_f32=True))


def emulate_step(acc, w, lat, hist, guidance, coef, fma=False, bug=None):
    """ap_cfg_multistep_step_f16 in fp32 numpy. Returns (latents fp16 [L*HW, 4], unrounded fp32, history after the
    call fp32 [L*HW, 4]). hist: fp32 [L, HW, 4] before the call."""
    acc = acc.float().cpu().numpy()
    B = acc.shape[0]
    ww = w.float().cpu().numpy().reshape(1, -1, 1, 1).astype(np.float32)
    x = lat.half().float().cpu().numpy().reshape(-1, 4)
    h_in = hist.float().cpu().numpy().reshape(-1, 4)
    g = np.float32(guidance)
    if B == 2:
        u, c = (acc[0] * ww[0]).astype(np.float32), (acc[1] * ww[0]).astype(np.float32)
        v = (u + (g * (c - u)).astype(np.float32)).astype(np.float32)
    else:
        v = (acc[0] * ww[0]).astype(np.float32)
    v = v.reshape(-1, 4)
    cxx, cxv, kx, k0, k1 = (np.float32(_f32(c)) for c in (coef.c_xx, coef.c_xv, coef.k_x, coef.k_0, coef.k_1))

    def mad(p, q, r, s):
        if fma:
            return (np.float64(p) * q.astype(np.float64) + (r * s).astype(np.float32)).astype(np.float32)
        return ((p * q).astype(np.float32) + (r * s).astype(np.float32)).astype(np.float32)
    m = mad(cxx, x, cxv, v)
    y = mad(kx, x, k0, m)
    if k1 != 0 or bug == "hist_read_at_k1_zero":
        y = (y + (k1 * h_in).astype(np.float32)).astype(np.float32)
    h_out = h_in.copy()
    if coef.store and bug != "hist_not_updated":
        h_out = m.copy()
    y32 = torch.from_numpy(y)
    return y32.half(), y32, torch.from_numpy(h_out)


def gather_scaled_ref(lat, idx, dup, cpad, scale) -> Ref:
    """UNet input [(dup F) HW, cpad] of one window times `scale` (fp64 from the scheduler), fp16 lanes 0..3, 0 after."""
    lat = lat.cpu()
    L, HW, _ = lat.shape
    F = len(idx)
    o = torch.zeros(dup, F, HW, cpad, dtype=torch.float64)
    o[:, :, :, :4] = lat[list(idx)].double().unsqueeze(0) * float(scale)
    o = o.reshape(-1, cpad)
    bound = (2 * E24 + OUT_REL) * o.abs() + OUT_FLOOR
    bound[:, 4:] = 1e-300                 # the padding lanes must be exactly 0

    def locate(r, c):
        d, rem = divmod(r, F * HW)
        f, px = divmod(rem, HW)
        return f"dup plane {d}, window frame {f} (latent frame {idx[f]}), pixel {px}, lane {c}"
    return Ref(o, bound, locate)


def emulate_gather_scaled(lat, idx, dup, cpad, scale, bug=None):
    lat = lat.cpu()
    F = len(idx)
    s = np.float32(1.0 if bug == "scale_missing" else _f32(scale))
    xs = (lat[list(idx)].float().numpy() * s).astype(np.float32)
    o = torch.zeros(dup, F, lat.shape[1], cpad, dtype=torch.float16)
    o[:, :, :, :4] = torch.from_numpy(xs).half().unsqueeze(0)
    return o.reshape(-1, cpad)


def planted_table(table, bug):
    """A correct multistep_coefficients table turned into a model of a host mistake (midpoint DPM tables only):
    'order2_first_step' (the order counter starts at 1: the first step reads the history, with the next step's r0),
    'r0_inverted' (every second-order step uses 1 / r0)."""
    t = copy.deepcopy(table)
    second = [i for i, c in enumerate(t) if c.k_1 != 0]
    assert second, "the table has no second-order step"
    if bug == "order2_first_step":
        c1 = t[second[0]]
        e1 = -(c1.k_0 + c1.k_1)
        r0 = e1 / (2 * c1.k_1)
        e0 = -t[0].k_0
        t[0].k_1 = e0 / (2 * r0)
        t[0].k_0 = -e0 - t[0].k_1
    elif bug == "r0_inverted":
        for i in second:
            e = -(t[i].k_0 + t[i].k_1)
            r0 = e / (2 * t[i].k_1)
            t[i].k_1 = e * r0 / 2
            t[i].k_0 = -e - t[i].k_1
    else:
        raise ValueError(bug)
    return t


def stand_in_denoiser(x_in: torch.Tensor, t: float) -> torch.Tensor:
    """A fixed smooth function of the (scaled) UNet input and the timestep, fp64 [..., 4] -> [..., 4]."""
    return torch.sin(1.3 * x_in) - 0.2 * x_in + 1e-3 * t


def loop_check(sched_factory, guidance, table, bug=None, seed=0, L=3, HW=8):
    """A whole sampling run with the kernels' fp32 emulations (gather, stand-in denoiser, step), checked step by step
    against the scheduler object's own scale_model_input / step() in fp64 fed the emulation's latents (its history is
    the scheduler's, built from the same latents and predictions). table: the coefficients the emulation uses.
    Returns the worst ratio of error to bound; raises AssertionError at the first element out of bound."""
    import gemm_reference as GR
    sched = sched_factory()
    sched.sigmas = sched.sigmas.double()
    cfg = guidance > 1.0
    g = torch.Generator().manual_seed(seed)
    lat = (torch.randn(L, HW, 4, generator=g) * float(getattr(sched, "init_noise_sigma", 1.0))).half()
    hist = torch.full((L, HW, 4), float("nan"), dtype=torch.float32)
    w = torch.ones(L, dtype=torch.float32)
    e_hist = None
    worst = 0.0
    for i, t in enumerate(sched.timesteps):
        co = table[i]
        x_in = emulate_gather_scaled(lat, list(range(L)), 1, 4, co.scale, bug if bug == "scale_missing" else None)
        gref = gather_scaled_ref(lat, list(range(L)), 1, 4, co.scale)
        gref.o = sched.scale_model_input(lat.double(), t).reshape(-1, 4)       # the scheduler's own input scaling
        worst = max(worst, GR.check(x_in.double(), gref, f"step {i} (t={float(t):.4g}): scaled UNet input"))
        x_in = x_in.double().reshape(L, HW, 4)
        pu = stand_in_denoiser(x_in, float(t))
        pc = stand_in_denoiser(0.9 * x_in, float(t))
        acc = torch.stack([pu, pc] if cfg else [pc]).float()
        a64 = acc.double()
        v = a64[0] + guidance * (a64[1] - a64[0]) if cfg else a64[0]
        want = sched.step(v, t, lat.double()).prev_sample.reshape(-1, 4)
        ref, mref = step_ref(acc, w, lat, hist, guidance, co, hist_err=e_hist)
        ref.o = want
        y16, _, h_out = emulate_step(acc, w, lat, hist, guidance, co, bug=bug)
        worst = max(worst, GR.check(y16.double(), ref, f"step {i} (t={float(t):.4g})"))
        lat = y16.view(L, HW, 4)
        hist = h_out.view(L, HW, 4)
        e_hist = mref.bound
    return worst


def oracle_denoise_loop(sd_unet, sd_ref, sd_pose, latents, ref_latents, clip_embed, pose_cond, steps, sched, guidance,
                        c, context_frames=16, context_overlap=4):
    """oracle.functional.denoise_loop with any scheduler object, in the reference's call order
    (pipeline_pose2vid_long.py:373-559): set_timesteps, initial noise times init_noise_sigma, then per step the windows'
    UNet calls on scale_model_input(latents), overlap average, CFG and scheduler.step. latents: the unscaled initial
    noise. Returns the latents after every step."""
    from oracle import functional as OF
    ehs = torch.cat([torch.zeros_like(clip_embed), clip_embed], 0).unsqueeze(1)
    banks = OF.reference_unet_banks(sd_ref, ref_latents.repeat(2, 1, 1, 1), ehs, c=c)
    sched.set_timesteps(steps)
    latents = latents * sched.init_noise_sigma
    L = latents.shape[2]
    windows = OF.context_windows(L, context_frames, context_overlap)
    trace = []
    for t in sched.timesteps:
        noise = torch.zeros(2, *latents.shape[1:], dtype=latents.dtype)
        counter = torch.zeros(1, 1, L, 1, 1, dtype=latents.dtype)
        for wdw in windows:
            lat = sched.scale_model_input(latents[:, :, wdw].repeat(2, 1, 1, 1, 1), t)
            pose_fea = OF.pose_guider_forward(sd_pose, pose_cond[:, :, wdw].repeat(2, 1, 1, 1, 1),
                                              c0=c["block_out_channels"][0])
            noise[:, :, wdw] += OF.unet3d_forward(sd_unet, lat, t.reshape(1), ehs, pose_fea, banks, cfg=True, c=c)
            counter[:, :, wdw] += 1
        u, cnd = (noise / counter).chunk(2)
        latents = sched.step(u + guidance * (cnd - u), t, latents).prev_sample
        trace.append(latents)
    return trace
