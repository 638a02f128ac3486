"""fp64 references, per-element bounds and fp32 emulations of the denoising-loop and layout kernels (csrc/ap_misc.cu:
ap_gather_window_f16, ap_scatter_accumulate_f16, ap_cfg_ddim_step_f16, ap_ncfhw_to_nhwc_f16, ap_nhwc_to_ncfhw_f16; csrc/ap_clip.cu:
ap_patchify_nchw_f16). Imported by the CPU checker tests and the GPU contract tests; not a conftest. The checks (`check`,
`check_exact`, `headroom`) and `Ref` are those of gemm_reference.py. Below, u = 2**-24 (one fp32 rounding).

Layouts: latents fp16 [L, HW, 4]; acc fp32 [B, L, HW, 4] (B = 2 under CFG: plane 0 unconditional, plane 1 conditional);
a UNet input / output row is one (b, f, px) with `ld` channels. Every Ref is 2-D: rows (plane, frame, pixel), 4 columns.

Gather window (exact)
---------------------
out[(d, f), px, 0:4] = lat[idx[f], px] for every dup plane d, lanes 4..Cpad exactly 0. A repeated frame is copied twice.

Scatter-accumulate (exact)
--------------------------
Each (b, frame, px) of one call receives at most one fp32 add of an fp16 value (a frame repeated in a window contributes
its LAST occurrence once: sharding.accumulate, the reference's index assignment at pipeline_pose2vid_long.py:546-547),
and calls are ordered by the stream. So the only correct result is the fp32 replay in window order (`scatter_replay`),
bit for bit. Against the fp64 sum of the same terms a chain of n fp32 adds is within n u sum|terms| (`scatter_ref`).

CFG + DDIM step (bounded)
-------------------------
Given the fp32 acc, the fp32 per-frame weight w (inv_count) and the fp16 latents x, with alpha = alpha_t, alpha_prev the
scheduler's fp32 values widened to double, sa = sqrt(alpha), sb = sqrt(1 - alpha), sp = sqrt(alpha_prev),
sq = sqrt(1 - alpha_prev):
  u* = acc_u w, c* = acc_c w, v* = u* + g (c* - u*)  (CFG)       v* = acc w  (no CFG)
  x0* = c_xx x + c_xv v*, eps* = c_ex x + c_ev v*   with (DDIMScheduler.step, scheduler.py:92-115)
      v_prediction  x0 = sa x - sb v,   eps = sb x + sa v
      epsilon       x0 = (x - sb v) / sa,   eps = v
      sample        x0 = v,   eps = (x - sa v) / sb
  x0* clamped to [-clip, clip] when clip > 0 (eps is NOT recomputed: use_clipped_model_output = False)
  o* = sp x0* + sq eps*.
The host computes the coefficients in fp32: sqrtf(alpha) is correctly rounded (u), 1 - alpha adds u, so sqrtf(1 - alpha)
is within 1.5 u, and 1 / sa, -sb / sa, -sa / sb, 1 / sb are within 3.5 u. Every coefficient gets e_c = 4 u relative,
sp and sq get e_p = 2 u. The kernel's fp32 operations, each allowed one rounding whether or not nvcc contracts a
multiply-add into an FMA (an FMA drops one rounding, never adds one):
  e_u = |w| d_acc + (e_w + u) |u*|                        acc w: d_acc the error of acc itself (0 for a given acc),
                                                          e_w the relative error of w (0 for a given fp32 weight)
  e_v = e_u + |g| (e_u + e_c') + 2 u |g (c* - u*)| + u |v*|     c - u, g (c - u), u + g (c - u)  (CFG)
  e_v = e_u                                                     (no CFG)
  e_x0 = e_c (|c_xx x| + |c_xv v*|) + |c_xv| e_v + u (|c_xx x| + |c_xv v*| + |x0*|)        likewise e_eps
  the clamp is 1-Lipschitz: e_x0 passes through it unchanged
  pre  = e_p (|sp x0*| + |sq eps*|) + sp e_x0 + sq e_eps + u (|sp x0*| + |sq eps*| + |o*|)
then times SECOND_ORDER and the fp16 output rounding, OUT_REL |o*| + OUT_FLOOR (half an ulp). The guidance term
|g| (e_u + e_c) ~ |g| u (|u*| + |c*|) is the amplification of the branch errors by g. The step in fp16 arithmetic (the
reference's own dtype) misses this bound at most elements: its roundings are 2**13 times larger than u.
At the first step of a zero-terminal-SNR schedule alpha_t = 0 exactly (sa = 0, sb = 1); at the last step alpha_prev =
final_alpha_cumprod = 1 (sp = 1, sq = 0): both are exact in fp32 and need no special term.

Layout kernels (exact)
----------------------
ncfhw_to_nhwc: out[(b f), px, c] = x[b, c, f, px] for c < C, 0 for C <= c < Cpad. nhwc_to_ncfhw: out[b, c, f, px] =
x[(b f), px, c], reading only the first C of ld channels.

Patchify (exact)
----------------
Per image a CLS row (a single 1.0 at column 3 P**2) then the patches in flatten(2) order, columns (c, ky, kx), each the
pixel rounded once to fp16 (fp16 input: unchanged), columns 3 P**2 + 1 .. kpad of a patch row and all other CLS columns 0.

Emulations
----------
`emulate_step` reproduces the kernel's arithmetic in fp32 (numpy float32, with or without FMA contraction) and returns
the unrounded fp32 value and its fp16 rounding; `bug=` turns it (and `emulate_gather` / `emulate_scatter`) into models
of plausible kernel mistakes, which the checks must reject.
"""
from __future__ import annotations

import numpy as np
import torch

from gemm_reference import E24, OUT_FLOOR, OUT_REL, SECOND_ORDER, Ref

PRED = {"v_prediction": 0, "epsilon": 1, "sample": 2}      # AP_PRED_* in include/aniportrait_b200.h
E_COEF = 4 * E24
E_PREV = 2 * E24

# The reference configs' schedulers (configs/inference/inference_v2.yaml, inference_v1.yaml) and the `sample` type
SCHEDULES = {
    "v2_vpred_zero_snr": dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False,
                              steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                              timestep_spacing="trailing"),
    "v1_epsilon_clip": dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=True,
                            steps_offset=1, prediction_type="epsilon", timestep_spacing="leading"),
    "sample_clip": dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=True,
                        clip_sample_range=1.5, steps_offset=1, prediction_type="sample", timestep_spacing="leading"),
}


def scheduler(name, steps=25):
    from aniportrait_b200.pipelines.scheduler import DDIMScheduler
    s = DDIMScheduler(**SCHEDULES[name])
    s.set_timesteps(steps)
    return s


def clip_of(sch) -> float:
    return float(sch.config.clip_sample_range) if sch.config.clip_sample else 0.0


def locate_rows(L, HW, B=1):
    def locate(r, c):
        b, rem = divmod(r, L * HW)
        f, px = divmod(rem, HW)
        return f"plane {b}, frame {f}, pixel {px}, channel {c}" if B > 1 else f"frame {f}, pixel {px}, channel {c}"
    return locate


# ---------------------------------------------------------------------------------------------------- DDIM step
def coefficients(pred: str, alpha_t: float, dtype=np.float64):
    """(c_xx, c_xv, c_ex, c_ev) of DDIMScheduler.step. float64: exact from the fp32 alpha; float32: the host's fp32."""
    a = dtype(alpha_t)
    one = dtype(1.0)
    sa, sb = np.sqrt(a), np.sqrt(one - a)
    if pred == "v_prediction":
        return sa, -sb, sb, sa
    if pred == "epsilon":
        return one / sa, -sb / sa, dtype(0.0), one
    if pred == "sample":
        return dtype(0.0), one, one / sb, -sa / sb
    raise ValueError(pred)


def _exact_v(acc, w, g, cfg):
    """acc [B, L, HW, 4] float64, w [L] float64 -> (v*, |u*|, |c*|, |c* - u*|) as [L * HW, 4]."""
    ww = w.view(1, -1, 1, 1)
    a = acc * ww
    if cfg:
        u, c = a[0], a[1]
        v = u + g * (c - u)
        return v.reshape(-1, 4), u.abs().reshape(-1, 4), c.abs().reshape(-1, 4), (c - u).abs().reshape(-1, 4)
    v = a[0]
    z = torch.zeros_like(v).reshape(-1, 4)
    return v.reshape(-1, 4), v.abs().reshape(-1, 4), z, z


def step_ref(acc, w, lat, guidance, alpha_t, alpha_prev, pred, clip, cfg=None, acc_err=None, w_rel=0.0) -> Ref:
    """fp64 reference of ap_cfg_ddim_step_f16. acc [B, L, HW, 4] (fp32 given, or the exact fp64 window sums with their
    absolute error bound acc_err), w [L] (fp32 inv_count, or the exact weights with relative error w_rel), lat [L, HW, 4]
    fp16. Output rows (frame, pixel), 4 columns."""
    acc = acc.double().cpu()
    B, L, HW, _ = acc.shape
    cfg = (B == 2) if cfg is None else cfg
    w = w.double().cpu().reshape(-1)
    x = lat.double().cpu().reshape(-1, 4)
    g = float(guidance)
    cxx, cxv, cex, cev = (float(c) for c in coefficients(pred, float(np.float32(alpha_t))))
    a_p = float(np.float32(alpha_prev))
    sp, sq = np.sqrt(a_p), np.sqrt(1.0 - a_p)
    v, au, ac, acu = _exact_v(acc, w, g, cfg)
    x0 = cxx * x + cxv * v
    eps = cex * x + cev * v
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    o = sp * x0 + sq * eps
    # error of the weighted branches u = acc w, c
    wr = w.view(1, -1, 1, 1).abs().expand(B, L, HW, 1)
    da = torch.zeros_like(acc) if acc_err is None else acc_err.double().cpu()
    e_br = (wr * da).reshape(B, -1, 4) + (w_rel + E24) * (acc * w.view(1, -1, 1, 1)).abs().reshape(B, -1, 4)
    if cfg:
        e_v = e_br[0] + abs(g) * (e_br[0] + e_br[1]) + 2 * E24 * abs(g) * acu + E24 * v.abs()
    else:
        e_v = e_br[0]
    tx0 = abs(cxx) * x.abs() + abs(cxv) * v.abs()
    te = abs(cex) * x.abs() + abs(cev) * v.abs()
    x0u = cxx * x + cxv * v
    e_x0 = E_COEF * tx0 + abs(cxv) * e_v + E24 * (tx0 + x0u.abs())
    e_eps = E_COEF * te + abs(cev) * e_v + E24 * (te + eps.abs())
    to = sp * x0.abs() + sq * eps.abs()
    pre = (E_PREV * to + sp * e_x0 + sq * e_eps + E24 * (to + o.abs())) * SECOND_ORDER
    bound = pre + OUT_REL * o.abs() + OUT_FLOOR
    return Ref(o, bound, locate_rows(L, HW), pre=pre)


def _f32(a):
    return np.asarray(a, dtype=np.float32)


def _fma32(a, b, c):
    """fl32(a b + c): the fp32 product is exact in float64; the double sum then rounds once more only far below u."""
    return (_f32(a).astype(np.float64) * _f32(b).astype(np.float64) + _f32(c).astype(np.float64)).astype(np.float32)


def emulate_step(acc, w, lat, guidance, alpha_t, alpha_prev, pred, clip, fma=False, bug=None):
    """ap_cfg_ddim_step_f16 in fp32 numpy in the kernel's order. Returns (unrounded fp32 [L*HW, 4], fp16 result).
    bug: 'inv_count_prev' / 'inv_count_next' (the weight of frame f -+ 1), 'eps_from_clipped_x0', 'clamp_output',
    'flip_c_xv', 'fp16' (every operation and coefficient in fp16)."""
    acc = acc.float().cpu().numpy()
    B, L, HW, _ = acc.shape
    cfg = B == 2
    wv = w.float().cpu().numpy().astype(np.float32).reshape(-1)
    if bug == "inv_count_prev":
        wv = np.roll(wv, 1)
    elif bug == "inv_count_next":
        wv = np.roll(wv, -1)
    x = lat.half().float().cpu().numpy().reshape(-1, 4)
    T = np.float16 if bug == "fp16" else np.float32
    cxx, cxv, cex, cev = (T(c) for c in coefficients(pred, float(np.float32(alpha_t)), np.float32))
    if bug == "flip_c_xv":
        cxv = -cxv
    sa_t = T(np.sqrt(np.float32(alpha_t)))
    sb_t = T(np.sqrt(np.float32(1.0) - np.float32(alpha_t)))
    sp = T(np.sqrt(np.float32(alpha_prev)))
    sq = T(np.sqrt(np.float32(1.0) - np.float32(alpha_prev)))
    g = T(guidance)
    ww = wv.reshape(1, -1, 1, 1).astype(T)
    a = acc.astype(T)
    x = x.astype(T)
    if cfg:
        u = (a[0] * ww[0]).astype(T)
        c = (a[1] * ww[0]).astype(T)
        d = (c - u).astype(T)
        v = _fma32(g, d, u).astype(T) if fma and T is np.float32 else (u + (g * d).astype(T)).astype(T)
    else:
        v = (a[0] * ww[0]).astype(T)
    v = v.reshape(-1, 4)

    def mad(p, q, r, s):    # p q + r s
        if fma and T is np.float32:
            return _fma32(p, q, _f32(r * s))
        return ((p * q).astype(T) + (r * s).astype(T)).astype(T)
    x0 = mad(cxx, x, cxv, v)
    eps = mad(cex, x, cev, v)
    if clip > 0 and bug != "clamp_output":
        x0 = np.minimum(np.maximum(x0, T(-clip)), T(clip))
        if bug == "eps_from_clipped_x0":      # use_clipped_model_output = True: eps = (x - sa x0) / sb
            eps = ((x - (sa_t * x0).astype(T)).astype(T) / sb_t).astype(T)
    y = mad(sp, x0, sq, eps).astype(np.float32)
    if bug == "clamp_output" and clip > 0:
        y = np.minimum(np.maximum(y, np.float32(-clip)), np.float32(clip))
    y = torch.from_numpy(y.astype(np.float32))
    return y, y.half()


def scheduler_step64(sch, acc, w, lat, guidance, t):
    """The same step through DDIMScheduler.step in float64 (combine by the reference's rule, then step)."""
    acc = acc.double().cpu()
    a = acc * w.double().cpu().view(1, -1, 1, 1)
    v = a[0] + guidance * (a[1] - a[0]) if acc.shape[0] == 2 else a[0]
    return sch.step(v, t, lat.double().cpu()).prev_sample.reshape(-1, 4)


# ---------------------------------------------------------------------------------------------------- gather / scatter
def gather_ref(lat, idx, dup, cpad) -> Ref:
    """Exact UNet input [(dup F) HW, cpad] of one window."""
    lat = lat.cpu()
    L, HW, _ = lat.shape
    F = len(idx)
    o = torch.zeros(dup, F, HW, cpad, dtype=torch.float64)
    o[:, :, :, :4] = lat[list(idx)].double().unsqueeze(0)

    def locate(r, c):
        d, rem = divmod(r, F * HW)
        f, px = divmod(rem, HW)
        return f"dup plane {d}, window frame {f} (latent frame {idx[f]}), pixel {px}, lane {c}"
    return Ref(o.reshape(-1, cpad), torch.zeros(dup * F * HW, cpad, dtype=torch.float64), locate, exact=True)


def emulate_gather(lat, idx, dup, cpad, bug=None):
    """bug 'dup_plane': planes d > 0 take the window's frames shifted by one (frame f + 1 of plane 0)."""
    lat = lat.cpu()
    L, HW, _ = lat.shape
    F = len(idx)
    o = torch.zeros(dup, F, HW, cpad, dtype=torch.float16)
    for d in range(dup):
        sel = list(idx) if (d == 0 or bug != "dup_plane") else list(idx[1:]) + list(idx[:1])
        o[d, :, :, :4] = lat[sel]
    return o.reshape(-1, cpad)


def last_occurrence(window):
    """frame -> position of its last occurrence in the window (sharding.accumulate)."""
    return {f: j for j, f in enumerate(window)}


def scatter_replay(acc0, calls, bug=None):
    """fp32 CPU replay of ap_scatter_accumulate_f16 calls in stream order. acc0 fp32 [P, L, HW, 4] (all planes of the
    buffer); calls: list of (pred [B F, HW, >=4] fp16, window, plane0) writing planes plane0 .. plane0 + B - 1.
    bug: 'first_occurrence' (a repeated frame takes its first occurrence) or 'count_twice' (every occurrence added)."""
    acc = acc0.float().cpu().clone()
    for pred, window, p0 in calls:
        F = len(window)
        pr = pred[..., :4].float().cpu()
        B = pr.shape[0] // F
        pr = pr.view(B, F, *pr.shape[1:])
        if bug == "count_twice":
            pairs = list(enumerate(window))
        elif bug == "first_occurrence":
            first = {}
            for j, f in enumerate(window):
                first.setdefault(f, j)
            pairs = [(j, f) for f, j in first.items()]
        else:
            pairs = [(j, f) for f, j in last_occurrence(window).items()]
        for j, f in pairs:
            acc[p0:p0 + B, f] = acc[p0:p0 + B, f] + pr[:, j]
    return acc


def scatter_ref(acc0, calls) -> Ref:
    """fp64 sum of the same terms, bound n u sum|terms| (n adds per element), rows (plane, frame, pixel)."""
    acc = acc0.double().cpu().clone()
    mag = acc.abs()
    n = torch.zeros_like(acc)
    for pred, window, p0 in calls:
        F = len(window)
        pr = pred[..., :4].double().cpu()
        B = pr.shape[0] // F
        pr = pr.view(B, F, *pr.shape[1:])
        for f, j in last_occurrence(window).items():
            acc[p0:p0 + B, f] += pr[:, j]
            mag[p0:p0 + B, f] += pr[:, j].abs()
            n[p0:p0 + B, f] += 1
    P, L, HW, _ = acc.shape
    bound = n * E24 * mag + 1e-300
    return Ref(acc.reshape(-1, 4), bound.reshape(-1, 4), locate_rows(L, HW, P), out_f32=True)


def exact_f32(want: torch.Tensor, locate) -> Ref:
    """An exact Ref of an fp32 result (check_exact compares bit for bit)."""
    w = want.double().reshape(-1, want.shape[-1])
    return Ref(w, torch.zeros_like(w), locate, exact=True, out_f32=True)


# ---------------------------------------------------------------------------------------------------- layouts
def ncfhw_to_nhwc_ref(x, cpad) -> Ref:
    B, C, F, H, W = x.shape
    o = torch.zeros(B, F, H * W, cpad, dtype=torch.float64)
    o[..., :C] = x.double().cpu().permute(0, 2, 3, 4, 1).reshape(B, F, H * W, C)

    def locate(r, c):
        bf, px = divmod(r, H * W)
        return f"batch {bf // F}, frame {bf % F}, pixel {px}, channel {c}"
    return Ref(o.reshape(-1, cpad), torch.zeros(B * F * H * W, cpad, dtype=torch.float64), locate, exact=True)


def nhwc_to_ncfhw_ref(x, B, C, F) -> Ref:
    """x [(B F), H, W, ld] -> rows (b, c, f, h), columns w."""
    _, H, W, _ = x.shape
    o = x[..., :C].double().cpu().reshape(B, F, H, W, C).permute(0, 4, 1, 2, 3).reshape(B * C * F * H, W)

    def locate(r, c):
        bcf, h = divmod(r, H)
        bc, f = divmod(bcf, F)
        return f"batch {bc // C}, channel {bc % C}, frame {f}, row {h}, column {c}"
    return Ref(o, torch.zeros_like(o), locate, exact=True)


def patchify_ref(px, P, kpad) -> Ref:
    """px [B, 3, H, W] fp16 / fp32 -> [B (1 + Gh Gw), kpad]: each element fp16_rn of its pixel (an exact double here,
    check_exact rounds it once)."""
    B, _, H, W = px.shape
    gh, gw = H // P, W // P
    pt = px.double().cpu().reshape(B, 3, gh, P, gw, P).permute(0, 2, 4, 1, 3, 5).reshape(B, gh * gw, 3 * P * P)
    o = torch.zeros(B, 1 + gh * gw, kpad, dtype=torch.float64)
    o[:, 0, 3 * P * P] = 1.0
    o[:, 1:, :3 * P * P] = pt
    tokens = 1 + gh * gw

    def locate(r, c):
        b, t = divmod(r, tokens)
        return f"image {b}, " + ("CLS row" if t == 0 else f"patch {t - 1} (row {(t - 1) // gw}, col {(t - 1) % gw})") + \
            f", column {c}"
    return Ref(o.reshape(-1, kpad), torch.zeros(B * tokens, kpad, dtype=torch.float64), locate, exact=True)


# ---------------------------------------------------------------------------------------------------- reference loop
def reference_window_sums(preds, windows, L, HW, dup):
    """Reference :519-548 in float64: noise_pred[:, :, c] += pred and counter[c] += 1 per window; a frame repeated in a
    window takes its last occurrence once (index assignment). preds[k]: [dup F, HW, >=4]. Returns (sums [dup, L, HW, 4],
    counter [L], magnitude sum|terms| and number of adds per element, for the fp32 accumulation bound)."""
    s = torch.zeros(dup, L, HW, 4, dtype=torch.float64)
    mag = torch.zeros_like(s)
    n = torch.zeros_like(s)
    counter = torch.zeros(L, dtype=torch.float64)
    for pred, window in zip(preds, windows):
        F = len(window)
        pr = pred[..., :4].double().cpu().view(dup, F, HW, 4)
        for f, j in last_occurrence(window).items():
            s[:, f] += pr[:, j]
            mag[:, f] += pr[:, j].abs()
            n[:, f] += 1
            counter[f] += 1
    return s, counter, mag, n


def reference_loop_step(preds, windows, lat, guidance, alpha_t, alpha_prev, pred_type, clip) -> Ref:
    """One step of the reference loop (pipeline_pose2vid_long.py:459-559) in float64 on the kernel's latents: the window
    sums are divided by the counter ONLY under CFG (:551-555); without CFG the scheduler steps on the sum."""
    L, HW, _ = lat.shape
    cfg = guidance > 1.0
    dup = 2 if cfg else 1
    s, counter, mag, n = reference_window_sums(preds, windows, L, HW, dup)
    w = 1.0 / counter if cfg else torch.ones_like(counter)
    w_rel = E24 if cfg else 0.0            # fp32(1 / count) differs from 1 / count by at most one rounding
    return step_ref(s, w, lat, guidance, alpha_t, alpha_prev, pred_type, clip, cfg=cfg, acc_err=n * E24 * mag,
                    w_rel=w_rel)
