"""DPMSolverMultistepScheduler / EulerDiscreteScheduler on the CPU (-m "not gpu"):
  tables      pipelines/scheduler.py::multistep_coefficients reproduces the scheduler object's own scale_model_input and
              step() sequence in float64, every step of 10-, 15- and 25-step schedules, every supported configuration
  refusals    what the fused multistep update cannot reproduce raises NotImplementedError
  goldens     the oracle's denoising loop with the restated schedulers (diffusers_samplers.py) reproduces
              pipeline_small_dpm / pipeline_small_euler,
              the outputs of the unmodified reference pipeline
  checker     sampler_reference.py accepts an fp32 emulation of the kernels and rejects planted kernel and table bugs
"""
import itertools
import os
import sys

import pytest
import torch

import gemm_reference as GR
import sampler_reference as SR
from helpers import build_unet2d, build_unet3d, rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
STEPS = (10, 15, 25)
SPACINGS = ("linspace", "leading", "trailing")
PREDS = ("epsilon", "v_prediction", "sample")


def _table_vs_step(make, steps, guidance, seed):
    """Runs the scheduler's own step() (float64 operands and sigmas) and the coefficient table side by side from the same
    latents; returns the worst relative difference over the steps (latents and input scale)."""
    from aniportrait_b200.pipelines.scheduler import multistep_coefficients
    sch = make(steps)
    try:
        table = multistep_coefficients(sch)
    except NotImplementedError:
        # only where the library's own step is not finite either (Karras sigmas repeat the last one: h = 0 at a
        # second-order last step, and heun's (e^-h - 1) / h is 0 / 0)
        sch.sigmas = sch.sigmas.double()
        x = torch.ones(2, 3, dtype=torch.float64)
        for t in sch.timesteps:
            x = sch.step(torch.sin(x), t, x).prev_sample
        assert not torch.isfinite(x).all()
        return 0.0
    sch.sigmas = sch.sigmas.double()
    assert len(table) == len(sch.timesteps)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 3, 5, generator=g, dtype=torch.float64) * 3
    m_prev = None
    worst = 0.0
    for co, t in zip(table, sch.timesteps):
        assert co.timestep == float(t)
        xin = sch.scale_model_input(x, t)
        worst = max(worst, ((xin - co.scale * x).abs().max() / xin.abs().max()).item())
        u = torch.sin(xin) + 0.1 * torch.randn(x.shape, generator=g, dtype=torch.float64)
        c = torch.cos(xin) - 0.2 * xin
        v = u + guidance * (c - u) if guidance > 1 else c
        want = sch.step(v, t, x).prev_sample
        m = co.c_xx * x + co.c_xv * v
        got = co.k_x * x + co.k_0 * m + (co.k_1 * m_prev if co.k_1 != 0 else 0.0)
        worst = max(worst, ((got - want).abs().max() / want.abs().max()).item())
        m_prev = m if co.store else None
        x = want
    return worst


DPM_CASES = list(itertools.product(("dpmsolver++", "dpmsolver"), (1, 2), ("midpoint", "heun"), (False, True)))


@pytest.mark.parametrize("algo,order,solver,karras", DPM_CASES,
                         ids=[f"{a}-o{o}-{s}-{'karras' if k else 'plain'}" for a, o, s, k in DPM_CASES])
def test_dpm_table_reproduces_scheduler_step(algo, order, solver, karras):
    worst = 0.0
    for sp, pt, steps, guidance in itertools.product(SPACINGS, PREDS, STEPS, (1.0, 3.5)):
        def make(n):
            return SR.make_scheduler("DPMSolverMultistepScheduler", n, algorithm_type=algo, solver_order=order,
                                     solver_type=solver, use_karras_sigmas=karras, timestep_spacing=sp,
                                     prediction_type=pt)
        worst = max(worst, _table_vs_step(make, steps, guidance, seed=steps))
    assert worst <= 1e-12, worst


@pytest.mark.parametrize("variant", ["no_lower_order_final", "euler_at_final", "lambda_min_clipped",
                                     "final_sigmas_zero", "scaled_linear"])
def test_dpm_table_reproduces_scheduler_step_variants(variant):
    kw = dict(no_lower_order_final=dict(lower_order_final=False), euler_at_final=dict(euler_at_final=True),
              lambda_min_clipped=dict(lambda_min_clipped=-3.0), scaled_linear=dict(beta_schedule="scaled_linear"),
              final_sigmas_zero={})[variant]
    worst = 0.0
    for steps, sp in itertools.product(STEPS, SPACINGS):
        def make(n):
            s = SR.make_scheduler("DPMSolverMultistepScheduler", n, timestep_spacing=sp, **kw)
            if variant == "final_sigmas_zero":       # a later diffusers option: last sigma 0, order 1 at the last step
                s.config["final_sigmas_type"] = "zero"
                s.sigmas[-1] = 0.0
                s.step_orig = s.step
            return s
        if variant == "final_sigmas_zero":
            from aniportrait_b200.pipelines.scheduler import multistep_coefficients
            s = make(steps)
            table = multistep_coefficients(s)
            assert table[-1].k_1 == 0.0 and table[-1].k_x == 0.0 and table[-1].k_0 == pytest.approx(1.0)
            continue
        worst = max(worst, _table_vs_step(make, steps, 3.5, seed=steps))
    assert worst <= 1e-12, worst


EULER_CASES = list(itertools.product(SPACINGS, PREDS, (False, True)))


@pytest.mark.parametrize("sp,pt,karras", EULER_CASES,
                         ids=[f"{s}-{p}-{'karras' if k else 'plain'}" for s, p, k in EULER_CASES])
def test_euler_table_reproduces_scheduler_step(sp, pt, karras):
    worst = 0.0
    for steps, guidance in itertools.product(STEPS, (1.0, 3.5)):
        def make(n):
            return SR.make_scheduler("EulerDiscreteScheduler", n, timestep_spacing=sp, prediction_type=pt,
                                     use_karras_sigmas=karras)
        worst = max(worst, _table_vs_step(make, steps, guidance, seed=steps))
    assert worst <= 1e-12, worst


def test_orders_follow_the_class():
    """2M at 6 steps (the pipeline_small_dpm golden): order 1 first, order 2, order 1 at the end (lower_order_final, fewer
    than 15 steps); at 15 steps the last step stays second order. Euler never reads the history."""
    from aniportrait_b200.pipelines.scheduler import multistep_coefficients
    t6 = multistep_coefficients(SR.make_scheduler("DPMSolverMultistepScheduler", 6, timestep_spacing="trailing",
                                                  prediction_type="v_prediction"))
    assert [c.k_1 != 0 for c in t6] == [False, True, True, True, True, False]
    assert [c.store for c in t6] == [True, True, True, True, False, False]
    t15 = multistep_coefficients(SR.make_scheduler("DPMSolverMultistepScheduler", 15))
    assert t15[-1].k_1 != 0 and t15[0].k_1 == 0
    te = multistep_coefficients(SR.make_scheduler("EulerDiscreteScheduler", 5))
    assert all(c.k_1 == 0 and not c.store for c in te)
    assert [c.timestep for c in te] == [999.0, 749.25, 499.5, 249.75, 0.0]


def _zero_snr_betas():
    from aniportrait_b200.pipelines.scheduler import rescale_zero_terminal_snr
    return rescale_zero_terminal_snr(torch.linspace(0.00085, 0.012, 1000)).tolist()


def test_unsupported_schedulers_raise():
    from aniportrait_b200.pipelines import scheduler as S

    def named(name):
        return type(name, (), dict(config=dict(prediction_type="epsilon"), alphas_cumprod=torch.ones(10)))()
    for name in ("EulerAncestralDiscreteScheduler", "LMSDiscreteScheduler", "PNDMScheduler"):
        with pytest.raises(NotImplementedError, match=name):
            S.update_family(named(name))

    def table(cls, **kw):
        return S.multistep_coefficients(SR.make_scheduler(cls, 10, **kw))
    with pytest.raises(NotImplementedError, match="SDE"):
        table("DPMSolverMultistepScheduler", algorithm_type="sde-dpmsolver++")
    with pytest.raises(NotImplementedError, match="order 3"):
        table("DPMSolverMultistepScheduler", solver_order=3)
    with pytest.raises(NotImplementedError, match="thresholding"):
        table("DPMSolverMultistepScheduler", thresholding=True)
    with pytest.raises(NotImplementedError, match="s_churn"):
        S.multistep_coefficients(SR.make_scheduler("EulerDiscreteScheduler", 10), s_churn=0.5)
    # zero terminal SNR: sigma = inf at t = 999 (the 0.24 classes have no rescale_betas_zero_snr; a beta table can)
    for cls in ("DPMSolverMultistepScheduler", "EulerDiscreteScheduler"):
        with pytest.raises(NotImplementedError, match="non-finite sigma"):
            table(cls, trained_betas=_zero_snr_betas(), timestep_spacing="trailing")
        with pytest.raises(TypeError):
            getattr(S, cls)(rescale_betas_zero_snr=True)
    # DDIM and DDIM-style schedulers keep the DDIM path
    assert S.update_family(S.DDIMScheduler()) == "ddim"


def test_from_config_takes_a_ddim_config():
    """The INTEGRATION.md recipe: DPMSolverMultistepScheduler.from_config(pipe.scheduler.config) drops the DDIM-only keys
    (clip_sample, set_alpha_to_one, rescale_betas_zero_snr) like diffusers' ConfigMixin."""
    from aniportrait_b200.pipelines import scheduler as S
    ddim = S.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1,
                           prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    d = S.DPMSolverMultistepScheduler.from_config(ddim.config)
    assert d.config.prediction_type == "v_prediction" and d.config.timestep_spacing == "trailing"
    assert d.config.beta_start == 0.00085 and "rescale_betas_zero_snr" not in d.config and "clip_sample" not in d.config
    e = S.EulerDiscreteScheduler.from_config(ddim.config, prediction_type="epsilon")
    assert e.config.prediction_type == "epsilon" and e.config.steps_offset == 1
    assert S.update_family(d) == "dpm" and S.update_family(e) == "euler"


def test_oracle_restatements_match_the_product_copies():
    """The oracle's restated classes (diffusers_samplers.py, what the goldens were generated with) and the product's
    copies step identically."""
    from diffusers_samplers import DPMSolverMultistepScheduler as SD, EulerDiscreteScheduler as SE
    from aniportrait_b200.pipelines import scheduler as S
    g = torch.Generator().manual_seed(3)
    for a, b, kw in ((SD, S.DPMSolverMultistepScheduler, dict(prediction_type="v_prediction", timestep_spacing="trailing")),
                     (SD, S.DPMSolverMultistepScheduler, dict(solver_type="heun", use_karras_sigmas=True)),
                     (SE, S.EulerDiscreteScheduler, dict(timestep_spacing="leading"))):
        sa, sb = a(**dict(SR.BASE, **kw)), b(**dict(SR.BASE, **kw))
        assert float(sa.init_noise_sigma) == float(sb.init_noise_sigma)
        sa.set_timesteps(12)
        sb.set_timesteps(12)
        assert torch.equal(sa.timesteps, sb.timesteps) and torch.equal(sa.sigmas, sb.sigmas)
        assert float(sa.init_noise_sigma) == float(sb.init_noise_sigma)
        xa = xb = torch.randn(1, 4, 2, 3, 3, generator=g)
        for t in sa.timesteps:
            v = torch.sin(sa.scale_model_input(xa, t))
            assert torch.equal(sb.scale_model_input(xb, t), sa.scale_model_input(xa, t))
            xa = sa.step(v, t, xa).prev_sample
            xb = sb.step(v, t, xb).prev_sample
            assert torch.equal(xa, xb)


# ---------------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("case", ["pipeline_small_dpm", "pipeline_small_euler"])
def test_oracle_loop_reproduces_the_reference_golden(case):
    """The oracle's denoising loop with the restated scheduler the golden was made with, against the unmodified reference
    pipeline's output: scale_model_input, init_noise_sigma, the call order and the history are wired as there."""
    from oracle import ref_import
    from oracle import functional as OF
    ref_import.activate_shim()
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import make_golden as MG
    import make_golden_samplers as MGS
    from diffusers import AutoencoderKL
    from diffusers.image_processor import VaeImageProcessor
    from transformers import CLIPImageProcessor
    gold = torch.load(os.path.join(GOLDEN, case + ".pt"))
    P = gold["params"]
    seeds = P["seeds"]
    from aniportrait_b200.models.pose_guider import PoseGuider
    from aniportrait_b200.synthetic import randomize_state_dict
    _, sd3 = build_unet3d(P["chans"], seeds["unet3d"])
    _, sd2 = build_unet2d(P["chans"], seeds["unet2d"])
    sdp = randomize_state_dict(PoseGuider(noise_latent_channels=P["chans"][0], use_ca=True).state_dict(),
                               seed=seeds["pose"])
    vae = AutoencoderKL(block_out_channels=P["vae_chans"])
    sdv = randomize_state_dict(vae.state_dict(), seed=seeds["vae"])
    vae.load_state_dict(sdv)
    clip = MG.small_clip_encoder(seeds["clip"])
    size, L = P["size"], P["L"]
    ref_image, poses, _ = MG.pipeline_inputs(size, L, seeds["inputs"])
    sched, kw = MGS.sampler(gold["scheduler"]["cls"], **gold["scheduler"]["kwargs"])
    assert kw == gold["scheduler"]["kwargs"]
    with torch.no_grad():
        clip_px = CLIPImageProcessor().preprocess(ref_image.resize((224, 224)), return_tensors="pt").pixel_values
        clip_embed = clip(clip_px).image_embeds
        ref_t = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True).preprocess(ref_image, height=size, width=size)
        ref_lat = vae.encode(ref_t).latent_dist.mean * 0.18215
        cond = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True, do_normalize=True)
        pose_cond = torch.cat([cond.preprocess(p, height=size, width=size) for p in poses], 0)
        pose_cond = pose_cond.permute(1, 0, 2, 3).unsqueeze(0)
        lat0 = torch.randn((1, 4, L, size // 8, size // 8), generator=torch.manual_seed(seeds["latents"]))
        trace = SR.oracle_denoise_loop(sd3, sd2, sdp, lat0, ref_lat, clip_embed, pose_cond, P["steps"], sched,
                                       P["guidance"], c=dict(OF.SD15, block_out_channels=tuple(P["chans"])))
        frames = [0, 7, L - 1]
        video = (OF.vae_decode(sdv, trace[-1][0, :, frames].permute(1, 0, 2, 3) / 0.18215) / 2 + 0.5).clamp(0, 1)
    assert len(trace) == P["steps"]
    e_first, e_final = rel_l2(trace[0], gold["first_step_latents"]), rel_l2(trace[-1], gold["final_latents"])
    print(f"{case}: oracle loop vs reference golden: first step {e_first:.2e}, final {e_final:.2e}")
    assert e_first < 1e-4 and e_final < 1e-4
    assert rel_l2(video.permute(1, 0, 2, 3).unsqueeze(0), gold["video_frames"].float()) < 2e-3   # fp16 in the fixture


# ---------------------------------------------------------------------------------------------------- checker
def _golden_tables():
    from aniportrait_b200.pipelines.scheduler import multistep_coefficients
    dpm = lambda: SR.make_scheduler("DPMSolverMultistepScheduler", 6, timestep_spacing="trailing",   # noqa: E731
                                    prediction_type="v_prediction")
    eul = lambda: SR.make_scheduler("EulerDiscreteScheduler", 5)                                     # noqa: E731
    return dict(dpm=(dpm, multistep_coefficients(dpm())), euler=(eul, multistep_coefficients(eul())))


@pytest.mark.parametrize("fma", [False, True])
@pytest.mark.parametrize("guidance", [1.0, 3.5])
@pytest.mark.parametrize("family", ["dpm", "euler"])
def test_checker_accepts_the_fp32_emulation(family, guidance, fma):
    make, table = _golden_tables()[family]
    L, HW = 3, 16
    g = torch.Generator().manual_seed(5)
    hist = torch.full((L, HW, 4), float("nan"))
    lat = (torch.randn(L, HW, 4, generator=g) * 2).half()
    worst = 0.0
    for i, co in enumerate(table):
        acc = torch.randn(2 if guidance > 1 else 1, L, HW, 4, generator=g) * 2
        w = torch.tensor([1.0, 0.5, 1 / 3], dtype=torch.float32)
        ref, mref = SR.step_ref(acc, w, lat, hist, guidance, co)
        y16, y32, h_out = SR.emulate_step(acc, w, lat, hist, guidance, co, fma=fma)
        worst = max(worst, GR.check(y16.double(), ref, f"step {i}"))
        assert GR.headroom(y32, ref) <= 1.0
        if co.store:
            GR.check(h_out.double(), mref, f"step {i}: history")
        else:
            assert torch.equal(h_out.view(L, HW, 4).isnan(), hist.isnan())
        lat, hist = y16.view(L, HW, 4), h_out.view(L, HW, 4)
    assert 0.0 < worst <= 1.0
    assert SR.loop_check(make, guidance, table) <= 1.0


@pytest.mark.parametrize("bug", ["hist_not_updated", "order2_first_step", "r0_inverted", "scale_missing",
                                 "hist_read_at_k1_zero"])
def test_checker_rejects_planted_bugs(bug):
    tables = _golden_tables()
    family = "euler" if bug == "scale_missing" else "dpm"
    make, table = tables[family]
    if bug in ("order2_first_step", "r0_inverted"):
        table, kernel_bug = SR.planted_table(table, bug), None
    else:
        kernel_bug = bug
    with pytest.raises(AssertionError):
        SR.loop_check(make, 3.5, table, bug=kernel_bug)
