"""TEST INFRASTRUCTURE — generates tests/golden/pipeline_small_dpm.pt and pipeline_small_euler.pt by running the
UNMODIFIED reference Pose2VideoPipeline (an AniPortrait checkout's src/, imported through oracle/diffusers_shim) on CPU
in fp32 with the seeded synthetic weights and inputs of oracle/make_golden.py's `pipeline_small`, and the scheduler
objects of diffusers_samplers.py (the reference's `scheduler` argument is duck-typed: it calls set_timesteps,
init_noise_sigma, scale_model_input and step).

    ANIPORTRAIT_REFERENCE=<checkout> python tests/make_golden_samplers.py [case ...]

The schedulers are built from make_golden.SCHED_KWARGS without the keys the 0.24 classes do not take (clip_sample,
rescale_betas_zero_snr), which is what diffusers' `from_config(ddim.config)` yields, then the case's overrides.
"""
from __future__ import annotations

import inspect
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_golden as MG  # noqa: E402
import diffusers_samplers  # noqa: E402

CASES = {
    # DPM-Solver++(2M), v-prediction, trailing spacing, 6 steps: an order-1 first step, order-2 steps and the order-1
    # final step (lower_order_final, fewer than 15 steps)
    "pipeline_small_dpm": (dict(steps=6), "DPMSolverMultistepScheduler", dict(solver_order=2)),
    # Euler, epsilon, linspace spacing, 5 steps: fractional timesteps (999 / 4 apart) reach the UNet's time embedding,
    # the initial noise is scaled by init_noise_sigma and every UNet input by scale_model_input
    "pipeline_small_euler": (dict(steps=5), "EulerDiscreteScheduler",
                             dict(prediction_type="epsilon", timestep_spacing="linspace")),
}


def sampler(cls_name, **overrides):
    """(scheduler, the keyword arguments it was built with): SCHED_KWARGS restricted to what the class takes, then
    `overrides`."""
    cls = getattr(diffusers_samplers, cls_name)
    names = set(inspect.signature(cls.__init__).parameters)
    kw = {k: v for k, v in MG.SCHED_KWARGS.items() if k in names}
    kw.update(overrides)
    return cls(**kw), kw


def case(name):
    """make_golden.case_pipeline with the case's scheduler: CLIP -> ReferenceNet -> windowed CFG loop with in-loop
    PoseGuider and the scheduler's scale_model_input / step -> frame-wise VAE decode; L = 20 (two overlapping windows)."""
    MG.ref_import.activate()
    from diffusers import AutoencoderKL
    from src.pipelines.pipeline_pose2vid_long import Pose2VideoPipeline
    over, cls_name, sched_over = CASES[name]
    P = dict(MG.PIPE_SMALL, **over)
    t0 = time.time()
    sd = P["seeds"]
    unet3d = MG.ref_import.build_unet3d(P["chans"]); MG._load(unet3d, sd["unet3d"])      # noqa: E702
    unet2d = MG.ref_import.build_unet2d(P["chans"]); MG._load(unet2d, sd["unet2d"])      # noqa: E702
    pose = MG.ref_import.build_pose_guider(P["chans"][0]); MG._load(pose, sd["pose"])   # noqa: E702
    vae = AutoencoderKL(block_out_channels=P["vae_chans"]); MG._load(vae, sd["vae"])     # noqa: E702
    clip = MG.small_clip_encoder(sd["clip"])
    sched, kw = sampler(cls_name, **sched_over)
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=unet2d, denoising_unet=unet3d,
                              pose_guider=pose, scheduler=sched)
    ref_image, poses, ref_pose = MG.pipeline_inputs(P["size"], P["L"], sd["inputs"])
    lat_trace = []
    out = pipe(ref_image, poses, ref_pose, P["size"], P["size"], P["L"], P["steps"], P["guidance"],
               generator=torch.manual_seed(sd["latents"]), callback=lambda i, t, l: lat_trace.append(l.clone()),
               callback_steps=1)
    videos = out.videos
    torch.save(dict(case=name, params=dict(P), final_latents=lat_trace[-1].float(),
                    first_step_latents=lat_trace[0].float(), video_frames=videos[:, :, [0, 7, P["L"] - 1]].half(),
                    video_mean=float(videos.mean()), torch_version=str(torch.__version__),
                    scheduler=dict(cls=cls_name, kwargs=kw),
                    generator="reference Pose2VideoPipeline via oracle/diffusers_shim + tests/diffusers_samplers.py, "
                              "fp32 CPU"),
               os.path.join(MG.GOLDEN, name + ".pt"))
    print(f"{name}: videos {tuple(videos.shape)} mean={videos.mean():.4f} steps traced={len(lat_trace)} "
          f"in {time.time() - t0:.1f}s")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 8)
    for n in sys.argv[1:] or list(CASES):
        case(n)
