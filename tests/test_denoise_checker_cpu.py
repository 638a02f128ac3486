"""The checker of the denoising-loop contract (denoise_reference.py) on the CPU: an fp32 emulation of ap_cfg_ddim_step_f16,
with and without FMA contraction, passes every bound at reduced size and uses at most half of the pre-rounding bound;
the fp64 references agree with DDIMScheduler.step; each modelled kernel bug is rejected by a message naming the element."""
import numpy as np
import pytest
import torch

import denoise_reference as DR
import gemm_reference as GR

L, HW = 20, 12


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _operands(cfg, seed=0, scale=1.0):
    """acc as the sum of `count` window predictions per frame, the plan_windows weights of L = 20 (counts 1 and 2)
    followed by a 1 / 3 frame, latents with |x0| on both sides of the clip ranges."""
    from aniportrait_b200.pipelines.sharding import plan_windows
    g = _gen(seed)
    _, inv = plan_windows(L, 25)
    inv = inv.clone()
    inv[3] = 1.0 / 3.0
    cnt = (1.0 / inv).round()
    acc = (torch.randn(2 if cfg else 1, L, HW, 4, generator=g) * cnt.view(1, -1, 1, 1)).float()
    lat = (scale * torch.randn(L, HW, 4, generator=g)).half()
    return acc, inv.float(), lat


def _steps(name):
    sch = DR.scheduler(name)
    return sch, [int(t) for t in sch.timesteps]


CASES = [(s, g) for s in DR.SCHEDULES for g in (1.0, 3.5, 7.5)]


@pytest.mark.parametrize("fma", [False, True], ids=["no_fma", "fma"])
@pytest.mark.parametrize("sched,guidance", CASES, ids=[f"{s}-g{g}" for s, g in CASES])
def test_emulation_within_half_the_bound(sched, guidance, fma):
    sch, ts = _steps(sched)
    acc, inv, lat = _operands(guidance > 1.0, seed=len(sched), scale=1.5)
    worst = 0.0
    clipped = unclipped = 0
    for t in ts:
        a_t, a_p = sch.alpha_pair(t)
        ref = DR.step_ref(acc, inv, lat, guidance, a_t, a_p, sch.config.prediction_type, DR.clip_of(sch))
        y32, y16 = DR.emulate_step(acc, inv, lat, guidance, a_t, a_p, sch.config.prediction_type, DR.clip_of(sch),
                                   fma=fma)
        GR.check(y16, ref, f"{sched} t={t}")
        worst = max(worst, GR.headroom(y32, ref))
        if DR.clip_of(sch):
            x0 = DR.step_ref(acc, inv, lat, guidance, a_t, 1.0, sch.config.prediction_type, 0.0).o   # alpha_prev 1: x0
            clipped += int((x0.abs() > DR.clip_of(sch)).sum())
            unclipped += int((x0.abs() < DR.clip_of(sch)).sum())
    print(f"{sched} g={guidance} fma={fma}: headroom {worst:.3f}")
    assert 0.0 < worst <= 0.5
    if DR.clip_of(sch):
        assert clipped and unclipped, "the clip range must be crossed"


def test_schedules_reach_the_edge_steps():
    """The zero-SNR schedule's first step has alpha_t = 0 exactly; every schedule's last step has alpha_prev = 1."""
    sch, ts = _steps("v2_vpred_zero_snr")
    assert sch.alpha_pair(ts[0])[0] == 0.0
    for name in DR.SCHEDULES:
        sch, ts = _steps(name)
        assert sch.alpha_pair(ts[-1])[1] == 1.0


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("pred", list(DR.PRED))
def test_reference_equals_scheduler_step(pred, clip):
    from aniportrait_b200.pipelines.scheduler import DDIMScheduler
    kw = dict(DR.SCHEDULES["v1_epsilon_clip"], prediction_type=pred, clip_sample=clip, clip_sample_range=1.0)
    sch = DDIMScheduler(**kw)
    sch.set_timesteps(25)
    for cfg in (False, True):
        acc, inv, lat = _operands(cfg, seed=3, scale=1.5)
        for t in [int(x) for x in sch.timesteps][::6]:
            a_t, a_p = sch.alpha_pair(t)
            ref = DR.step_ref(acc, inv, lat, 3.5, a_t, a_p, pred, 1.0 if clip else 0.0)
            want = DR.scheduler_step64(sch, acc, inv, lat, 3.5, t)
            assert torch.allclose(ref.o, want, rtol=1e-12, atol=1e-12), (pred, clip, t)


BUGS = ["inv_count_prev", "inv_count_next", "eps_from_clipped_x0", "clamp_output", "flip_c_xv", "fp16"]


@pytest.mark.parametrize("bug", BUGS)
def test_step_bug_is_rejected(bug):
    """Each modelled bug fails the bound somewhere in the 25 steps of its schedule."""
    sched = "v2_vpred_zero_snr" if bug in ("inv_count_prev", "inv_count_next", "flip_c_xv", "fp16") else \
        "v1_epsilon_clip"
    sch, ts = _steps(sched)
    acc, inv, lat = _operands(True, seed=5, scale=1.5)
    for t in ts:
        a_t, a_p = sch.alpha_pair(t)
        ref = DR.step_ref(acc, inv, lat, 3.5, a_t, a_p, sch.config.prediction_type, DR.clip_of(sch))
        _, y16 = DR.emulate_step(acc, inv, lat, 3.5, a_t, a_p, sch.config.prediction_type, DR.clip_of(sch), bug=bug)
        try:
            GR.check(y16, ref, f"{bug} t={t}")
        except AssertionError as e:
            assert "frame" in str(e) and "channel" in str(e)
            print(f"{bug}: rejected: {e}")
            return
    pytest.fail(f"{bug} was not rejected")


def _windows(Lv, stride):
    from aniportrait_b200.pipelines.sharding import plan_windows
    return plan_windows(Lv, 25, "uniform", 16, stride, 4)[0]


def _scatter_calls(windows, dup, hw, seed):
    g = _gen(seed)
    return [(torch.randn(dup * len(w), hw, 6, generator=g).half(), w, 0) for w in windows]


def test_scatter_replay_matches_fp64_and_repeats_count_once():
    windows = _windows(24, 2)
    assert any(len(set(w)) < len(w) for w in windows)
    calls = _scatter_calls(windows, 2, 5, 7)
    acc0 = torch.zeros(2, 24, 5, 4)
    got = DR.scatter_replay(acc0, calls)
    ref = DR.scatter_ref(acc0, calls)
    assert GR.check(got.reshape(-1, 4), ref, "replay") < 1.0
    from aniportrait_b200.pipelines.sharding import accumulate
    want = acc0.clone()
    for pred, w, _ in calls:
        accumulate(want, pred[..., :4].float().view(2, len(w), 5, 4), w)
    assert torch.equal(got, want)


@pytest.mark.parametrize("bug", ["first_occurrence", "count_twice"])
def test_scatter_bug_is_rejected(bug):
    windows = _windows(24, 2)
    calls = _scatter_calls(windows, 2, 5, 8)
    acc0 = torch.zeros(2, 24, 5, 4)
    want = DR.exact_f32(DR.scatter_replay(acc0, calls), DR.locate_rows(24, 5, 2))
    bad = DR.scatter_replay(acc0, calls, bug=bug)
    with pytest.raises(AssertionError, match=r"plane \d, frame \d+, pixel \d, channel \d") as e:
        GR.check_exact(bad.reshape(-1, 4), want, bug)
    print(f"{bug}: rejected: {e.value}")


def test_gather_emulation_exact_and_dup_plane_bug_rejected():
    g = _gen(9)
    lat = torch.randn(24, 6, 4, generator=g).half()
    window = _windows(24, 2)[1]
    ref = DR.gather_ref(lat, window, 2, 16)
    GR.check_exact(DR.emulate_gather(lat, window, 2, 16), ref, "gather")
    with pytest.raises(AssertionError, match=r"dup plane 1, window frame \d+ \(latent frame \d+\), pixel \d") as e:
        GR.check_exact(DR.emulate_gather(lat, window, 2, 16, bug="dup_plane"), ref, "dup_plane")
    print(f"dup_plane: rejected: {e.value}")


def test_no_cfg_reference_loop_steps_on_the_sum():
    """The restated reference loop without CFG steps on the window sum; the product's step weights are 1 there, and
    1 / count under CFG (sharding.step_weights): the emulated kernel with those weights passes the loop reference, the
    averaged weights fail it without CFG."""
    from aniportrait_b200.pipelines.sharding import plan_windows, step_weights
    windows, inv = plan_windows(L, 25)
    sch, ts = _steps("v2_vpred_zero_snr")
    g = _gen(11)
    lat = torch.randn(L, HW, 4, generator=g).half()
    for guidance in (1.0, 3.5):
        cfg = guidance > 1.0
        dup = 2 if cfg else 1
        preds = [torch.randn(dup * len(w), HW, 4, generator=g).half() for w in windows]
        acc = DR.scatter_replay(torch.zeros(dup, L, HW, 4), [(p, w, 0) for p, w in zip(preds, windows)])
        a_t, a_p = sch.alpha_pair(ts[5])
        ref = DR.reference_loop_step(preds, windows, lat, guidance, a_t, a_p, "v_prediction", 0.0)
        _, y16 = DR.emulate_step(acc, step_weights(inv, cfg).float(), lat, guidance, a_t, a_p, "v_prediction", 0.0)
        GR.check(y16, ref, f"g={guidance}")
        if not cfg:
            _, avg = DR.emulate_step(acc, inv.float(), lat, guidance, a_t, a_p, "v_prediction", 0.0)
            with pytest.raises(AssertionError, match="frame"):
                GR.check(avg, ref, "averaged without CFG")


def test_layout_and_patchify_references():
    g = _gen(12)
    x = torch.randn(2, 4, 3, 5, 7, generator=g).half()
    ref = DR.ncfhw_to_nhwc_ref(x, 8)
    assert torch.equal(ref.o.view(2, 3, 35, 8)[..., 4:], torch.zeros(2, 3, 35, 4))
    nhwc = ref.o.view(6, 5, 7, 8).half()
    back = DR.nhwc_to_ncfhw_ref(nhwc, 2, 4, 3)
    assert torch.equal(back.o.view(2, 4, 3, 5, 7), x.double())
    px = torch.randn(2, 3, 28, 28, generator=g)
    pr = DR.patchify_ref(px, 14, 640)
    conv = torch.nn.functional.conv2d(px.double(), torch.eye(588, dtype=torch.float64).view(588, 3, 14, 14), stride=14)
    assert torch.equal(pr.o.view(2, 5, 640)[:, 1:, :588], conv.flatten(2).transpose(1, 2))
    assert torch.equal(pr.o.view(2, 5, 640)[:, 0], torch.nn.functional.one_hot(torch.tensor([588, 588]), 640).double())
    assert np.isclose(float(pr.o.view(2, 5, 640)[:, 1:, 588:].abs().sum()), 0.0)
