"""DPMSolverMultistepScheduler / EulerDiscreteScheduler on the H100:
  step        ap_cfg_multistep_step_f16 element by element against float64 (sampler_reference.py) on its own inputs, at
              every step of 2M midpoint (v-prediction, trailing), dpmsolver 2M heun (epsilon, Karras) and Euler
              (epsilon, linspace), with and without CFG, at the geometries of test_denoise_contract_gpu.py; the latents
              and the fp32 history both, the history untouched where the next step does not read it
  gather      ap_gather_window_scaled_f16 per element, its zero padding lanes, and the scale read from device memory
  refusals    bad arguments return AP_ERR_INVALID and write nothing
  pipeline    the product pipeline against pipeline_small_dpm / pipeline_small_euler (unmodified reference); graph replay,
              eager and repeated runs bit-identical; DDIM -> DPM -> DDIM on one pipe equal to fresh pipes; two GPUs in
              `windows` mode equal to one
"""
import os
import sys

import pytest
import torch

import gemm_reference as GR
import sampler_reference as SR
from helpers import build_pipeline, pipeline_inputs, rel_l2
from test_denoise_contract_gpu import GEOMS, _gather_plan, _gen, _idx, _report, _step_operands
from test_norm_contract_gpu import _abi, _f

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

SCHEDULES = {
    "dpmpp_2m_v_trailing": ("DPMSolverMultistepScheduler", 15, dict(prediction_type="v_prediction",
                                                                      timestep_spacing="trailing")),
    "dpm_2m_heun_eps_karras": ("DPMSolverMultistepScheduler", 10, dict(algorithm_type="dpmsolver", solver_type="heun",
                                                                        use_karras_sigmas=True)),
    "euler_eps_linspace": ("EulerDiscreteScheduler", 25, dict()),
}


def _table(name):
    from aniportrait_b200.pipelines.scheduler import multistep_coefficients
    cls, steps, kw = SCHEDULES[name]
    return multistep_coefficients(SR.make_scheduler(cls, steps, **kw))


def step_call(acc_p, w, cfg, g, co, hist_p, lat_p, L, HW, store=None):
    from aniportrait_b200._lib import I, fptr
    _abi("ap_cfg_multistep_step_f16", acc_p, fptr(w), I(1 if cfg else 0), _f(g), _f(co.c_xx), _f(co.c_xv), _f(co.k_x),
         _f(co.k_0), _f(co.k_1), I(int(co.store if store is None else store)), hist_p, lat_p, I(L), I(HW))


CASES = [(s, g, m) for s in SCHEDULES for g in (1.0, 3.5) for m in GEOMS]


@pytest.mark.parametrize("sched,guidance,geom", CASES, ids=[f"{s}-g{g}-{m}" for s, g, m in CASES])
def test_multistep_step_every_step(cuda_dev, sched, guidance, geom):
    from aniportrait_b200._lib import fptr, ptr
    gm = GEOMS[geom]
    L, HW = gm["L"], gm["h"] * gm["w"]
    cfg = guidance > 1.0
    P = 2 if cfg else 1
    table = _table(sched)
    lat = (1.5 * torch.randn(L, HW, 4, generator=_gen(7))).half()
    hist = torch.full((L, HW, 4), float("nan"))          # what the buffer holds before a video's first step
    worst = 0.0
    for i, co in enumerate(table):
        acc, w = _step_operands(L, HW, cfg, 200 + i)
        w_d = w.to(cuda_dev)
        runs = []
        for _ in range(2):
            la = GR.Guarded(L * HW, 4, 4, torch.float16, cuda_dev)
            hi = GR.Guarded(L * HW, 4, 4, torch.float32, cuda_dev)
            ac = GR.Guarded(P * L * HW, 4, 4, torch.float32, cuda_dev)
            la.view.copy_(lat.view(-1, 4))
            hi.view.copy_(hist.view(-1, 4))
            ac.view.copy_(acc.view(-1, 4))
            step_call(fptr(ac.view), w_d, cfg, guidance, co, fptr(hi.view), ptr(la.view), L, HW)
            torch.cuda.synchronize()
            for buf, what in ((la, "latents"), (hi, "history"), (ac, "acc")):
                buf.check(f"{sched} step {i}: {what}")
            assert bool((ac.view == 0).all()), f"{sched} step {i}: acc not zeroed"
            runs.append((la, hi))
        assert torch.equal(runs[0][0].bits, runs[1][0].bits) and torch.equal(runs[0][1].bits, runs[1][1].bits)
        ref, mref = SR.step_ref(acc, w, lat, hist, guidance, co)
        out, h_out = runs[0][0].view.cpu(), runs[0][1].view.cpu()
        what = f"{sched} g={guidance} {geom} step {i} (t={co.timestep:.6g}, k_1={co.k_1:.4g})"
        worst = max(worst, GR.check(out, ref, what))
        if co.store:
            GR.check(h_out, mref, what + ": history")
        else:
            assert torch.equal(h_out.view(torch.int32), hist.view(-1, 4).view(torch.int32)), what + ": history written"
        lat, hist = out.view(L, HW, 4), h_out.view(L, HW, 4)
    assert worst > 0.0
    _report("cfg_multistep_step", f"{sched} g={guidance} {geom}", worst)


@pytest.mark.parametrize("mode", ["window", "window_no_cfg", "group", "unit"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_gather_window_scaled(cuda_dev, geom, mode):
    from aniportrait_b200._lib import I, fptr, ptr
    g = GEOMS[geom]
    L, HW, cpad = g["L"], g["h"] * g["w"], 64
    lat = (3 * torch.randn(L, HW, 4, generator=_gen(3))).half()
    lat_d = lat.to(cuda_dev)
    scale_d = torch.zeros(1, dtype=torch.float32, device=cuda_dev)
    table = _table("euler_eps_linspace")
    for window, dup in _gather_plan(geom, mode):
        idx = _idx(window, cuda_dev)
        F = len(window)
        out = GR.Guarded(dup * F * HW, cpad, cpad, torch.float16, cuda_dev)
        for co in (table[0], table[12], table[-1]):              # the same launch reads each step's device value
            scale_d.fill_(co.scale)
            _abi("ap_gather_window_scaled_f16", ptr(lat_d), ptr(idx), fptr(scale_d), ptr(out.view), I(dup), I(F), I(HW),
                 I(cpad))
            torch.cuda.synchronize()
            out.check(f"{geom} {mode}")
            ref = SR.gather_scaled_ref(lat, window, dup, cpad, co.scale)
            got = out.view.cpu()
            GR.check(got, ref, f"{geom} {mode} scale {co.scale:.6g}")
            assert bool((got[:, 4:] == 0).all()) and not torch.signbit(got[:, 4:]).any(), "padding lanes must be +0"
    assert torch.equal(lat_d.cpu(), lat)


def test_refusals(cuda_dev):
    from aniportrait_b200._lib import ApError, I, fptr, ptr
    table = _table("dpmpp_2m_v_trailing")
    L, HW = 4, 16
    acc = torch.zeros(2, L, HW, 4, device=cuda_dev)
    w = torch.ones(L, device=cuda_dev)
    lat = GR.Guarded(L * HW, 4, 4, torch.float16, cuda_dev)
    lat.view.zero_()
    before = lat.bits.clone()
    nul = fptr(None)
    bad = [("k_1 != 0 without history", lambda: step_call(fptr(acc), w, True, 3.5, table[1], nul, ptr(lat.view), L, HW)),
           ("store without history", lambda: step_call(fptr(acc), w, True, 3.5, table[0], nul, ptr(lat.view), L, HW)),
           ("L = 0", lambda: step_call(fptr(acc), w, True, 3.5, table[2], fptr(acc), ptr(lat.view), 0, HW))]
    import copy
    nan = copy.copy(table[1])
    nan.k_0 = float("nan")
    bad.append(("non-finite k_0", lambda: step_call(fptr(acc), w, True, 3.5, nan, fptr(acc), ptr(lat.view), L, HW)))
    out = torch.empty(16, 8, dtype=torch.float16, device=cuda_dev)
    idx = torch.zeros(1, dtype=torch.int32, device=cuda_dev)
    bad.append(("gather without scale", lambda: _abi("ap_gather_window_scaled_f16", ptr(lat.view), ptr(idx), nul,
                                                     ptr(out), I(1), I(1), I(HW), I(8))))
    for what, call in bad:
        with pytest.raises(ApError, match="rc=-1"):
            call()
    torch.cuda.synchronize()
    assert torch.equal(lat.bits, before), "a refused call wrote the latents"


# ---------------------------------------------------------------------------------------------------- pipeline
def _sched(name_or_gold):
    from aniportrait_b200.pipelines import scheduler as S
    if isinstance(name_or_gold, dict):
        return getattr(S, name_or_gold["cls"])(**name_or_gold["kwargs"])
    cls, _, kw = SCHEDULES[name_or_gold]
    return getattr(S, cls)(**dict(SR.BASE, **kw))


@pytest.mark.parametrize("case", ["pipeline_small_dpm", "pipeline_small_euler"])
def test_pipeline_against_reference_golden(cuda_dev, case):
    gold = torch.load(os.path.join(GOLDEN, case + ".pt"))
    P = gold["params"]
    pipe = build_pipeline(P, cuda_dev)
    pipe.scheduler = _sched(gold["scheduler"])
    ref_image, poses, ref_pose = pipeline_inputs(P["size"], P["L"], P["seeds"]["inputs"])
    trace = []
    lat0 = torch.randn((1, 4, P["L"], P["size"] // 8, P["size"] // 8), generator=torch.manual_seed(P["seeds"]["latents"]))
    out = pipe(ref_image, poses, ref_pose, P["size"], P["size"], P["L"], P["steps"], P["guidance"],
               latents=lat0.to(torch.float16), callback=lambda i, t, l: trace.append(l.clone()), callback_steps=1)
    assert len(trace) == P["steps"]
    e_first = rel_l2(trace[0], gold["first_step_latents"])
    e_final = rel_l2(trace[-1], gold["final_latents"])
    e_video = rel_l2(out.videos[:, :, [0, 7, P["L"] - 1]], gold["video_frames"])
    print(f"{case} rel-L2: first step {e_first:.3e}, final latents {e_final:.3e}, video frames {e_video:.3e}")
    assert e_first < 1e-2 and e_final < 1e-2 and e_video < 1e-2


def _args(P, L, steps):
    ref_image, poses, ref_pose = pipeline_inputs(P["size"], L, P["seeds"]["inputs"])
    return (ref_image, poses, ref_pose, P["size"], P["size"], L, steps, P["guidance"])


@pytest.mark.parametrize("name", ["dpmpp_2m_v_trailing", "euler_eps_linspace"])
def test_graph_replay_eager_and_repeats_are_bit_identical(cuda_dev, name):
    """Captured session (first video), replays with other latents in between, and the eager path: the same bytes. The
    history of the previous video must not leak into the next (its first step never reads it)."""
    P = torch.load(os.path.join(GOLDEN, "pipeline_small_dpm.pt"))["params"]
    pipe = build_pipeline(P, cuda_dev)
    pipe.scheduler = _sched(name)
    L = 24
    args = _args(P, L, 4)
    shape = (1, 4, L, P["size"] // 8, P["size"] // 8)
    lat_a = torch.randn(shape, generator=torch.manual_seed(5)).to(torch.float16)
    lat_b = torch.randn(shape, generator=torch.manual_seed(6)).to(torch.float16)

    def run(lat, graph):
        pipe.use_cuda_graph = graph
        v = pipe(*args, latents=lat.clone(), output_type="cuda").videos.clone()
        return pipe.last_latents.clone(), v
    a1, va1 = run(lat_a, True)
    b1, _ = run(lat_b, True)
    a2, va2 = run(lat_a, True)
    ae, vae_ = run(lat_a, False)
    assert len(pipe._sessions) == 1
    assert rel_l2(b1, a1) > 1e-1
    assert torch.equal(a2, a1) and torch.equal(ae, a1) and torch.equal(va2, va1) and torch.equal(vae_, va1)


def test_ddim_dpm_ddim_on_one_pipe_equals_fresh_pipes(cuda_dev):
    from aniportrait_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    P = torch.load(os.path.join(GOLDEN, "pipeline_small.pt"))["params"]
    args = _args(P, 20, 4)
    lat = torch.randn((1, 4, 20, P["size"] // 8, P["size"] // 8), generator=torch.manual_seed(8)).to(torch.float16)

    def video(pipe):
        pipe(*args, latents=lat.clone())
        return pipe.last_latents.clone()
    shared = build_pipeline(P, cuda_dev)
    ddim = shared.scheduler
    dpm = DPMSolverMultistepScheduler.from_config(ddim.config)
    got = []
    for s in (ddim, dpm, ddim):
        shared.scheduler = s
        got.append(video(shared))
    fresh = []
    for s in (ddim, dpm):
        p = build_pipeline(P, cuda_dev)
        p.scheduler = s
        fresh.append(video(p))
    assert rel_l2(fresh[1], fresh[0]) > 1e-2, "the two samplers must differ"
    assert torch.equal(got[0], fresh[0]) and torch.equal(got[1], fresh[1]) and torch.equal(got[2], fresh[0])


def _worker(rank, world, port, q):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    from aniportrait_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    P = torch.load(os.path.join(GOLDEN, "pipeline_small.pt"))["params"]
    pipe = build_pipeline(P, dev)
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)
    L = 24
    args = _args(P, L, 5)
    lat0 = torch.randn((1, 4, L, P["size"] // 8, P["size"] // 8), generator=torch.manual_seed(5)).to(torch.float16)
    single = None
    if rank == 0:
        pipe(*args, latents=lat0.clone())
        single = pipe.last_latents.cpu()
    pipe(*args, latents=lat0.clone(), dist_mode="windows")
    q.put((rank, single, pipe.last_latents.cpu()))
    dist.barrier()
    dist.destroy_process_group()


def test_windows_mode_two_gpus_matches_one(cuda_dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        r, single, sharded = q.get(timeout=900)
        res[r] = (single, sharded)
    for p in procs:
        p.join(timeout=120)
    assert all(p.exitcode == 0 for p in procs)
    assert torch.equal(res[0][1], res[0][0]) and torch.equal(res[1][1], res[0][0])
