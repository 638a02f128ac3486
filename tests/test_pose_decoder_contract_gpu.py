"""The call contract of the Audio2Pose decoder kernel (ap_pose_decoder_f16 and its traced twin ap_pose_decoder_trace_f16),
element by element against float64 (pose_decoder_reference.py): every cache row, every stage of every layer at every
step (q, attention, LN2, feed-forward, LN3), the poses and the next tokens, each against fp64 evaluated on what the kernel
itself consumed.

  caller       the seeded full-size a2p, its ALiBi mask and positional table at 600 positions, cross from the library
               GEMM on synthetic features, T = 1 .. 600
  boundaries   T around the 64-key P.V groups and the 512-key second score slot, T = 1024, mask_len > T, pe_len != mask_len
  geometry     layers 1, 2, 3, 12 (odd counts flip the parameter-block parity between steps), out_dim 1 and 8
  masks        NaN above the diagonal (only j <= i may be read), rows left with the diagonal only, offsets of +-60
  scales       q / k rows of in_proj x 4 (sharp softmax), a linear2 bias of +30 (LayerNorm with mean / sigma >> 1)
  identity     traced and untraced calls give equal bytes; AP_POSE_CTAS=8 in a child process gives the 16-CTA bytes,
               through the test hook and through ap_pose_decoder_f16 (the shipped 8-CTA fallback);
               AP_PDL=1 in a child process gives the same poses through PoseDecoder.decode
  refusals     misaligned pointers and out-of-contract shapes return AP_ERR_INVALID, write nothing and launch nothing

Every call goes through the C ABI into guarded buffers whose interiors start as NaN; it runs twice and both results must
be bit-identical; the inputs must be unchanged. The worst ratio of error to bound is printed per case (run with -s).
"""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

import gemm_reference as GR
import pose_decoder_reference as PR
from test_gemm_contract_gpu import _snapshot, _unchanged

pytestmark = pytest.mark.gpu

SAVE = "AP_POSE_CONTRACT_SAVE"          # set in the child processes: the directory the parent compares against
SAVED = ("caller_T150", "boundary_T513", "geometry_L3", "geometry_od8")
INPUTS = ("w_qkv", "w_out", "w_ff1", "w_ff2", "vec", "pose_map_w", "pose_map_b", "pose_map_r_w", "pose_map_r_b", "pe",
          "id_row", "mask", "cross")


def _report(family, name, worst):
    print(f"\n[{family}] {name}: worst error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def _params_struct(P, T, **over):
    from aniportrait_b200 import _lib
    L, od = P["w_qkv"].shape[0], P["pose_map_r_w"].shape[0]
    kw = dict(layers=L, out_dim=od, embed_dim=PR.E, heads=PR.HEADS, ffn_dim=PR.FF, mask_len=P["mask"].shape[1],
              pe_len=P["pe"].shape[0], eps=P["eps"], **{k: P[k].data_ptr() for k in INPUTS})
    kw.update(over)
    return _lib.PoseDecoderParams(**kw)


class _Bufs:
    """kv fp16 [L, 2, 8, T, 64], out fp32 [T, od], trace fp32 [T, 5 L + 1, 512] in guard bands, interiors NaN."""

    def __init__(self, P, T, dev):
        L, od = P["w_qkv"].shape[0], P["pose_map_r_w"].shape[0]
        self.T, self.L, self.od = T, L, od
        self.g = [GR.Guarded(L * 2 * PR.HEADS * T, PR.D, PR.D, torch.float16, dev),
                  GR.Guarded(T, od, od, torch.float32, dev),
                  GR.Guarded(T * (PR.STAGES * L + 1), PR.E, PR.E, torch.float32, dev)]
        for b in self.g:
            b.view.fill_(math.nan)

    def views(self):
        kv, out, tr = (b.view for b in self.g)
        return (out, kv.view(self.L, 2, PR.HEADS, self.T, PR.D), tr.view(self.T, PR.STAGES * self.L + 1, PR.E))

    def bits(self):
        return [b.bits.clone() for b in self.g]

    def check(self, what):
        for b in self.g:
            b.check(what)


def _abi(P, T, bufs, traced=True, **over):
    from aniportrait_b200 import _lib, ops
    ops._ensure(P["cross"])
    prm = _params_struct(P, T, **over)
    kv, out, tr = (b.view for b in bufs.g)
    if traced:
        rc = _lib.lib().ap_pose_decoder_trace_f16(ctypes.byref(prm), _lib.I(T), _lib.ptr(kv), _lib.fptr(out),
                                                 _lib.fptr(tr), _lib.stream_ptr())
    else:
        rc = _lib.lib().ap_pose_decoder_f16(ctypes.byref(prm), _lib.I(T), _lib.ptr(kv), _lib.fptr(out),
                                           _lib.stream_ptr())
    return rc


def run_traced(P, T, name, dev, traced=True):
    """Two calls into guarded buffers: bit-identical, guard bands intact, inputs unchanged -> (out, kv, trace)."""
    from aniportrait_b200 import _lib
    entry = "ap_pose_decoder_trace_f16" if traced else "ap_pose_decoder_f16"
    bufs = _Bufs(P, T, dev)
    snap = _snapshot(*(P[k] for k in INPUTS))
    _lib.check(_abi(P, T, bufs, traced), entry)
    torch.cuda.synchronize()
    first = bufs.bits()
    _lib.check(_abi(P, T, bufs, traced), entry)
    torch.cuda.synchronize()
    for a, b in zip(first, bufs.bits()):
        assert torch.equal(a, b), f"{name}: two calls differ"
    bufs.check(name)
    _unchanged(snap, name)
    return bufs.views()


def _check_case(P, T, name, family, dev):
    out, kv, trace = run_traced(P, T, name, dev)
    if os.environ.get(SAVE) and name in SAVED:
        torch.save(dict(out=out.cpu(), kv=kv.cpu(), trace=trace.cpu()), os.path.join(os.environ[SAVE], name + ".pt"))
    worst = PR.check(P, T, out, kv, trace, name)
    _report(family, name, worst)
    return out, kv, trace


# ---------------------------------------------------------------------------------------------------- operands
@pytest.fixture(scope="module")
def a2p(cuda_dev):
    from aniportrait_b200.audio_models.pose_decoder import pack_decoder
    from pose_decoder_helpers import build_a2p_full
    m = build_a2p_full().to(cuda_dev)
    pk = pack_decoder(m, True, 1)
    pe = m.PPE.pe.detach().reshape(-1, PR.E).to(cuda_dev, torch.float32).contiguous()
    mask = m.biased_mask.detach().to(cuda_dev, torch.float32).contiguous()
    return pk, pe, mask


def _a2p_params(a2p, T, seed=None):
    """The a2p decoder's packed operands with cross from the library GEMM on features(T), as PoseDecoder._run does."""
    from aniportrait_b200 import ops
    from pose_decoder_helpers import features
    pk, pe, mask = a2p
    dev = pe.device
    feats = features(T, seed=T if seed is None else seed)[0].to(dev).half()
    cross = ops.gemm(feats, pk["cross_w"], bias=pk["cross_b"], out_f32=True)
    return dict(pk["layers"], pose_map_w=pk["pose_map_w"], pose_map_b=pk["pose_map_b"], pose_map_r_w=pk["pose_map_r_w"],
                pose_map_r_b=pk["pose_map_r_b"], pe=pe, id_row=pk["id_w"][3].contiguous(), mask=mask,
                cross=cross.contiguous(), eps=pk["eps"])


def _synthetic(dev, L=2, od=6, T=64, ml=None, pl=None, seed=0, mask="alibi"):
    return PR.synthetic_params(L, od, T, ml or T, pl or T, seed=seed, device=dev, mask=mask)


# ---------------------------------------------------------------------------------------------------- cases
@pytest.mark.parametrize("T", [1, 2, 42, 150, 299, 600])
def test_caller(cuda_dev, a2p, T):
    _check_case(_a2p_params(a2p, T), T, f"caller_T{T}", "caller", cuda_dev)


@pytest.mark.parametrize("T", [63, 64, 65, 511, 512, 513])
def test_boundary(cuda_dev, a2p, T):
    _check_case(_a2p_params(a2p, T), T, f"boundary_T{T}", "boundaries", cuda_dev)


@pytest.mark.parametrize("name,kw,T", [
    ("T1024", dict(T=1024, ml=1024, pl=1024), 1024),
    ("mask_len_gt_T", dict(T=100, ml=130, pl=130), 100),
    ("mask_len_eq_T", dict(T=100, ml=100, pl=100), 100),
    ("pe_len_ne_mask_len", dict(T=90, ml=97, pl=150), 90),
])
def test_boundary_synthetic(cuda_dev, name, kw, T):
    _check_case(_synthetic(cuda_dev, **kw), T, name, "boundaries", cuda_dev)


@pytest.mark.parametrize("name,L,od", [("geometry_L1", 1, 6), ("geometry_L2", 2, 6), ("geometry_L3", 3, 6),
                                       ("geometry_L12", 12, 6), ("geometry_od1", 2, 1), ("geometry_od8", 3, 8)])
def test_geometry(cuda_dev, name, L, od):
    T = 70
    _check_case(_synthetic(cuda_dev, L=L, od=od, T=T, seed=L * 10 + od), T, name, "geometry", cuda_dev)


def _mask_variant(P, kind, seed=5):
    m = P["mask"].clone()
    n = m.shape[1]
    i = torch.arange(n, device=m.device).view(n, 1)
    j = torch.arange(n, device=m.device).view(1, n)
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "nan_above":
        rnd = (torch.randn(m.shape, generator=g) * 2).to(m.device)
        m = torch.where(j <= i, rnd, torch.full_like(m, math.nan))
    elif kind == "diagonal_only_rows":
        m[:, ::3] = torch.where(j < i, torch.full_like(m, -math.inf), m)[:, ::3]
    else:
        m = m + (60.0 if kind == "offset_plus_60" else -60.0)
    P["mask"] = m.contiguous()
    return P


@pytest.mark.parametrize("kind", ["nan_above", "diagonal_only_rows", "offset_plus_60", "offset_minus_60"])
def test_masks(cuda_dev, a2p, kind):
    T = 150
    _check_case(_mask_variant(_a2p_params(a2p, T), kind), T, f"mask_{kind}", "masks", cuda_dev)


@pytest.mark.parametrize("kind", ["qk_x4", "linear2_bias_30"])
def test_operand_scales(cuda_dev, a2p, kind):
    T = 150
    P = _a2p_params(a2p, T)
    if kind == "qk_x4":
        w = P["w_qkv"].clone()
        w[:, :2 * PR.E] *= 4
        P["w_qkv"] = w
    else:
        v = P["vec"].clone()
        v[:, PR.B_FF2:PR.B_FF2 + PR.E] += 30.0
        P["vec"] = v
    _check_case(P, T, f"scale_{kind}", "scales", cuda_dev)


# ---------------------------------------------------------------------------------------------------- identity
UNTRACED_T = (42, 513)


@pytest.mark.parametrize("T", UNTRACED_T)
def test_traced_equals_untraced(cuda_dev, a2p, T):
    """The production entry point (pose_decoder_kernel<NC, false>) gives the test hook's out and kv; in the AP_POSE_CTAS=8
    child this runs the 8-CTA production kernel, whose bytes the parent compares with its own."""
    P = _a2p_params(a2p, T)
    out_t, kv_t, _ = run_traced(P, T, f"traced_T{T}", cuda_dev)
    out_u, kv_u, _ = run_traced(P, T, f"untraced_T{T}", cuda_dev, traced=False)
    assert torch.equal(out_t, out_u) and torch.equal(kv_t, kv_u)
    if os.environ.get(SAVE):
        torch.save(dict(out=out_u.cpu(), kv=kv_u.cpu()), os.path.join(os.environ[SAVE], f"untraced_T{T}.pt"))


def test_cluster_size(cuda_dev):
    from aniportrait_b200 import ops
    n = ops.pose_decoder_ctas(0)
    print(f"\n[cluster] ap_pose_decoder_ctas: {n}")
    want = os.environ.get("AP_POSE_CTAS")
    assert n == (int(want) if want else n) and n in (8, 16)


def _child(env_extra, k, tmp):
    env = dict(os.environ, **env_extra, **{SAVE: str(tmp)})
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__),
           "-k", k]
    r = subprocess.run(cmd, env=env, cwd=root, timeout=1500, capture_output=True, text=True)
    tail = r.stdout + r.stderr
    for line in tail.splitlines():
        if line.startswith("[cluster]"):
            print("\n(child) " + line)
    assert r.returncode == 0, tail[-4000:]
    assert " passed" in tail
    return tail


def test_eight_ctas_in_child_process(cuda_dev, a2p, tmp_path):
    """AP_POSE_CTAS=8 is read when the cluster size is first chosen, so once per process: the per-element cases again in
    a child, whose out / kv / trace must equal the 16-CTA bytes (every row's dot product, LayerNorm and attention is
    computed the same way whichever CTA owns it)."""
    if os.environ.get(SAVE):
        pytest.skip("already running in a child")
    from aniportrait_b200 import ops
    if ops.pose_decoder_ctas(0) != 16:
        pytest.skip("this device runs the 8-CTA kernel already")
    tail = _child({"AP_POSE_CTAS": "8"}, "(caller or boundary or geometry or cluster or untraced) and not child",
                  tmp_path)
    assert "[cluster] ap_pose_decoder_ctas: 8" in tail
    for name in SAVED:
        kind, arg = name.split("_", 1)
        if kind in ("caller", "boundary"):
            T = int(arg[1:])
            P = _a2p_params(a2p, T)
        else:
            L, od = {"L3": (3, 6), "od8": (3, 8)}[arg]
            T = 70
            P = _synthetic(cuda_dev, L=L, od=od, T=T, seed=L * 10 + od)
        out, kv, trace = run_traced(P, T, name, cuda_dev)
        got = torch.load(os.path.join(tmp_path, name + ".pt"))
        for k, v in (("out", out), ("kv", kv), ("trace", trace)):
            assert torch.equal(got[k], v.cpu()), f"{name}: {k} of the 8-CTA kernel differs from the 16-CTA kernel"
    for T in UNTRACED_T:                             # the production kernels: <8, false> against <16, false>
        out, kv, _ = run_traced(_a2p_params(a2p, T), T, f"untraced_T{T}", cuda_dev, traced=False)
        got = torch.load(os.path.join(tmp_path, f"untraced_T{T}.pt"))
        assert torch.equal(got["out"], out.cpu()) and torch.equal(got["kv"], kv.cpu()), \
            f"T={T}: ap_pose_decoder_f16 with 8 CTAs differs from 16 CTAs"


PDL_T = (150, 600)


def test_pdl_decode_chain_in_child_process(cuda_dev, a2p, tmp_path):
    """AP_PDL=1 (programmatic dependent launch, read once per process): PoseDecoder.decode (cross GEMM -> decoder) in a
    child gives the bytes of this process's decode."""
    if os.environ.get(SAVE):
        pytest.skip("already running in a child")
    from aniportrait_b200.audio_models.pose_decoder import PoseDecoder
    from pose_decoder_helpers import build_a2p_full, features
    m = build_a2p_full().to(cuda_dev)
    for T in PDL_T:
        out = PoseDecoder(m).decode(features(T, seed=T).to(cuda_dev).half(), T, torch.tensor([3], device=cuda_dev))
        torch.save(out.cpu(), os.path.join(tmp_path, f"pdl_ref_T{T}.pt"))
    _child({"AP_PDL": "1"}, "pdl_decode_matches_parent", tmp_path)


def test_pdl_decode_matches_parent(cuda_dev):
    if not os.environ.get(SAVE) or os.environ.get("AP_PDL") != "1":
        pytest.skip("runs in the AP_PDL=1 child of test_pdl_decode_chain_in_child_process")
    from aniportrait_b200.audio_models.pose_decoder import PoseDecoder
    from pose_decoder_helpers import build_a2p_full, features
    m = build_a2p_full().to(cuda_dev)
    for T in PDL_T:
        out = PoseDecoder(m).decode(features(T, seed=T).to(cuda_dev).half(), T, torch.tensor([3], device=cuda_dev))
        want = torch.load(os.path.join(os.environ[SAVE], f"pdl_ref_T{T}.pt"))
        assert torch.equal(out.cpu(), want), f"T={T}: AP_PDL=1 changed the poses"


# ---------------------------------------------------------------------------------------------------- refusals
def _refusals(P, T):
    """(name, T, struct overrides, buffer offsets in elements) of calls the contract refuses."""
    two = 2                                          # bytes off the 16-byte grid
    r = [(f"{k}_misaligned", T, {k: P[k].data_ptr() + two}, None) for k in ("vec", "cross", "w_qkv", "w_out", "w_ff1",
                                                                            "w_ff2")]
    ml, pl = P["mask"].shape[1], P["pe"].shape[0]
    r += [("kv_misaligned", T, {}, "kv"), ("T_0", 0, {}, None), ("T_gt_mask_len", ml + 1, {"pe_len": ml + 5}, None),
          ("T_gt_pe_len", T, {"pe_len": T - 1}, None), ("T_1025", 1025, {"mask_len": 1025, "pe_len": 1025}, None),
          ("layers_0", T, {"layers": 0}, None), ("out_dim_0", T, {"out_dim": 0}, None),
          ("out_dim_9", T, {"out_dim": 9}, None), ("heads_4", T, {"heads": 4}, None), ("eps_0", T, {"eps": 0.0}, None)]
    return r


def test_refusals_write_nothing_and_launch_nothing(cuda_dev, a2p):
    from torch.profiler import ProfilerActivity, profile
    from aniportrait_b200 import _lib, ops
    T = 20
    P = _a2p_params(a2p, T)
    bufs = _Bufs(P, T, cuda_dev)
    before = bufs.bits()
    ops._ensure(P["cross"])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, t, over, buf in _refusals(P, T):
            if buf == "kv":
                kv, out, tr = (b.view for b in bufs.g)
                prm = _params_struct(P, t, **over)
                rc = _lib.lib().ap_pose_decoder_trace_f16(ctypes.byref(prm), _lib.I(t),
                                                         ctypes.c_void_p(kv.data_ptr() + 2), _lib.fptr(out),
                                                         _lib.fptr(tr), _lib.stream_ptr())
            else:
                rc = _abi(P, t, bufs, **over)
            assert rc == -1, f"{name}: rc {rc}, expected AP_ERR_INVALID"
            rc = _abi(P, t, bufs, traced=False, **over) if buf is None else rc
            assert rc == -1, f"{name} (untraced): rc {rc}"
        torch.cuda.synchronize()
    for a, b in zip(before, bufs.bits()):
        assert torch.equal(a, b), "a refused call wrote into the buffers"
    launched = [e.key for e in prof.key_averages() if "pose_decoder" in e.key]
    assert not launched, launched
