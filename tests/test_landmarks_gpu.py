"""Landmark pose frames and face-mesh projection on the device (ap_draw_landmarks_u8 / ap_project_points_f64) against the
UNMODIFIED reference's frames and projections (tests/golden/landmark_frames_reference.npz) and the integer restatement
(tests/landmark_reference.py); the pipeline's CUDA uint8 pose-frame intake against the numpy one."""
import os
from collections import namedtuple

import numpy as np
import pytest
import torch

import landmark_reference as LR

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "landmark_frames_reference.npz")
Spec = namedtuple("Spec", "color thickness circle_radius")


class StandInVisualizer:
    """The two attributes of FaceMeshVisualizer the kernels use: face_connection_spec and draw_landmarks."""

    def __init__(self, edges, colors, thickness=2):
        self.face_connection_spec = {tuple(int(v) for v in e): Spec(tuple(int(v) for v in c), thickness, 1)
                                     for e, c in zip(edges, colors)}

    def draw_landmarks(self, image_size, keypoints, normed=False):
        raise AssertionError("enable_kernels did not rebind draw_landmarks")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def vis(gold):
    from aniportrait_b200.pipelines import landmarks as LM
    return [LM.enable_kernels(StandInVisualizer(gold[f"spec{s}_edges"], gold[f"spec{s}_colors"])) for s in (0, 1)]


def test_device_frames_equal_the_reference_frames(cuda_dev, gold, vis):
    for i, name in enumerate(gold["case_names"]):
        s, normed = int(gold["case_spec"][i]), bool(gold["case_normed"][i])
        kp = torch.from_numpy(gold["case_keypoints"][i][None]).to(cuda_dev)
        out = vis[s].draw_landmarks_batch((512, 512), kp, normed=normed)
        assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (1, 512, 512, 3)
        assert torch.equal(out[0].cpu(), torch.from_numpy(gold["case_frames"][i])), name


def test_draw_landmarks_returns_the_reference_numpy_frame(cuda_dev, gold, vis):
    for i in range(len(gold["case_names"])):
        s, normed = int(gold["case_spec"][i]), bool(gold["case_normed"][i])
        img = vis[s].draw_landmarks((512, 512), gold["case_keypoints"][i], normed=normed)
        assert isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.shape == (512, 512, 3)
        assert np.array_equal(img, gold["case_frames"][i]), gold["case_names"][i]


@pytest.mark.parametrize("normed", [True, False])
def test_device_frames_equal_the_restatement_on_seeded_keypoints(cuda_dev, gold, vis, normed):
    rng = np.random.default_rng(31 if normed else 32)
    kp = rng.uniform(-0.05, 1.05, (64, 468, 2)) * (1.0 if normed else 512.0)
    kp[5, 7] = np.nan
    s = 1 if normed else 0
    out = vis[s].draw_landmarks_batch((512, 512), torch.from_numpy(kp).to(cuda_dev), normed=normed).cpu().numpy()
    ref = LR.draw_frames(kp, gold[f"spec{s}_edges"], gold[f"spec{s}_colors"], normed=normed)
    bad = [i for i in range(len(kp)) if not np.array_equal(out[i], ref[i])]
    assert not bad, f"frames {bad} differ"


def test_one_launch_of_600_frames_equals_the_restatement(cuda_dev, gold, vis):
    from aniportrait_b200 import ops
    rng = np.random.default_rng(33)
    L = 600
    kp = gold["proj_a"][rng.integers(0, len(gold["proj_a"]), L)] + rng.normal(0, 3.0, (L, 1, 2)) \
        + rng.normal(0, 0.7, (L, 468, 2))
    dev = torch.from_numpy(kp).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    out = vis[0].draw_landmarks_batch((512, 512), dev)
    assert ops.KERNEL_LAUNCHES - n0 == 1
    again = vis[0].draw_landmarks_batch((512, 512), dev)
    assert torch.equal(out, again)
    out = out.cpu().numpy()
    ref = LR.draw_frames(kp, gold["spec0_edges"], gold["spec0_colors"])
    bad = [i for i in range(L) if not np.array_equal(out[i], ref[i])]
    assert not bad, f"frames {bad} differ"


def test_device_projection_matches_the_reference(cuda_dev, gold):
    from aniportrait_b200.pipelines import landmarks as LM
    from aniportrait_b200 import ops
    offs = torch.from_numpy(gold["offsets"]).to(cuda_dev)               # fp32, as a2m_model.infer leaves it on the device
    n0 = ops.KERNEL_LAUNCHES
    a = LM.project_points(offs, gold["trans_mat"], gold["pose_seq"], [512, 512], base=gold["mesh_base"])
    assert ops.KERNEL_LAUNCHES - n0 == 1
    assert a.is_cuda and a.dtype == torch.float64 and a.shape == gold["proj_a"].shape
    assert (a.cpu().numpy() - gold["proj_a"]).__abs__().max() <= 1e-9
    host_sum = LM.project_points(gold["offsets"] + gold["mesh_base"], gold["trans_mat"], gold["pose_seq"], [512, 512])
    assert torch.equal(host_sum, a)                                       # the fp64 add on the device is numpy's add
    b = LM.project_points_with_trans(gold["vid_verts"], gold["vid_mats"], [512, 512])
    assert (b.cpu().numpy() - gold["proj_b"]).__abs__().max() <= 1e-9
    # projection -> drawing gives the reference's bytes
    for i, name in enumerate(gold["case_names"]):
        if name.startswith("projected_a"):
            k = int(name[len("projected_a"):].split("_")[0])
            s = int(gold["case_spec"][i])
            vis = LM.enable_kernels(StandInVisualizer(gold[f"spec{s}_edges"], gold[f"spec{s}_colors"]))
            out = vis.draw_landmarks_batch((512, 512), a[k:k + 1])
            assert torch.equal(out[0].cpu(), torch.from_numpy(gold["case_frames"][i])), name
    out = LM.enable_kernels(StandInVisualizer(gold["spec0_edges"], gold["spec0_colors"])).draw_landmarks_batch(
        (512, 512), b[:1])
    i = list(gold["case_names"]).index("projected_b0_s0")
    assert torch.equal(out[0].cpu(), torch.from_numpy(gold["case_frames"][i]))


def test_draws_the_landmarkers_three_column_output_as_the_reference(cuda_dev, gold, vis):
    """vis.draw_landmarks(size, lmks, normed=True) with LMKExtractor's float32 [478, 3] (x, y, z) landmarks, as
    audio2vid.py:153-155 and vid2vid.py:139-140 draw the reference pose; the batch form takes [L, 478, 3] on the device."""
    lmks = gold["lmks478"]
    for s in (0, 1):
        img = vis[s].draw_landmarks((512, 512), lmks, normed=True)
        assert np.array_equal(img, gold["lmks478_frames"][s]), s
        batch = vis[s].draw_landmarks_batch((512, 512), torch.from_numpy(np.stack([lmks, lmks])).to(cuda_dev),
                                            normed=True)
        assert torch.equal(batch.cpu(), torch.from_numpy(np.stack([gold["lmks478_frames"][s]] * 2))), s


def test_errors_raise_before_any_launch(cuda_dev, gold, vis):
    from aniportrait_b200 import _lib, ops
    from aniportrait_b200.pipelines import landmarks as LM
    kp = torch.rand(2, 468, 2, dtype=torch.float64, device=cuda_dev) * 512
    n0 = ops.KERNEL_LAUNCHES
    with pytest.raises(ValueError):
        vis[0].draw_landmarks_batch((512, 512), kp[:, :300])              # edge indices beyond N
    with pytest.raises(ValueError):
        vis[0].draw_landmarks_batch((512, 512), kp[:, :, :1])              # fewer than two columns
    with pytest.raises(NotImplementedError):
        vis[0].draw_landmarks_batch((256, 512), kp)
    with pytest.raises(NotImplementedError):
        vis[0].draw_landmarks((512, 768), kp[0].cpu().numpy())
    with pytest.raises(NotImplementedError):
        LM.enable_kernels(StandInVisualizer(gold["spec0_edges"], gold["spec0_colors"], thickness=3))
    with pytest.raises(_lib.ApError):
        ops.draw_landmarks(kp, 512.0, 512.0, False, gold["spec0_edges"], gold["spec0_colors"], thickness=1)
    with pytest.raises(_lib.ApError):
        ops.draw_landmarks(kp, 512.0, 512.0, False, [[0, 468]], [[1, 2, 3]])
    torch.cuda.synchronize()
    assert ops.KERNEL_LAUNCHES == n0


def test_pipeline_takes_device_pose_frames(cuda_dev):
    """The same pose bytes as numpy frames and as a CUDA uint8 tensor [L, H, W, 3] give bit-identical videos, eager and
    under graph replay."""
    from helpers import build_pipeline, pipeline_inputs
    gold = torch.load(os.path.join(os.path.dirname(GOLDEN), "pipeline_small.pt"))
    P = gold["params"]
    pipe = build_pipeline(P, cuda_dev)
    L = 8
    ref_image, poses, ref_pose = pipeline_inputs(P["size"], L, P["seeds"]["inputs"])
    dev_poses = torch.from_numpy(np.stack(poses)).to(cuda_dev)
    lat = torch.randn((1, 4, L, P["size"] // 8, P["size"] // 8), generator=torch.manual_seed(9)).to(torch.float16)
    pose_np = pipe._pose_maps_to_tensor(poses, P["size"], P["size"], cuda_dev)
    pose_dev = pipe._pose_maps_to_tensor(dev_poses, P["size"], P["size"], cuda_dev)
    assert pose_dev.dtype == torch.float32 and torch.equal(pose_np, pose_dev)
    for graph in (False, True):
        pipe.use_cuda_graph = graph
        args = (ref_image, None, ref_pose, P["size"], P["size"], L, 2, P["guidance"])
        va = pipe(args[0], poses, *args[2:], latents=lat.clone()).videos
        vb = pipe(args[0], dev_poses, *args[2:], latents=lat.clone()).videos
        assert torch.equal(va, vb), f"graph={graph}"
