"""The cv2 INTER_LINEAR resize on the device (ap_resize_linear_u8 through landmarks.resize_frames and
vis.draw_pose_frames) against the integer restatement (tests/resize_reference.py) on seeded random frames, and against
the UNMODIFIED reference's landmark frames at sizes other than 512 x 512 and through vid2vid's two resizes
(tests/golden/landmark_frames_resized_reference.npz); the pipeline's intake of the resized frames."""
import hashlib
import os
from collections import namedtuple

import numpy as np
import pytest
import torch

import landmark_reference as LR
import resize_reference as RR

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "landmark_frames_resized_reference.npz")
Spec = namedtuple("Spec", "color thickness circle_radius")

# (w, h) -> (W, H): the canvas to every size the scripts draw at, back to 512 x 512, odd and degenerate sizes
SIZES = [((512, 512), s) for s in [(1080, 1920), (1920, 1080), (768, 768), (720, 1280), (1024, 1024), (513, 511),
                                   (600, 900), (3840, 2160), (576, 1024), (256, 256), (300, 200), (512, 768),
                                   (768, 512)]] \
    + [(s, (512, 512)) for s in [(1080, 1920), (1920, 1080), (720, 1280), (1000, 700), (1024, 1024)]] \
    + [((1, 1), (7, 5)), ((5, 7), (1, 1)), ((1, 9), (4, 13)), ((9, 1), (13, 4)), ((7, 3), (1, 17)), ((37, 23), (37, 23)),
       ((64, 64), (128, 128)), ((101, 61), (50, 30)), ((333, 17), (5, 1000)), ((8192, 2), (3, 8192))]
# src -> mid -> dst: vid2vid's chains (1024 -> 512 is cv2's exact 2x case), upscale then upscale, odd sizes
CHAINS = [((512, 512), (1080, 1920), (512, 512)), ((512, 512), (1920, 1080), (512, 512)),
          ((512, 512), (720, 1280), (512, 512)), ((512, 512), (1024, 1024), (512, 512)),
          ((512, 512), (768, 768), (1024, 1024)), ((300, 200), (513, 511), (97, 1201)), ((5, 3), (1, 1), (6, 9))]


class StandInVisualizer:
    """The two attributes of FaceMeshVisualizer the kernels use: face_connection_spec and draw_landmarks."""

    def __init__(self, edges, colors):
        self.face_connection_spec = {tuple(int(v) for v in e): Spec(tuple(int(v) for v in c), 2, 1)
                                     for e, c in zip(edges, colors)}

    def draw_landmarks(self, image_size, keypoints, normed=False):
        raise AssertionError("enable_kernels did not rebind draw_landmarks")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def vis(gold):
    from aniportrait_b200.pipelines import landmarks as LM
    return LM.enable_kernels(StandInVisualizer(gold["edges"], gold["colors"]))


def _frames(seed, L, w, h):
    return np.random.default_rng(seed).integers(0, 256, (L, h, w, 3), dtype=np.uint8)


def _sha(t):
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("src,dst", SIZES)
def test_resize_frames_equal_the_restatement(cuda_dev, src, dst):
    from aniportrait_b200 import ops
    from aniportrait_b200.pipelines import landmarks as LM
    L = 1 if max(src + dst) > 2048 else 3
    frames = _frames(src[0] * 131 + dst[1], L, *src)
    n0 = ops.KERNEL_LAUNCHES
    out = LM.resize_frames(torch.from_numpy(frames).to(cuda_dev), dst)
    assert ops.KERNEL_LAUNCHES - n0 == 1
    assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (L, dst[1], dst[0], 3)
    want = RR.resize_frames(frames, dst)
    got = out.cpu().numpy()
    bad = int((got != want).sum())
    assert bad == 0, f"{bad} bytes differ"


@pytest.mark.parametrize("src,mid,dst", CHAINS)
def test_fused_chain_equals_two_resizes(cuda_dev, src, mid, dst):
    from aniportrait_b200 import ops
    frames = torch.from_numpy(_frames(mid[0] + src[1], 2, *src)).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    fused = ops.resize_linear_u8(frames, dst, mid=mid)
    assert ops.KERNEL_LAUNCHES - n0 == 1
    two = ops.resize_linear_u8(ops.resize_linear_u8(frames, mid), dst)
    assert fused.shape == (2, dst[1], dst[0], 3)
    assert torch.equal(fused, two)
    want = RR.resize_frames(RR.resize_frames(frames.cpu().numpy(), mid), dst)
    assert np.array_equal(fused.cpu().numpy(), want)


def test_draw_pose_frames_equal_the_reference_at_one_resize(cuda_dev, gold, vis):
    """audio2vid at -W/-H other than 512: draw_landmarks((W, H), kp) of the reference, one draw and one resize launch."""
    from aniportrait_b200 import ops
    for name in gold["one_names"]:
        key = f"one_{name}"
        W, H = (int(v) for v in gold[f"{key}_size"])
        kp = torch.from_numpy(gold[f"{key}_keypoints"][None]).to(cuda_dev)
        n0 = ops.KERNEL_LAUNCHES
        out = vis.draw_pose_frames((W, H), kp, normed=bool(gold[f"{key}_normed"]))
        assert ops.KERNEL_LAUNCHES - n0 == 2
        assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (1, H, W, 3), key
        if f"{key}_frame" in gold:
            assert torch.equal(out[0].cpu(), torch.from_numpy(gold[f"{key}_frame"])), key
        else:
            assert _sha(out[0]) == str(gold[f"{key}_sha256"]), key
        again = vis.draw_pose_frames((W, H), kp, normed=bool(gold[f"{key}_normed"]), out_size=(W, H))
        assert torch.equal(again, out), key                    # a resize to the same size is the identity


def test_draw_pose_frames_equal_the_vid2vid_chain(cuda_dev, gold, vis):
    """vid2vid: draw at the source size, cv2.resize to 512 x 512 — 2 launches, no frame at the source size allocated."""
    from aniportrait_b200 import ops
    for name in gold["chain_names"]:
        key = f"chain_{name}"
        W, H = (int(v) for v in gold[f"{key}_size"])
        normed = bool(gold[f"{key}_normed"])
        kp = torch.from_numpy(gold[f"{key}_keypoints"][None]).to(cuda_dev)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = ops.KERNEL_LAUNCHES
        out = vis.draw_pose_frames((W, H), kp, normed=normed, out_size=(512, 512))
        torch.cuda.synchronize()
        assert ops.KERNEL_LAUNCHES - n0 == 2
        assert torch.cuda.max_memory_allocated() - base < W * H * 3, f"{key}: a frame at the source size was allocated"
        assert torch.equal(out[0].cpu(), torch.from_numpy(gold[f"{key}_frame"])), key
        source = vis.draw_pose_frames((W, H), kp, normed=normed)
        assert source.shape == (1, H, W, 3) and _sha(source[0]) == str(gold[f"{key}_source_sha256"]), key


def test_draw_pose_frames_over_several_chunks(cuda_dev, gold, vis):
    """300 frames: ceil(300 / POSE_CHUNK) chunks of one draw and one resize launch each; the same bytes as one draw of
    every frame followed by one resize, and frame 0 and the last frame equal the restatement."""
    from aniportrait_b200 import ops
    from aniportrait_b200.pipelines import landmarks as LM
    rng = np.random.default_rng(7)
    key = "chain_" + next(n for n in gold["chain_names"] if n.startswith("1080x1920_b"))
    L = 300
    kp = gold[f"{key}_keypoints"][None] + rng.normal(0, 4.0, (L, 1, 2)) + rng.normal(0, 0.8, (L, 468, 2))
    dev = torch.from_numpy(kp).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    out = vis.draw_pose_frames((1080, 1920), dev, out_size=(512, 512))
    chunks = -(-L // LM.POSE_CHUNK)
    assert chunks > 1 and ops.KERNEL_LAUNCHES - n0 == 2 * chunks
    canvas = ops.draw_landmarks(dev, 1080.0, 1920.0, False, gold["edges"], gold["colors"])
    assert torch.equal(out, ops.resize_linear_u8(canvas, (512, 512), mid=(1080, 1920)))
    for i in (0, L - 1):
        want = RR.resize(RR.resize(LR.draw_frame(kp[i], gold["edges"], gold["colors"], image_size=(1080, 1920)),
                                   (1080, 1920)), (512, 512))
        assert np.array_equal(out[i].cpu().numpy(), want), i
    n0 = ops.KERNEL_LAUNCHES
    plain = vis.draw_pose_frames((512, 512), dev[:5])        # no resize at all: one draw launch
    assert ops.KERNEL_LAUNCHES - n0 == 1 and torch.equal(plain, vis.draw_landmarks_batch((512, 512), dev[:5]))


def test_bad_sizes_and_dtypes_raise_before_any_launch(cuda_dev, gold, vis):
    from aniportrait_b200 import _lib, ops
    from aniportrait_b200.pipelines import landmarks as LM
    frames = torch.zeros(2, 16, 24, 3, dtype=torch.uint8, device=cuda_dev)
    kp = torch.from_numpy(gold[f"one_{gold['one_names'][0]}_keypoints"][None]).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    for size in [(0, 8), (8, 0), (8193, 8), (8, 8193), (-4, 8), (8, 8, 8)]:
        with pytest.raises(ValueError):
            LM.resize_frames(frames, size)
        with pytest.raises(ValueError):
            vis.draw_pose_frames((512, 512), kp, out_size=size)
        with pytest.raises(ValueError):
            vis.draw_pose_frames(size, kp, out_size=(512, 512))
        with pytest.raises(ValueError):
            ops.resize_linear_u8(frames, (8, 8), mid=size)
    with pytest.raises(TypeError):
        LM.resize_frames(frames.float(), (8, 8))
    with pytest.raises(TypeError):
        LM.resize_frames(frames.cpu(), (8, 8))
    with pytest.raises(ValueError):
        LM.resize_frames(frames[..., :2], (8, 8))
    with pytest.raises(ValueError):
        LM.resize_frames(frames[0], (8, 8))
    with pytest.raises(ValueError):
        vis.draw_pose_frames((768, 768), kp[:, :100])                 # edge indices beyond N
    # the C ABI refuses what the wrappers would have caught
    out = torch.empty(2, 8, 8, 3, dtype=torch.uint8, device=cuda_dev)
    lib, I, p = _lib.lib(), _lib.I, _lib.ptr
    for args in [(2, 24, 16, 0, 0, 8, 8193), (2, 0, 16, 0, 0, 8, 8), (2, 24, 16, 5, 0, 8, 8), (2, 24, 16, 0, 9000, 8, 8),
                 (0, 24, 16, 0, 0, 8, 8)]:
        rc = lib.ap_resize_linear_u8(p(frames), *(I(v) for v in args), p(out), _lib.stream_ptr())
        assert rc != 0 and b"resize_linear_u8" in lib.ap_last_error()
    with pytest.raises(_lib.ApError):
        ops.resize_linear_u8(frames[:0], (8, 8))
    torch.cuda.synchronize()
    assert ops.KERNEL_LAUNCHES == n0


def test_pipeline_takes_resized_frames_at_a_non_square_size(cuda_dev, gold, vis):
    """_pose_maps_to_tensor on the device frames of draw_pose_frames equals it on the same frames as numpy arrays, at
    512 x 768 (width x height)."""
    from aniportrait_b200.pipelines.pipeline_pose2vid_long import Pose2VideoPipeline
    W, H = 512, 768
    keys = [f"one_{n}" for n in gold["one_names"]
            if tuple(gold[f"one_{n}_size"]) == (W, H) and not gold[f"one_{n}_normed"]]
    kp = torch.from_numpy(np.stack([gold[f"{k}_keypoints"] for k in keys])).to(cuda_dev)
    frames = vis.draw_pose_frames((W, H), kp)
    assert frames.shape == (len(keys), H, W, 3)
    pipe = Pose2VideoPipeline.__new__(Pose2VideoPipeline)
    dev = pipe._pose_maps_to_tensor(frames, H, W, cuda_dev)
    host = pipe._pose_maps_to_tensor(list(frames.cpu().numpy()), H, W, cuda_dev)
    assert dev.shape == (len(keys), 3, H, W) and dev.dtype == torch.float32
    assert torch.equal(dev, host)
