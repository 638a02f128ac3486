"""Pillow's bilinear resize (ap_resize_pil_bilinear_u8) and the comparison grid (ap_video_grid_u8) on the device against
the numpy restatements (tests/pil_resize_reference.py) on seeded frames, and against the frames of the UNMODIFIED
reference save_videos_grid on script-shaped cases (tests/golden/video_grid_reference.npz); launch counts, memory, the
refusals, and the pipeline's output_type="cuda"."""
import os

import numpy as np
import pytest
import torch

import pil_resize_reference as PR
import video_grid_cases as VC
from test_pil_resize_cpu import SIZES

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_grid_reference.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def _frames(seed, L, w, h):
    return np.random.default_rng(seed).integers(0, 256, (L, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("src,dst", SIZES)
def test_resize_equals_the_restatement(cuda_dev, src, dst):
    from aniportrait_b200 import ops
    L = 1 if max(src) >= 4096 else 3
    frames = _frames(src[0] * 131 + dst[1], L, *src)
    n0 = ops.KERNEL_LAUNCHES
    out = ops.resize_pil_bilinear_u8(torch.from_numpy(frames).to(cuda_dev), dst)
    assert ops.KERNEL_LAUNCHES - n0 == (0 if src == dst else 1)
    assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (L, dst[1], dst[0], 3)
    want = PR.resize_frames(frames, dst)
    bad = int((out.cpu().numpy() != want).sum())
    assert bad == 0, f"{bad} bytes differ"


def _device_grid(case, dev, host_lists=True):
    """The case through pose_transform_frames (host frames, as the scripts hold them) and one grid_frames call."""
    from aniportrait_b200 import ops
    from aniportrait_b200.pipelines import video_grid as VG
    n_rows, (height, width), tiles = case
    parts, bgr, resizes = [], [], 0
    for kind, data, flag in tiles:
        if kind == "video":
            parts.append(torch.from_numpy(data).to(dev))
        else:
            n0 = ops.KERNEL_LAUNCHES
            parts.append(VG.pose_transform_frames(list(data) if host_lists else data, (height, width)))
            resizes += ops.KERNEL_LAUNCHES - n0
        bgr.append(flag)
    n0 = ops.KERNEL_LAUNCHES
    out = VG.grid_frames(parts, n_rows, bgr=bgr)
    assert ops.KERNEL_LAUNCHES - n0 == 1
    return out, parts, resizes


def test_grid_equals_the_reference_goldens(cuda_dev, gold):
    """Every script-shaped case: the frames of the reference's save_videos_grid, byte for byte, and the restatements."""
    for name, case in VC.cases().items():
        assert VC.input_digest(case[2]) == str(gold[f"{name}_input_sha256"]), name
        out, _, _ = _device_grid(case, cuda_dev, host_lists=name.startswith(("audio", "pose")))
        got = out.cpu().numpy()
        assert got.shape == tuple(gold[f"{name}_shape"]), name
        if f"{name}_frames" in gold:
            assert np.array_equal(got, gold[f"{name}_frames"]), name
        else:
            assert VC.frames_digest(got) == str(gold[f"{name}_sha256"]), name
        if max(got.shape[1:3]) <= 600:
            assert np.array_equal(got, VC.restated_grid(case)), name


@pytest.mark.parametrize("n_rows", [1, 2, 3, 6])
@pytest.mark.parametrize("B", range(1, 8))
def test_grid_equals_the_numpy_composition(cuda_dev, B, n_rows):
    """Mixed tiles: uint8 frames (one broadcast, one longer than T, BGR), fp16 and fp32 videos with strided layouts."""
    from aniportrait_b200 import ops
    rng = np.random.default_rng(100 * B + n_rows)
    T, H, W = 3, 9, 13
    tiles, want, bgr = [], [], []
    for i in range(B):
        kind = i % 4
        if kind == 0:                                                   # one frame, repeated over T
            f = rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8)
            tiles.append(torch.from_numpy(f).to(cuda_dev))
            want.append(np.repeat(f, T, 0))
            bgr.append(False)
        elif kind == 1:                                                 # longer than T, BGR
            f = rng.integers(0, 256, (T + 2, H, W, 3), dtype=np.uint8)
            tiles.append(torch.from_numpy(f).to(cuda_dev))
            want.append(f[:T, :, :, ::-1])
            bgr.append(True)
        elif kind == 2:                                                 # fp16 frames [T, 3, H, W] viewed as a video
            v = torch.from_numpy(rng.random((T, 3, H, W), dtype=np.float32)).half()
            tiles.append(v.to(cuda_dev).permute(1, 0, 2, 3).unsqueeze(0))
            want.append(PR.video_bytes(v.float().numpy()).transpose(0, 2, 3, 1))
            bgr.append(False)
        else:                                                           # fp32, a column-strided view of a wider video
            v = rng.random((1, 3, T, H, 2 * W), dtype=np.float32)
            tiles.append(torch.from_numpy(v).to(cuda_dev)[..., ::2])
            want.append(PR.video_bytes(v[0, :, :, :, ::2]).transpose(1, 2, 3, 0))
            bgr.append(False)
    n0 = ops.KERNEL_LAUNCHES
    out = ops.video_grid_u8(tiles, n_rows, T, bgr=bgr)
    assert ops.KERNEL_LAUNCHES - n0 == 1
    assert np.array_equal(out.cpu().numpy(), PR.compose_grid(want, n_rows))


def test_grid_writes_into_a_given_buffer_and_unaligned_widths(cuda_dev):
    """out= is reused with no allocation; a grid width that is not a multiple of 4 takes the byte-store path."""
    from aniportrait_b200.pipelines import video_grid as VG
    rng = np.random.default_rng(3)
    for W in (13, 14, 15, 16):
        v = rng.random((1, 3, 2, 7, W), dtype=np.float32)
        f = rng.integers(0, 256, (1, 7, W, 3), dtype=np.uint8)
        tiles = [torch.from_numpy(f).to(cuda_dev), torch.from_numpy(v).to(cuda_dev)]
        want = PR.compose_grid([np.repeat(f, 2, 0), PR.video_bytes(v[0]).transpose(1, 2, 3, 0)], 3)
        buf = torch.full(want.shape, 77, dtype=torch.uint8, device=cuda_dev)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = VG.grid_frames(tiles, 3, out=buf)
        assert out.data_ptr() == buf.data_ptr() and torch.cuda.max_memory_allocated() == base
        assert np.array_equal(buf.cpu().numpy(), want), W


def test_pose_transform_frames_launches(cuda_dev):
    """One resize launch per upload chunk for host frames, one for a CUDA tensor, none for a matching size."""
    from aniportrait_b200 import ops
    from aniportrait_b200.pipelines import video_grid as VG
    frames = _frames(11, 12, 96, 64)
    old = VG.UPLOAD_CHUNK_BYTES
    try:
        VG.UPLOAD_CHUNK_BYTES = 5 * 96 * 64 * 3                          # 5 frames per chunk -> 3 chunks
        n0 = ops.KERNEL_LAUNCHES
        out = VG.pose_transform_frames(list(frames), (40, 56))
        assert ops.KERNEL_LAUNCHES - n0 == 3
        assert np.array_equal(out.cpu().numpy(), PR.resize_frames(frames, (56, 40)))
        n0 = ops.KERNEL_LAUNCHES
        same = VG.pose_transform_frames(frames, (64, 96))                # uint8 array at the size: the upload only
        assert ops.KERNEL_LAUNCHES == n0 and np.array_equal(same.cpu().numpy(), frames)
    finally:
        VG.UPLOAD_CHUNK_BYTES = old
    dev = torch.from_numpy(frames).to(cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    assert VG.pose_transform_frames(dev, (64, 96)) is dev
    assert ops.KERNEL_LAUNCHES == n0
    out = VG.pose_transform_frames(dev, (40, 56))
    assert ops.KERNEL_LAUNCHES - n0 == 1 and np.array_equal(out.cpu().numpy(), PR.resize_frames(frames, (56, 40)))


def test_pose_transform_frames_memory_does_not_grow_with_L(cuda_dev):
    """300 source frames of 1080 x 1920 to 512 x 512: beyond the output, the device holds at most one upload chunk
    (UPLOAD_CHUNK_BYTES, 64 MiB) plus 1 MiB, whatever L is. Frame 0 and the last frame equal the restatement."""
    from aniportrait_b200.pipelines import video_grid as VG
    L, h, w = 300, 1920, 1080
    base_frame = _frames(5, 1, w, h)[0]
    frames = [np.roll(base_frame, i, axis=1) for i in range(L)]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = VG.pose_transform_frames(frames, (512, 512))
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - out.numel()
    assert extra <= VG.UPLOAD_CHUNK_BYTES + (1 << 20), extra
    for i in (0, L - 1):
        assert np.array_equal(out[i].cpu().numpy(), PR.resize(frames[i], (512, 512))), i


def test_refused_inputs_raise_before_any_launch(cuda_dev):
    from aniportrait_b200 import _lib, ops
    from aniportrait_b200.pipelines import video_grid as VG
    u8 = torch.zeros(3, 8, 10, 3, dtype=torch.uint8, device=cuda_dev)
    vid = torch.zeros(1, 3, 3, 8, 10, dtype=torch.float16, device=cuda_dev)
    n0 = ops.KERNEL_LAUNCHES
    with pytest.raises(ValueError):                                  # tile sizes differ
        VG.grid_frames([u8, torch.zeros(1, 3, 3, 8, 11, dtype=torch.float16, device=cuda_dev)], 3)
    with pytest.raises(ValueError):                                  # a uint8 tile with 1 < T' < T
        VG.grid_frames([u8[:2], vid], 3)
    with pytest.raises(ValueError):                                  # a video shorter than `frames`
        VG.grid_frames([u8, vid], 3, frames=4)
    with pytest.raises(TypeError):                                   # host tensor
        VG.grid_frames([u8.cpu(), vid], 3)
    with pytest.raises(TypeError):                                   # dtype
        VG.grid_frames([u8.short(), vid], 3)
    with pytest.raises(TypeError):
        VG.grid_frames([u8, vid.double()], 3)
    with pytest.raises(ValueError):                                  # bgr on a video tile
        VG.grid_frames([u8, vid], 3, bgr=[False, True])
    with pytest.raises(ValueError):                                  # no video tile, no frames
        VG.grid_frames([u8], 3)
    with pytest.raises(ValueError):                                  # out of the wrong shape
        VG.grid_frames([u8, vid], 3, out=torch.empty(3, 12, 27, 3, dtype=torch.uint8, device=cuda_dev))
    with pytest.raises(ValueError):
        VG.grid_frames([vid] * 17, 3)
    for size in [(0, 8), (8, 8193), (8, 8, 8)]:
        with pytest.raises(ValueError):
            VG.pose_transform_frames(u8, size)
    with pytest.raises(ValueError):                                  # 33x on an axis
        ops.resize_pil_bilinear_u8(torch.zeros(1, 66, 4, 3, dtype=torch.uint8, device=cuda_dev), (4, 2))
    with pytest.raises(ValueError):
        VG.pose_transform_frames(u8[..., :2], (4, 4))
    # the C ABI refuses what the wrappers would have caught
    out = torch.empty(1, 8, 8, 3, dtype=torch.uint8, device=cuda_dev)
    lib, I, p = _lib.lib(), _lib.I, _lib.ptr
    for args in [(1, 10, 8, 8, 8193), (1, 0, 8, 8, 8), (0, 10, 8, 8, 8), (1, 66, 8, 2, 8), (1, 10, 8193, 8, 8)]:
        rc = lib.ap_resize_pil_bilinear_u8(p(u8), *(I(v) for v in args), p(out), _lib.stream_ptr())
        assert rc != 0 and b"resize_pil_bilinear_u8" in lib.ap_last_error()
    tiles = (_lib.GridTile * 1)(_lib.GridTile(u8.data_ptr(), 7, 0, 0, 30, 3, 1))
    assert lib.ap_video_grid_u8(tiles, I(1), I(1), I(1), I(8), I(10), p(out), _lib.stream_ptr()) != 0
    assert lib.ap_video_grid_u8(tiles, I(0), I(1), I(1), I(8), I(10), p(out), _lib.stream_ptr()) != 0
    torch.cuda.synchronize()
    assert ops.KERNEL_LAUNCHES == n0


def test_pipeline_cuda_output_and_its_grid(cuda_dev):
    """output_type="cuda" is the fp16 video whose fp32 widening is output_type="tensor"; the device grid built from it
    equals the scripts' host tail (pose_transform, torch.cat, save_videos_grid's make_grid and uint8 cast) on that tensor."""
    import torchvision
    from PIL import Image
    from torchvision import transforms
    from helpers import build_pipeline, pipeline_inputs
    from aniportrait_b200.pipelines import video_grid as VG
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pipeline_small.pt"))
    P = dict(gold["params"])
    S = P["size"]
    pipe = build_pipeline(P, cuda_dev)
    ref_image, poses, ref_pose = pipeline_inputs(S, 4, P["seeds"]["inputs"])
    host = pipe(ref_image, poses, ref_pose, S, S, 4, 2, 1.0, generator=torch.manual_seed(1)).videos
    dev = pipe(ref_image, poses, ref_pose, S, S, 4, 2, 1.0, generator=torch.manual_seed(1), output_type="cuda").videos
    assert dev.is_cuda and dev.dtype == torch.float16 and dev.shape == host.shape
    assert torch.equal(dev.float().cpu(), host)
    # the scripts' tail on the host tensor
    pose_transform = transforms.Compose([transforms.Resize((S, S)), transforms.ToTensor()])
    ref_t = pose_transform(ref_image).unsqueeze(1).unsqueeze(0).repeat(1, 1, 4, 1, 1)
    pose_t = torch.stack([pose_transform(Image.fromarray(np.asarray(p))) for p in poses], 0).transpose(0, 1)[None]
    x = torch.cat([ref_t, pose_t[:, :, :4], host], dim=0).permute(2, 0, 1, 3, 4)
    want = np.stack([(torchvision.utils.make_grid(f, nrow=3) * 255).numpy().astype(np.uint8).transpose(1, 2, 0)
                     for f in x])
    ref_u8 = VG.pose_transform_frames([ref_image], (S, S))
    pose_u8 = VG.pose_transform_frames([np.asarray(p) for p in poses], (S, S))
    got = VG.grid_frames([ref_u8, pose_u8, dev], n_rows=3)
    assert np.array_equal(got.cpu().numpy(), want)
