"""The Pillow BILINEAR restatement (tests/pil_resize_reference.py) against PIL.Image.resize itself, the ToTensor / x255
round trip of every byte through real torchvision, the numpy grid composition against torchvision.utils.make_grid, and the
restatements together against the frames of the UNMODIFIED reference save_videos_grid
(tests/golden/video_grid_reference.npz, oracle/make_golden_video_grid.py); the host-side refusals of video_grid."""
import os

import numpy as np
import pytest
import torch

import pil_resize_reference as PR
import video_grid_cases as VC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_grid_reference.npz")

# (w, h) -> (W, H): the scripts' frames to their output sizes (vid2vid's sources, audio2vid / pose2vid's frames)
SCRIPT = [((1920, 1080), (512, 512)), ((1080, 1920), (512, 512)), ((640, 480), (512, 512)), ((1000, 700), (512, 512)),
          ((720, 1280), (512, 512)), ((512, 512), (768, 768)), ((300, 200), (512, 768)), ((480, 640), (512, 512))]
# odd and degenerate sizes: 1 x 1, 1 x N, N x 1, prime sides, the identity
ODD = [((1, 1), (1, 1)), ((1, 1), (9, 4)), ((5, 7), (1, 1)), ((1, 40), (1, 3)), ((40, 1), (3, 1)), ((7, 1), (1, 3)),
       ((1, 9), (4, 13)), ((37, 23), (5, 301)), ((513, 511), (512, 512)), ((101, 61), (53, 29)), ((37, 23), (37, 23)),
       ((97, 89), (131, 113))]
# one axis only: Pillow runs one pass
ONE_AXIS = [((64, 48), (64, 31)), ((64, 48), (29, 48)), ((1, 200), (1, 7)), ((200, 1), (7, 1)), ((96, 96), (96, 512))]
# an 8x downscale (4096-pixel photo to 512), and the largest supported 32x per axis
SCALE = [((4096, 4096), (512, 512)), ((2048, 64), (64, 2)), ((8192, 32), (256, 1)), ((64, 8192), (2, 256))]
SIZES = SCRIPT + ODD + ONE_AXIS + SCALE


def _image(rng, w, h):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _pil_resize(img, size):
    """Image.fromarray(img).resize(size, Image.BILINEAR), one call of Pillow's C resampler as Pillow 9.5.0 (the version
    the reference pins) makes it. Newer Pillow splits a resize of an image more than 100 times taller than wide into a
    vertical resize followed by a horizontal one; that order rounds differently, and no script frame has that shape, so
    the C resampler is called directly there."""
    from PIL import Image
    im = Image.fromarray(img)
    h, w = img.shape[:2]
    if h > 100 * w and size[1] < h:
        return np.asarray(im._new(im.im.resize(tuple(size), Image.BILINEAR, (0, 0, w, h))))
    return np.asarray(im.resize(tuple(size), Image.BILINEAR))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("src,dst", SIZES)
def test_restatement_equals_pil_resize(src, dst):
    img = _image(np.random.default_rng(src[0] * 7 + dst[1]), *src)
    want = _pil_resize(img, dst)
    got = PR.resize(img, dst)
    assert got.shape == want.shape == (dst[1], dst[0], 3)
    assert int((got != want).sum()) == 0


def test_restatement_equals_pil_resize_at_seeded_sizes():
    rng = np.random.default_rng(43)
    for _ in range(200):
        w, h, W, H = (int(v) for v in rng.integers(1, 200, 4))
        img = _image(rng, w, h)
        want = _pil_resize(img, (W, H))
        assert np.array_equal(PR.resize(img, (W, H)), want), ((w, h), (W, H))


def test_largest_scale_needs_65_taps():
    """ksize = 2 ceil(in / out) + 1 bounds the taps: 9 for 1920 -> 512, 17 for 8x, 65 for the largest scale, 32x."""
    for n_in, n_out, ksize in [(1920, 512, 9), (4096, 512, 17), (8192, 256, 65), (64, 2, 65)]:
        _, taps, k = PR.coeffs(n_in, n_out)
        assert k.shape[1] == ksize and 0 < taps.min() and taps.max() <= ksize


def test_to_tensor_times_255_gives_every_byte_back():
    """ToTensor then save_videos_grid's `(x * 255).numpy().astype(np.uint8)`: trunc(fl(fl(v / 255) * 255)) = v for all
    256 values, so uint8 tiles pass through the grid unchanged."""
    from PIL import Image
    from torchvision import transforms
    v = np.arange(256, dtype=np.uint8)
    img = np.stack([v, v[::-1], np.roll(v, 7)], -1).reshape(16, 16, 3)
    x = transforms.ToTensor()(Image.fromarray(img))
    assert x.dtype == torch.float32
    back = (x * 255).numpy().astype(np.uint8).transpose(1, 2, 0)
    assert np.array_equal(back, img)
    assert np.array_equal(PR.to_tensor_bytes(img), img)


@pytest.mark.parametrize("n_rows", [1, 2, 3, 6])
@pytest.mark.parametrize("B", range(1, 8))
def test_compose_grid_equals_make_grid(B, n_rows):
    import torchvision
    rng = np.random.default_rng(B * 10 + n_rows)
    H, W = 5, 7
    tiles = [rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8) for _ in range(B)]
    x = torch.from_numpy(np.concatenate(tiles)).permute(0, 3, 1, 2).float() / 255
    want = (torchvision.utils.make_grid(x, nrow=n_rows) * 255).numpy().astype(np.uint8).transpose(1, 2, 0)
    got = PR.compose_grid(tiles, n_rows)[0]
    assert got.shape == want.shape and got.shape[:2] == PR.grid_geometry(B, n_rows, H, W)[2:]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("B,n_rows,shape", [(3, 3, (68, 296)), (1, 1, (64, 96)), (2, 3, (68, 198)), (4, 3, (134, 296)),
                                            (3, 1, (200, 100))])
def test_grid_shapes(B, n_rows, shape):
    from aniportrait_b200 import ops
    assert PR.grid_geometry(B, n_rows, 64, 96)[2:] == shape
    assert ops.grid_shape(B, n_rows, 64, 96) == shape


def test_restatements_reproduce_the_golden_grids(gold):
    """Pillow's resize, the byte round trip, the BGR swap, the repeat and cut to T and make_grid, all restated, give the
    frames the reference's save_videos_grid produced on every script-shaped case."""
    cases = VC.cases()
    assert set(str(n) for n in gold["names"]) == set(cases)
    for name, case in cases.items():
        assert VC.input_digest(case[2]) == str(gold[f"{name}_input_sha256"]), f"{name}: the seeded inputs changed"
        frames = VC.restated_grid(case)
        assert tuple(frames.shape) == tuple(gold[f"{name}_shape"]), name
        if f"{name}_frames" in gold:
            assert np.array_equal(frames, gold[f"{name}_frames"]), name
        else:
            assert VC.frames_digest(frames) == str(gold[f"{name}_sha256"]), name


def test_golden_records_versions_and_size(gold):
    assert str(gold["pillow_version"]) and str(gold["torchvision_version"])
    assert {int(gold[f"{n}_n_rows"]) for n in gold["names"]} == {1, 3}
    assert os.path.getsize(GOLDEN) < 1_000_000


def test_video_grid_refuses_host_input_before_anything():
    from aniportrait_b200.pipelines import video_grid as VG
    with pytest.raises(TypeError):
        VG.grid_frames([torch.zeros(1, 3, 2, 4, 4)], n_rows=1)
    with pytest.raises(TypeError):
        VG.pose_transform_frames(torch.zeros(1, 4, 4, 3, dtype=torch.uint8), (8, 8))
    with pytest.raises(TypeError):
        VG.pose_transform_frames([np.zeros((4, 4, 3), np.float32)], (8, 8))
    with pytest.raises(ValueError):
        VG.pose_transform_frames([np.zeros((4, 4, 3), np.uint8), np.zeros((4, 5, 3), np.uint8)], (8, 8))
    for size in [(0, 8), (8, 8193), (8, 8, 8)]:
        with pytest.raises(ValueError):
            VG.pose_transform_frames([np.zeros((4, 4, 3), np.uint8)], size)
    with pytest.raises(ValueError):                                   # 33x on the width
        VG.pose_transform_frames([np.zeros((4, 66, 3), np.uint8)], (4, 2))
