"""The cv2 INTER_LINEAR restatement (tests/resize_reference.py) against cv2.resize itself where cv2 imports, and, with the
landmark restatement, against the frames of the UNMODIFIED reference FaceMeshVisualizer at sizes other than 512 x 512 and
through vid2vid's two resizes (tests/golden/landmark_frames_resized_reference.npz, oracle/make_golden_landmarks_resized.py);
the host side of draw_pose_frames (which resizes it launches)."""
import hashlib
import os

import numpy as np
import pytest

import landmark_reference as LR
import resize_reference as RR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "landmark_frames_resized_reference.npz")

# (w, h) -> (W, H): the canvas to every size the scripts draw at, those sizes back to 512 x 512 (vid2vid), odd sizes
SIZES = [((512, 512), s) for s in [(1080, 1920), (1920, 1080), (768, 768), (720, 1280), (1024, 1024), (513, 511),
                                   (600, 900), (3840, 2160), (576, 1024), (256, 256), (300, 200), (512, 768),
                                   (768, 512)]] \
    + [(s, (512, 512)) for s in [(1080, 1920), (1920, 1080), (720, 1280), (1000, 700), (1024, 1024)]]
# degenerate and exact-ratio cases: 1 x 1, 1 x N, N x 1, exact 2x down (cv2's INTER_AREA path) and up, the identity
SMALL = [((1, 1), (7, 5)), ((5, 7), (1, 1)), ((1, 1), (1, 1)), ((1, 9), (4, 13)), ((9, 1), (13, 4)), ((7, 3), (1, 17)),
         ((1, 40), (1, 3)), ((40, 1), (3, 1)), ((100, 60), (50, 30)), ((64, 64), (128, 128)), ((101, 61), (50, 30)),
         ((37, 23), (37, 23)), ((333, 17), (5, 1000))]


def _image(rng, w, h):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("src,dst", SIZES + SMALL)
def test_restatement_equals_cv2_resize(src, dst):
    cv2 = pytest.importorskip("cv2")
    img = _image(np.random.default_rng(src[0] * 7 + dst[1]), *src)
    want = cv2.resize(img, dst)
    got = RR.resize(img, dst)
    assert got.shape == want.shape == (dst[1], dst[0], 3)
    assert int((got != want).sum()) == 0


def test_restatement_equals_cv2_resize_at_seeded_sizes():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(41)
    for _ in range(300):
        w, h, W, H = (int(v) for v in rng.integers(1, 260, 4))
        img = _image(rng, w, h)
        assert np.array_equal(RR.resize(img, (W, H)), cv2.resize(img, (W, H))), ((w, h), (W, H))


def test_exact_2x_downscale_is_the_area_average():
    """cv2 switches to INTER_AREA here; the linear formula gives (a + b + c + d + 2) >> 2 with every coefficient 1024."""
    img = _image(np.random.default_rng(5), 64, 48).astype(np.int64)
    quad = img[0::2, 0::2] + img[0::2, 1::2] + img[1::2, 0::2] + img[1::2, 1::2]
    assert np.array_equal(RR.resize(img.astype(np.uint8), (32, 24)), ((quad + 2) >> 2).astype(np.uint8))


def test_restatement_reproduces_the_golden_frames(gold):
    """Each golden frame is the reference's draw_landmarks at `size` (its 512 x 512 canvas, then cv2.resize) — for
    vid2vid, resized once more to 512 x 512. The restated canvas and restated resizes give the same bytes."""
    edges, colors = gold["edges"], gold["colors"]
    for kind in ("one", "chain"):
        for name in gold[f"{kind}_names"]:
            key = f"{kind}_{name}"
            size = tuple(int(v) for v in gold[f"{key}_size"])
            canvas = LR.draw_frame(gold[f"{key}_keypoints"], edges, colors, image_size=size,
                                   normed=bool(gold[f"{key}_normed"]))
            frame = RR.resize(canvas, size)
            assert frame.shape == (size[1], size[0], 3)
            if kind == "chain":
                assert hashlib.sha256(frame.tobytes()).hexdigest() == str(gold[f"{key}_source_sha256"]), key
                frame = RR.resize(frame, (512, 512))
            if f"{key}_frame" in gold:
                assert gold[f"{key}_frame"].any(axis=2).sum() > 500, f"{key}: nearly blank golden frame"
                assert np.array_equal(frame, gold[f"{key}_frame"]), key
            else:
                assert hashlib.sha256(frame.tobytes()).hexdigest() == str(gold[f"{key}_sha256"]), key


def test_golden_covers_the_script_sizes(gold):
    assert str(gold["cv2_version"]).startswith("4.")
    one = {tuple(int(v) for v in gold[f"one_{n}_size"]) for n in gold["one_names"]}
    assert one >= {(768, 768), (512, 768), (768, 512), (1080, 1920), (1920, 1080), (720, 1280), (1024, 1024)}
    chain = {tuple(int(v) for v in gold[f"chain_{n}_size"]) for n in gold["chain_names"]}
    assert (1024, 1024) in chain and len(chain) >= 4        # 1024 -> 512 is cv2's exact 2x (INTER_AREA) case
    assert os.path.getsize(GOLDEN) < 1_000_000


def test_pose_stages_drop_resizes_to_the_same_size():
    from aniportrait_b200.pipelines.landmarks import _pose_stages
    assert _pose_stages((512, 512), None) == []
    assert _pose_stages((512, 512), (512, 512)) == []
    assert _pose_stages((768, 512), None) == [(768, 512)]
    assert _pose_stages((768, 512), (768, 512)) == [(768, 512)]
    assert _pose_stages((512, 512), (768, 768)) == [(768, 768)]
    assert _pose_stages((1080, 1920), (512, 512)) == [(1080, 1920), (512, 512)]
    for image_size, out_size in [((0, 512), None), ((512, 8193), None), ((512, 512), (-1, 4)), ((512, 512, 3), None),
                                 ((512, 512), (512,))]:
        with pytest.raises(ValueError):
            _pose_stages(image_size, out_size)


def test_resize_frames_refuses_host_and_non_uint8_frames():
    import torch
    from aniportrait_b200.pipelines import landmarks as LM
    with pytest.raises(TypeError):
        LM.resize_frames(torch.zeros(1, 4, 4, 3, dtype=torch.uint8), (8, 8))
    with pytest.raises(TypeError):
        LM.resize_frames(np.zeros((1, 4, 4, 3), np.uint8), (8, 8))
