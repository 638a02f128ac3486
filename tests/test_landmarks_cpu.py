"""Landmark pose frames and face-mesh projection, host side: the integer restatement of the rasteriser
(tests/landmark_reference.py) against the golden frames of the UNMODIFIED reference FaceMeshVisualizer
(tests/golden/landmark_frames_reference.npz, oracle/make_golden_landmarks.py) and against cv2 itself where it imports;
the host half of the projection (matrices, smoothing) against the golden and scipy; the edge table read from a
visualizer."""
import os
from collections import namedtuple

import numpy as np
import pytest

import landmark_reference as LR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "landmark_frames_reference.npz")
Spec = namedtuple("Spec", "color thickness circle_radius")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def test_restatement_equals_the_reference_frames(gold):
    for i, name in enumerate(gold["case_names"]):
        s = int(gold["case_spec"][i])
        img = LR.draw_frame(gold["case_keypoints"][i], gold[f"spec{s}_edges"], gold[f"spec{s}_colors"],
                            normed=bool(gold["case_normed"][i]))
        assert np.array_equal(img, gold["case_frames"][i]), name


def test_restatement_equals_cv2_line_on_seeded_segments():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    color = np.array([7, 130, 250], np.uint8)
    n = 20000
    for t in range(n):
        W = 512 if t % 8 == 0 else 64
        kind = t % 6
        a = rng.integers(0, W, 2)
        if kind == 0:                                   # short
            b = a + rng.integers(-3, 4, 2)
        elif kind == 1:                                 # long, any direction
            b = rng.integers(0, W, 2)
        elif kind == 2:                                 # axis-aligned
            b = a.copy()
            b[t % 2] = rng.integers(0, W)
        elif kind == 3:                                 # diagonal
            d = int(rng.integers(-W, W))
            b = a + np.array([d, d if t % 4 else -d])
        elif kind == 4:                                 # on the border
            a = np.array([0 if t % 3 else W - 1, rng.integers(0, W)])
            b = np.array([rng.integers(0, W), W - 1 if t % 5 else 0])
        else:                                           # zero length
            b = a.copy()
        b = np.clip(b, 0, W - 1)
        p0, p1 = (int(a[0]), int(a[1])), (int(b[0]), int(b[1]))
        ref = np.zeros((W, W, 3), np.uint8)
        cv2.line(ref, p0, p1, tuple(int(c) for c in color), 2)
        mine = np.zeros((W, W, 3), np.uint8)
        LR.thick_line2(mine, p0, p1, color)
        assert np.array_equal(ref, mine), (W, p0, p1)


def test_restatement_equals_the_shim_draw_landmarks(gold):
    pytest.importorskip("cv2")
    import sys
    shim = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "mediapipe_shim")
    sys.path.insert(0, shim)
    try:
        from mediapipe.solutions import drawing_utils
        from mediapipe.framework.formats import landmark_pb2
    finally:
        sys.path.remove(shim)
    rng = np.random.default_rng(12)
    for s in (0, 1):
        edges, colors = gold[f"spec{s}_edges"], gold[f"spec{s}_colors"]
        spec = {tuple(int(v) for v in e): Spec(tuple(int(v) for v in c), 2, 1) for e, c in zip(edges, colors)}
        for t in range(6):
            kp = rng.uniform(-0.05, 1.05, (468, 2)) * (1 if t % 2 else 512)
            image = np.zeros((512, 512, 3), np.uint8)
            lms = landmark_pb2.NormalizedLandmarkList()
            for x, y in kp:
                lm = lms.landmark.add()
                lm.x, lm.y = (x, y) if t % 2 else (x / 512, y / 512)
            drawing_utils.draw_landmarks(image=image, landmark_list=lms, connections=spec.keys(),
                                         landmark_drawing_spec=None, connection_drawing_spec=spec)
            assert np.array_equal(LR.draw_frame(kp, edges, colors, normed=bool(t % 2)), image), (s, t)


def test_landmark_conversion_edges():
    kp = np.array([[0.0, 0.0], [1.0, 1.0], [-1e-9, 0.5], [0.5, 1 + 1e-7], [1 + 1e-10, 0.5], [np.nan, 0.2],
                   [0.99999999, 0.0]])
    px, kept = LR.landmark_pixels(kp, (512, 512), normed=True)
    assert kept.tolist() == [True, True, False, False, True, False, True]
    assert px[0].tolist() == [0, 0] and px[1].tolist() == [511, 511] and px[4].tolist() == [511, 256]
    px, kept = LR.landmark_pixels(kp * 512, (512, 512), normed=False)
    assert kept.tolist() == [True, True, False, False, True, False, True]


def test_host_projection_matches_the_reference(gold):
    from aniportrait_b200.pipelines import landmarks as LM
    for e, m in zip(gold["euler"], gold["euler_mats"]):
        mine = LM.euler_and_translation_to_matrix(e, [1.0, 2.0, 3.0])
        assert np.abs(mine - m).max() <= 1e-12 * np.abs(m).max()
    mats = np.stack([gold["trans_mat"] @ LM.euler_and_translation_to_matrix(p[:3], p[3:]) for p in gold["pose_seq"]])
    P = LM.perspective_matrix(1.0)
    assert P.dtype == np.float64 and np.array_equal(P, P.astype(np.float32).astype(np.float64))
    pts = gold["offsets"].astype(np.float64) + gold["mesh_base"]
    got = LR.project_points(pts, mats, P, (512, 512))
    assert np.abs(got - gold["proj_a"]).max() <= 1e-12 * np.abs(gold["proj_a"]).max()
    got = LR.project_points(gold["vid_verts"], gold["vid_mats"], P, (512, 512))
    assert np.abs(got - gold["proj_b"]).max() <= 1e-12 * np.abs(gold["proj_b"]).max()


def test_host_matrices_match_scipy():
    Rotation = pytest.importorskip("scipy.spatial.transform").Rotation
    from aniportrait_b200.pipelines import landmarks as LM
    rng = np.random.default_rng(13)
    for e in rng.uniform(-180, 180, (200, 3)):
        ref = Rotation.from_euler("xyz", e, degrees=True).as_matrix()
        assert np.abs(LM.euler_and_translation_to_matrix(e, [0, 0, 0])[:3, :3] - ref).max() <= 1e-12


def test_smooth_pose_seq_matches_the_reference(gold):
    from aniportrait_b200.pipelines import landmarks as LM
    assert np.array_equal(LM.smooth_pose_seq(gold["pose_temp"], 7), gold["smooth_7"])
    assert np.array_equal(LM.smooth_pose_seq(gold["pose_temp"][:40], 3), gold["smooth_3"])


def test_edge_table_follows_dict_order_and_last_spec():
    from aniportrait_b200.pipelines import landmarks as LM
    spec = {}
    spec[(1, 2)] = Spec((1, 1, 1), 2, 1)
    spec[(3, 4)] = Spec((2, 2, 2), 2, 1)
    spec[(1, 2)] = Spec((9, 8, 7), 2, 1)          # re-inserted: keeps its first position, takes the last colour
    spec[(0, 5)] = Spec((3, 3, 3), 2, 1)
    edges, colors = LM.edge_table(spec)
    assert edges.tolist() == [[1, 2], [3, 4], [0, 5]] and edges.dtype == np.int32
    assert colors.tolist() == [[9, 8, 7], [2, 2, 2], [3, 3, 3]] and colors.dtype == np.uint8
    with pytest.raises(NotImplementedError):
        LM.edge_table({(0, 1): Spec((1, 1, 1), 3, 1)})
    with pytest.raises(NotImplementedError):
        LM.edge_table({(i, i + 1): Spec((1, 1, 1), 2, 1) for i in range(256)})


def test_golden_specs_are_the_visualizers_tables(gold):
    """114 edges without the forehead edge, 124 with it; every edge thickness 2."""
    assert len(gold["spec0_edges"]) == 114 and len(gold["spec1_edges"]) == 124
    assert (gold["spec0_thickness"] == 2).all() and (gold["spec1_thickness"] == 2).all()


def test_restatement_equals_the_reference_on_landmarker_output(gold):
    """The reference pose of audio2vid.py:153-155 / vid2vid.py:139-140: LMKExtractor's float32 [478, 3] landmarks (x, y, z),
    normed; only columns 0 and 1 are read."""
    lmks = gold["lmks478"]
    assert lmks.shape == (478, 3) and lmks.dtype == np.float32
    for s in (0, 1):
        img = LR.draw_frame(lmks, gold[f"spec{s}_edges"], gold[f"spec{s}_colors"], normed=True)
        assert np.array_equal(img, gold["lmks478_frames"][s]), s


def test_projection_with_base_refuses_offsets_that_are_not_fp32(gold):
    from aniportrait_b200.pipelines import landmarks as LM
    with pytest.raises(TypeError):
        LM.project_points(gold["offsets"].astype(np.float64), gold["trans_mat"], gold["pose_seq"], [512, 512],
                          base=gold["mesh_base"])
    with pytest.raises(TypeError):
        LM.project_points_with_trans(gold["vid_verts"], gold["vid_mats"], [512, 512], base=gold["mesh_base"])
