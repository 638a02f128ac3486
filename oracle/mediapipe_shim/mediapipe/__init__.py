"""TEST INFRASTRUCTURE — a restatement of the mediapipe 0.10.11 names the reference's src/utils/draw_util.py imports
(solutions.drawing_utils.draw_landmarks, solutions.drawing_styles.DrawingSpec, solutions.face_mesh.FACEMESH_*,
framework.formats.landmark_pb2.NormalizedLandmarkList), so that the UNMODIFIED FaceMeshVisualizer runs on real cv2 when
oracle/make_golden_landmarks.py writes tests/golden/landmark_frames_reference.npz. Never imported by the product."""
from . import framework, solutions  # noqa: F401
