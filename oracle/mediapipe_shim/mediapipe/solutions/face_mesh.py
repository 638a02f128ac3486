"""mediapipe.solutions.face_mesh FACEMESH_* connection sets (frozensets of (start, end)), built from the connection lists
of the reference checkout's src/utils/face_landmark.py (FaceLandmarksConnections.FACE_LANDMARKS_*), parsed with ast."""
import ast
import os


def _connections():
    path = os.path.join(os.environ["ANIPORTRAIT_REFERENCE"], "src", "utils", "face_landmark.py")
    tree = ast.parse(open(path).read())
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.AnnAssign) and isinstance(node.target, ast.Name) and isinstance(node.value, ast.List):
            name = node.target.id
            if name.startswith("FACE_LANDMARKS_"):
                out[name[len("FACE_LANDMARKS_"):]] = frozenset(
                    (int(c.args[0].value), int(c.args[1].value)) for c in node.value.elts)
    return out


_C = _connections()
FACEMESH_LIPS = _C["LIPS"]
FACEMESH_LEFT_EYE = _C["LEFT_EYE"]
FACEMESH_LEFT_EYEBROW = _C["LEFT_EYEBROW"]
FACEMESH_LEFT_IRIS = _C["LEFT_IRIS"]
FACEMESH_RIGHT_EYE = _C["RIGHT_EYE"]
FACEMESH_RIGHT_EYEBROW = _C["RIGHT_EYEBROW"]
FACEMESH_RIGHT_IRIS = _C["RIGHT_IRIS"]
FACEMESH_FACE_OVAL = _C["FACE_OVAL"]
FACEMESH_TESSELATION = _C["TESSELATION"]
