"""NormalizedLandmarkList with the protobuf `float` (float32) fields x, y, z; visibility / presence are never set."""
import numpy as np


class NormalizedLandmark:
    __slots__ = ("_x", "_y", "_z")

    def __init__(self):
        self._x = self._y = self._z = np.float32(0)

    def HasField(self, name):
        return False

    x = property(lambda s: float(s._x), lambda s, v: setattr(s, "_x", np.float32(v)))
    y = property(lambda s: float(s._y), lambda s, v: setattr(s, "_y", np.float32(v)))
    z = property(lambda s: float(s._z), lambda s, v: setattr(s, "_z", np.float32(v)))


class _Repeated(list):
    def add(self):
        lm = NormalizedLandmark()
        self.append(lm)
        return lm


class NormalizedLandmarkList:
    def __init__(self):
        self.landmark = _Repeated()
