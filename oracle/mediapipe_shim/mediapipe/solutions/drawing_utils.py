"""mediapipe.solutions.drawing_utils (0.10.x): DrawingSpec and draw_landmarks, the connection-drawing part on real cv2."""
import dataclasses
import math
from typing import Mapping, Tuple

import cv2

_VISIBILITY_THRESHOLD = 0.5
_PRESENCE_THRESHOLD = 0.5


@dataclasses.dataclass
class DrawingSpec:
    color: Tuple[int, int, int] = (224, 224, 224)
    thickness: int = 2
    circle_radius: int = 2


def _normalized_to_pixel_coordinates(normalized_x, normalized_y, image_width, image_height):
    def is_valid_normalized_value(value):
        return (value > 0 or math.isclose(0, value)) and (value < 1 or math.isclose(1, value))

    if not (is_valid_normalized_value(normalized_x) and is_valid_normalized_value(normalized_y)):
        return None
    x_px = min(math.floor(normalized_x * image_width), image_width - 1)
    y_px = min(math.floor(normalized_y * image_height), image_height - 1)
    return x_px, y_px


def draw_landmarks(image, landmark_list, connections=None, landmark_drawing_spec=DrawingSpec(color=(0, 0, 255)),
                   connection_drawing_spec=DrawingSpec(), is_drawing_landmarks=True):
    if not landmark_list:
        return
    if image.shape[2] != 3:
        raise ValueError("Input image must contain three channel bgr data.")
    image_rows, image_cols, _ = image.shape
    idx_to_coordinates = {}
    for idx, landmark in enumerate(landmark_list.landmark):
        if ((landmark.HasField("visibility") and landmark.visibility < _VISIBILITY_THRESHOLD) or
                (landmark.HasField("presence") and landmark.presence < _PRESENCE_THRESHOLD)):
            continue
        landmark_px = _normalized_to_pixel_coordinates(landmark.x, landmark.y, image_cols, image_rows)
        if landmark_px:
            idx_to_coordinates[idx] = landmark_px
    if connections:
        num_landmarks = len(landmark_list.landmark)
        for connection in connections:
            start_idx, end_idx = connection[0], connection[1]
            if not (0 <= start_idx < num_landmarks and 0 <= end_idx < num_landmarks):
                raise ValueError(f"Landmark index is out of range. Invalid connection from landmark #{start_idx} to "
                                 f"landmark #{end_idx}.")
            if start_idx in idx_to_coordinates and end_idx in idx_to_coordinates:
                drawing_spec = (connection_drawing_spec[connection] if isinstance(connection_drawing_spec, Mapping)
                                else connection_drawing_spec)
                cv2.line(image, idx_to_coordinates[start_idx], idx_to_coordinates[end_idx], drawing_spec.color,
                         drawing_spec.thickness)
    if is_drawing_landmarks and landmark_drawing_spec:
        raise NotImplementedError("landmark circles are not restated (draw_util.py passes landmark_drawing_spec=None)")
