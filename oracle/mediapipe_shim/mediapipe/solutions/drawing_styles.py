from .drawing_utils import DrawingSpec  # noqa: F401
