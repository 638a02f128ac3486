from . import drawing_styles, drawing_utils  # noqa: F401


def __getattr__(name):
    # face_mesh reads the reference checkout: imported on first use only
    if name == "face_mesh":
        import importlib
        return importlib.import_module(".face_mesh", __name__)
    raise AttributeError(name)
