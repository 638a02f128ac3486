"""Audio front end of SURVEY.md 8f (N3): the KV-cached head-pose decoder loop and the wav2vec2 encoder / Audio2Mesh head
on the library's kernels."""
from .pose_infer import enable_kv_cache, kv_cached_infer  # noqa: F401
from .wav2vec2 import enable_kernels  # noqa: F401
