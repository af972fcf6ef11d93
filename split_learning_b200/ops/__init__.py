"""Hand-written sm_90a kernels (``csrc/*.cu`` → ``_slb200.so``) and their Python bindings."""
from . import build, native

__all__ = ["build", "native"]
