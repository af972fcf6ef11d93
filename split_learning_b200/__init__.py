"""split_learning_b200 — a Hopper-native (H100) split-learning engine (see DESIGN.md)."""
__version__ = "0.1.0"

import os as _os

# One hardware work queue per stream (the default is 8): several clients in one process (tests, N = 1 benchmark, launch.py
# on a one-GPU box) own 2-3 streams each; with queue aliasing a flag-waiting kernel of one stream can sit in front of the
# kernel of another stream that would publish that flag.  Must be set before the CUDA context exists.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

# NOTE on CUDA lazy module loading: a kernel that spins on a mailbox flag must not be the reason a
# sibling kernel's *first* launch blocks (lazy loading may wait for running kernels).  The pipelines
# therefore run every program once, sequentially, before any overlapped/graph execution
# (``DeviceStage._exec`` eager first pass).  Forcing CUDA_MODULE_LOADING=EAGER instead costs minutes
# of start-up (torch's fatbins) — measured, rejected.
