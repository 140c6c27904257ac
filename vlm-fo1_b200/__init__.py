"""vlm-fo1_b200 -- host-side mirror of the VLM-FO1 hot path over libfo1.so (sm_90a CUDA).

The directory name follows the repo convention (``vlm-fo1_b200``); import it as
``importlib.import_module("vlm-fo1_b200")`` or through the ``fo1_b200`` alias module at the repo root.
PyTorch is used only for device memory, streams and torch.distributed plumbing.
"""
from . import _lib  # noqa: F401
from ._lib import Fo1Error, lib  # noqa: F401
