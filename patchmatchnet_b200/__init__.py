"""patchmatchnet_b200 -- H100-native (sm_90a) learned-PatchMatch hot path of PatchmatchNet.

Public surface (mirrors the reference's ``models`` package for this path):

    PatchMatch      drop-in for reference models/patchmatch.py:PatchMatch
    PatchmatchNet   caller-side shell with the reference constructor/forward (models/net.py)
    ops             tensor-level wrappers over the C ABI (include/patchmatch_b200.h)
"""
import os as _os

from . import _native, data_io, distributed, engine, ops, synthetic  # noqa: F401
from .net import PatchmatchNet, load_reference_state, patchmatchnet_loss  # noqa: F401
from .patchmatch import PatchMatch  # noqa: F401

# torch.ops.pmb200.* (TorchScript-facing registration of the same C ABI): registered on import when the shim is built,
# so that `torch.jit.script(model)` / `torch.jit.load(path)` work after a plain `import patchmatchnet_b200`.
# Not when libpmb200.so is older than its sources: loading the shim would map the stale library into the process and the
# rebuild that build() is about to do could no longer be loaded under the same path.
# PMB200_SKIP_TORCH_OPS=1: a process that must not map the native libraries at all (bench.py --impl reference).
if (_os.environ.get("PMB200_SKIP_TORCH_OPS") != "1" and _os.path.exists(_native.TORCH_LIB_PATH)
        and not _native.needs_rebuild()):
    _native.load_torch_ops()

__all__ = ["PatchMatch", "PatchmatchNet", "load_reference_state", "patchmatchnet_loss"]
