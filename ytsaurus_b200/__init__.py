"""ytsaurus_b200 — H100-native sort/shuffle + scan→filter→hash-aggregate hot path of YTsaurus.

The compute lives in hand-written CUDA (csrc/, sm_90a) behind the C ABI of include/ytgpu.h
(libytgpu.so).  This package is the thin host side: ctypes binding (capi), the flat row model
(rowset), PyTorch-backed buffers/streams (runtime) and the in-box multi-GPU shuffle (shuffle).
"""
from . import capi, rowset  # noqa: F401
from .rowset import EValueType, ESortOrder, Rowset, U64, Sentinel, make_rowset, VALUE_DTYPE  # noqa: F401


def __getattr__(name):
    if name in ("GpuContext", "Column"):
        from . import runtime
        return getattr(runtime, name)
    raise AttributeError(name)
