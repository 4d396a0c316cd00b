"""uninext_b200 -- H100-native (sm_90a) multi-scale deformable attention (the package name is historical): the hot path of UNINEXT's deformable
transformer, behind the reference's own operator boundary.

Layout
    csrc/        hand-written CUDA kernels + the C ABI (include/msda_b200.h)  -> lib/libmsda_b200.so
    _cabi.py     ctypes binding (fails loudly when the library is missing; there is no fallback)
    dropin/      ``MultiScaleDeformableAttention`` -- module-level drop-in for the reference's pybind extension
    functions/   ``MSDeformAttnFunction`` (reference autograd signature) and a bf16 variant
    modules/     ``MSDeformAttn`` nn.Module with the reference's parameters / state_dict keys
"""
import os as _os
import sys as _sys

__version__ = "0.1.0"


def install_dropin() -> None:
    """Make ``import MultiScaleDeformableAttention`` (reference ops/functions/ms_deform_attn_func.py:18) resolve to
    the sm_90a implementation."""
    from uninext_b200.dropin import MultiScaleDeformableAttention as _m
    _sys.modules["MultiScaleDeformableAttention"] = _m


def dropin_path() -> str:
    """Directory to prepend to PYTHONPATH for the same effect without code changes."""
    return _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "dropin")
