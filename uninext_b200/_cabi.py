"""ctypes binding of libmsda_b200.so (the C ABI in include/msda_b200.h).

There is NO fallback: if the library is missing or does not export every declared symbol, importing the ops fails
with a RuntimeError that says how to build it. The product never routes through ``oracle/`` or a PyTorch
re-implementation.
"""
from __future__ import annotations

import ctypes
import os

import torch

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "lib", "libmsda_b200.so")

_vp, _i, _u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
_DIMS = [_i] * 7

# name -> (restype, argtypes); mirrors include/msda_b200.h one to one (tests/test_cabi_symbols.py checks it).
SIGNATURES = {
    "msda_abi_version": (_i, []),
    "msda_strerror": (ctypes.c_char_p, [_i]),
    "msda_uses_fast_path": (_i, [_i, _i, _i, _i]),
    "msda_launch_count": (_u64, []),
    "msda_set_knob": (_i, [_i, _i]),
    "msda_forward_f32": (_i, [_vp] * 5 + _DIMS + [_vp, _vp]),
    "msda_forward_f64": (_i, [_vp] * 5 + _DIMS + [_vp, _vp]),
    "msda_forward_bf16": (_i, [_vp] * 5 + _DIMS + [_vp, _vp]),
    "msda_backward_f32": (_i, [_vp] * 6 + _DIMS + [_vp] * 3 + [_vp]),
    "msda_backward_f64": (_i, [_vp] * 6 + _DIMS + [_vp] * 3 + [_vp]),
    "msda_backward_bf16": (_i, [_vp] * 6 + _DIMS + [_vp] * 4 + [_vp]),
    "msda_backward_det_workspace": (_i, [_i] * 9 + [_vp]),
    "msda_backward_det_f32": (_i, [_vp] * 6 + _DIMS + [_vp] * 3 + [_vp, ctypes.c_int64, _vp]),
    "msda_backward_det_f64": (_i, [_vp] * 6 + _DIMS + [_vp] * 3 + [_vp, ctypes.c_int64, _vp]),
    "msda_backward_det_bf16": (_i, [_vp] * 6 + _DIMS + [_vp] * 4 + [_vp, ctypes.c_int64, _vp]),
    "msda_prologue_forward_f32": (_i, [_vp] * 3 + [ctypes.c_int64, _i, _i, _i, _i] + [_vp] * 3),
    "msda_prologue_backward_f32": (_i, [_vp] * 5 + [ctypes.c_int64, _i, _i, _i, _i] + [_vp] * 2),
    "msda_colsum_f32": (_i, [_vp, ctypes.c_int64, _i, _vp, _vp]),
    "msda_relu_backward_colsum_f32": (_i, [_vp, _vp, ctypes.c_int64, _i, _vp, _vp, _vp]),
    "msda_add_layernorm_forward_f32": (_i, [_vp] * 4 + [ctypes.c_int64, _i, ctypes.c_float] + [_vp] * 5),
    "msda_layernorm_backward_f32": (_i, [_vp] * 5 + [ctypes.c_int64, _i] + [_vp] * 4),
    "msda_linear_tf32": (_i, [_vp] * 3 + [ctypes.c_int64, _i, _i, _vp, _vp]),
    "msda_linear_tf32_ex": (_i, [_vp] * 4 + [ctypes.c_int64, _i, _i, _i, _vp, _vp]),
    "msda_linear_tf32_ws_ok": (_i, [_i, _i]),
    "msda_valid_counts": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp]),
    "msda_encoder_ref_points_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp]),
    "msda_encoder_proposals_f32": (_i, [_vp] * 4 + [_i] * 3 + [ctypes.c_float, _vp, _vp, _vp]),
    "msda_sine_pos_embed_forward_f32": (_i, [_vp, ctypes.c_int64, _i, _i, ctypes.c_float, _i, _vp, _vp]),
    "msda_sine_pos_embed_backward_f32": (_i, [_vp, _vp, ctypes.c_int64, _i, _i, ctypes.c_float, _i, _vp, _vp]),
    "msda_condinst_forward_f32": (_i, [_vp] * 4 + [_i] * 7 + [_vp, _vp]),
    "msda_condinst_backward_f32": (_i, [_vp] * 5 + [_i] * 7 + [_vp] * 4),
    "msda_aligned_bilinear_forward_f32": (_i, [_vp, ctypes.c_int64, _i, _i, _i, _vp, _vp]),
    "msda_aligned_bilinear_backward_f32": (_i, [_vp, ctypes.c_int64, _i, _i, _i, _vp, _vp]),
    "msda_mask_paste_f32": (_i, [_vp, ctypes.c_int64] + [_i] * 7 + [ctypes.c_float, _i, _vp, _vp]),
    "msda_mask_rle_workspace": (_i, [ctypes.c_int64, _i, _i, _vp]),
    "msda_mask_rle_count_f32": (_i, [_vp, ctypes.c_int64] + [_i] * 7 + [ctypes.c_float, _vp, ctypes.c_int64, _vp]),
    "msda_mask_rle_count_u8": (_i, [_vp, ctypes.c_int64, _i, _i, _vp, ctypes.c_int64, _vp]),
    "msda_mask_rle_encode": (_i, [ctypes.c_int64, _i, _i, ctypes.c_int64, _vp, ctypes.c_int64] + [_vp] * 4),
    "msda_detpost_workspace": (_i, [_i] * 5 + [_vp]),
    "msda_detpost_f32": (_i, [_vp] * 6 + [_i] * 5 + [ctypes.c_float, _i] + [_vp] * 6 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_workspace": (_i, [_i] * 5 + [_vp]),
    "msda_vlfuse_forward_f32": (_i, [_vp] * 5 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 4 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_backward_f32": (_i, [_vp] * 10 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 5 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_dropout_mask_f32": (_i, [_vp] + [_i] * 4 + [ctypes.c_float] + [_vp] * 3),
    "msda_vlfuse_forward_tf32": (_i, [_vp] * 5 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 4 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_backward_tf32": (_i, [_vp] * 10 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 5 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_forward_bf16": (_i, [_vp] * 5 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 4 + [ctypes.c_int64, _vp]),
    "msda_vlfuse_backward_bf16": (_i, [_vp] * 10 + [_i] * 7 + [ctypes.c_float, _vp] + [_vp] * 5 + [ctypes.c_int64, _vp]),
}
ABI_VERSION = 11

# Optional groups: typed by load() when the library exports them; asking for one of a library that does not raises
# MSDALibraryError (entry(), or twostage() / flatten() for a whole group).  The two-stage query selection
# (include/msda_twostage.h):
_i64 = ctypes.c_int64
TWOSTAGE_SIGNATURES = {
    "msda_twostage_head_forward_f32": (_i, [_vp] * 7 + [_i] * 3 + [ctypes.c_float, _i] + [_vp] * 4 + [_vp]),
    "msda_twostage_head_workspace": (_i, [_i] * 3 + [_vp]),
    "msda_twostage_head_backward_f32": (_i, [_vp] * 11 + [_i] * 4 + [_vp] * 6 + [_vp, _i64, _vp]),
    "msda_twostage_select_workspace": (_i, [_i] * 3 + [_vp]),
    "msda_twostage_select_forward_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp] * 3 + [_vp, _i64, _vp]),
    "msda_twostage_select_backward_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp]),
}
# The encoder's input preparation (include/msda_flatten.h):
FLATTEN_SIGNATURES = {
    "msda_flatten_levels_forward_f32": (_i, [_vp] * 5 + [_i] * 3 + [_vp] * 4 + [_vp]),
    "msda_flatten_levels_workspace": (_i, [_vp] * 2 + [_i] * 3 + [_vp]),
    "msda_flatten_levels_backward_f32": (_i, [_vp] * 4 + [_i] * 3 + [_vp] * 4 + [_i64, _vp]),
}
# Typed by entry() on first use rather than by load(), so a library without them leaves load().missing as it was: the
# video trackers' detection selection (include/msda_trackpost.h).
TRACKPOST_SIGNATURES = {
    "msda_trackpost_workspace": (_i, [_i] * 4 + [_vp]),
    "msda_trackpost_f32": (_i, [_vp] * 6 + [_i] * 4 + [ctypes.c_float] * 2 + [_i] + [_vp] * 5 + [_vp, _i64, _vp]),
}
# Typed late in the same way: the IDOL tracker's association step (include/msda_tracker.h).
TRACKER_SIGNATURES = {
    "msda_idol_workspace": (_i, [_i] * 5 + [_vp]),
    "msda_idol_match_f32": (_i, [_vp] * 5 + [_i] * 5 + [ctypes.c_float] * 5 + [ctypes.c_double] + [_i] * 3 + [_vp] +
                            [_i] * 2 + [_vp] * 7 + [_vp, _i64, _vp]),
}
# And the QuasiDense tracker's (include/msda_qdtrack.h).
QDTRACK_SIGNATURES = {
    "msda_qdtrack_workspace": (_i, [_i] * 3 + [_vp]),
    "msda_qdtrack_match_f32": (_i, [_vp] * 6 + [_i] * 3 + [ctypes.c_float] * 6 + [ctypes.c_double] + [_i] * 4 +
                               [_vp] * 7 + [_vp, _i64, _vp]),
}
IDOL_LONG_MATCH, IDOL_FRAME_WEIGHT, IDOL_TEMPORAL_WEIGHT = 1, 2, 4                                # include/msda_tracker.h
IDOL_OVERFLOW, IDOL_BAD_ROW = 1, 2
QD_BACKDROPS, QD_MAX_BACKDROPS, QD_OVERFLOW, QD_BAD_ROW = 1, 1024, 1, 2                                  # include/msda_qdtrack.h
TRACKPOST_CXCYWH, TRACKPOST_XYXY_PIXELS = 0, 1                                                         # include/msda_trackpost.h
(KNOB_SLAB, KNOB_BWD_WIN_ROWS, KNOB_BWD_LIST_CAP, KNOB_FWD_SLAB_CTAS, KNOB_F32_VEC8_FWD, KNOB_F32_VEC8_BWD,
 KNOB_BF16_FINE_ROWS, KNOB_BF16_PACKED_FWD, KNOB_ZERO_FILL, KNOB_REGION_BWD) = range(10)                                                   # include/msda_b200.h

_lib = None


class MSDALibraryError(RuntimeError):
    pass


def load(path: str | None = None):
    """Load (once) and type the library. Raises MSDALibraryError loudly when it is absent or stale."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise MSDALibraryError(
            f"{p} not found: the CUDA extension is not built. Run `python -m uninext_b200.build` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU / PyTorch fallback.")
    try:
        lib = ctypes.CDLL(p)
    except OSError as exc:
        raise MSDALibraryError(f"cannot load {p}: {exc}") from exc
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:
            raise MSDALibraryError(f"{p} does not export `{name}` (stale build? run uninext_b200.build --force)") from exc
        fn.restype, fn.argtypes = res, args
    lib.missing = set()                    # the optional entry points this library does not export
    for name, (res, args) in {**TWOSTAGE_SIGNATURES, **FLATTEN_SIGNATURES}.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        else:
            lib.missing.add(name)
    if lib.msda_abi_version() != ABI_VERSION:
        raise MSDALibraryError(f"{p}: ABI version {lib.msda_abi_version()} != expected {ABI_VERSION}")
    if path is None:
        _lib = lib
    return lib


_entries = {}


def entry(name: str, path: str | None = None):
    """The typed entry point ``name`` of ``load(path)``.  MSDALibraryError when the library does not export it: an
    optional group it was built without."""
    fn = _entries.get(name) if path is None else None
    if fn is None:
        lib = load(path)
        late = TRACKPOST_SIGNATURES.get(name) or TRACKER_SIGNATURES.get(name) or QDTRACK_SIGNATURES.get(name)
        if name in lib.missing or (late and not hasattr(lib, name)):
            raise MSDALibraryError(f"{path or LIB_PATH} does not export `{name}` (stale build? run "
                                   "uninext_b200.build --force)")
        fn = getattr(lib, name)
        if late:
            fn.restype, fn.argtypes = late
        if path is None:
            _entries[name] = fn
    return fn


def _with_group(table, path):
    for name in table:
        entry(name, path)
    return load(path)


def twostage(path: str | None = None):
    """The library, after checking that it exports the two-stage selection (include/msda_twostage.h)."""
    return _with_group(TWOSTAGE_SIGNATURES, path)


def flatten(path: str | None = None):
    """The library, after checking that it exports the input preparation (include/msda_flatten.h)."""
    return _with_group(FLATTEN_SIGNATURES, path)


def trackpost(path: str | None = None):
    """The library, after checking that it exports the trackers' detection selection (include/msda_trackpost.h)."""
    return _with_group(TRACKPOST_SIGNATURES, path)


def tracker(path: str | None = None):
    """The library, after checking that it exports the IDOL tracker's association step (include/msda_tracker.h)."""
    return _with_group(TRACKER_SIGNATURES, path)


def qdtrack(path: str | None = None):
    """The library, after checking that it exports the QuasiDense tracker's association step (include/msda_qdtrack.h)."""
    return _with_group(QDTRACK_SIGNATURES, path)


def call(name: str, *args, device) -> None:
    """Run entry point ``name`` on ``device``: a tensor argument goes as its ``data_ptr()``, None as NULL, anything else
    (ints, floats, ctypes objects) unchanged, and the device's current stream is appended as the last argument.  A
    non-zero return code raises RuntimeError (``check``).  Nothing here synchronises or allocates, so calls can be
    captured into a CUDA graph."""
    fn = entry(name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(device):
        code = fn(*args, torch.cuda.current_stream(device).cuda_stream)
    if code:
        check(code, name)


def workspace(name: str, *args) -> int:
    """The size that the query ``name`` writes through its last parameter, an ``int64_t *``."""
    n = ctypes.c_int64(0)
    check(entry(name)(*args, ctypes.byref(n)), name)
    return n.value


def check(code: int, what: str) -> None:
    """Turn a non-zero C-ABI return code into a RuntimeError (the reference only printf()s launch failures,
    ms_deform_im2col_cuda.cuh:948-952)."""
    if code != 0:
        msg = load().msda_strerror(code)
        raise RuntimeError(f"{what} failed with code {code}: {msg.decode() if msg else '?'}")
