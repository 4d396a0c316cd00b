"""TEST / BENCH INFRASTRUCTURE ONLY -- ctypes face of oracle/_ref/libmsda_refcuda.so, i.e. the REFERENCE's own CUDA
kernels (ms_deform_im2col_cuda.cuh, compiled unmodified for sm_90a by oracle/build_refcuda.sh).

Used by tests/ (parity against the reference op itself on identical tensors) and by tools/opbench.py (the reference
kernels timed on the same GPU). Never imported by the product package.
"""
import ctypes
import os

import torch

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libmsda_refcuda.so")
_lib = None


def available() -> bool:
    return os.path.exists(_PATH)


def _load():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_PATH)
    return _lib


def _common(value, shapes, lsi, loc, attn):
    n, s, m, d = value.shape
    dims = [ctypes.c_int(int(x)) for x in (n, s, m, d, shapes.size(0), loc.size(1), loc.size(4))]
    sfx = {torch.float32: "f32", torch.float64: "f64"}[value.dtype]
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    return dims, sfx, vp


def forward(value, shapes, lsi, loc, attn):
    """Reference K1 (cuh:237-299) via its launcher (cuh:923-954). Output is zero-initialised like at::zeros (cu:54)."""
    dims, sfx, vp = _common(value, shapes, lsi, loc, attn)
    n, s, m, d = value.shape
    out = torch.zeros((n, loc.size(1), m * d), dtype=value.dtype, device=value.device)
    fn = getattr(_load(), "refcuda_forward_" + sfx)
    rc = fn(vp(value), vp(shapes), vp(lsi), vp(loc), vp(attn), *dims, vp(out),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc:
        raise RuntimeError(f"reference forward kernel launch failed: cudaError {rc}")
    return out


def backward(value, shapes, lsi, loc, attn, grad_out, outs=None):
    """Reference K2..K7 via ms_deformable_col2im_cuda (cuh:956-1327); zero-fills the three outputs (cu:121-123)."""
    dims, sfx, vp = _common(value, shapes, lsi, loc, attn)
    if outs is None:
        outs = (torch.zeros_like(value), torch.zeros_like(loc), torch.zeros_like(attn))
    else:
        for t in outs:
            t.zero_()
    gv, gl, ga = outs
    fn = getattr(_load(), "refcuda_backward_" + sfx)
    rc = fn(vp(grad_out), vp(value), vp(shapes), vp(lsi), vp(loc), vp(attn), *dims, vp(gv), vp(gl), vp(ga),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc:
        raise RuntimeError(f"reference backward kernel launch failed: cudaError {rc}")
    return gv, gl, ga
