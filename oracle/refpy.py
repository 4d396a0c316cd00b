"""TEST INFRASTRUCTURE ONLY -- the reference's OWN CPU path, ``ms_deform_attn_core_pytorch``
(``ops/functions/ms_deform_attn_func.py:43-63``), loaded from the reference file itself.

Where a reference checkout exists, ``stage()`` (run by hand, e.g. by tests/golden/make_reference_golden.py) copies the
one reference file byte for byte into the git-ignored ``oracle/_ref/``; it never enters history.  Users: the golden
generator, and ``bench.py``'s ``cpu_baseline`` leg and ``--impl reference`` arm, which report ``kind: "reference"``
when a staged copy exists and otherwise time the port (``kind: "port"``) that the stored reference results pin.  Nothing under ``uninext_b200/`` imports this module.

The file imports the compiled extension ``MultiScaleDeformableAttention`` at module level (``func.py:18``) although the
CPU function never touches it; it is loaded here against an EMPTY stand-in module so that the reference arm loads none
of this repo's native code.
"""
from __future__ import annotations

import importlib.util
import os
import shutil
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
_REL = "projects/UNINEXT/uninext/models/deformable_detr/ops/functions/ms_deform_attn_func.py"
REFERENCE = os.environ.get("UNINEXT_REFERENCE", "/root/reference")      # a checkout of the reference repository
SOURCE = os.path.join(REFERENCE, _REL)
STAGED = os.path.join(_HERE, "_ref", "ms_deform_attn_func.py")

_cached = None


def stage() -> bool:
    """Copy the reference file into oracle/_ref/ (where a reference checkout exists). True when a staged copy exists afterwards."""
    if os.path.isfile(SOURCE):
        os.makedirs(os.path.dirname(STAGED), exist_ok=True)
        if not os.path.exists(STAGED) or os.path.getmtime(STAGED) < os.path.getmtime(SOURCE):
            shutil.copyfile(SOURCE, STAGED)
    return os.path.isfile(STAGED)


def available() -> bool:
    return os.path.isfile(STAGED)


def core_pytorch():
    """-> the reference's ``ms_deform_attn_core_pytorch`` (value, value_spatial_shapes, sampling_locations,
    attention_weights) -> [N, Lq, M*D], or None when no staged copy of the reference file exists."""
    global _cached
    if _cached is not None:
        return _cached
    if not available():
        return None
    name = "MultiScaleDeformableAttention"
    had = sys.modules.get(name)
    sys.modules[name] = types.ModuleType(name)             # stand-in for the compiled extension (func.py:18)
    try:
        import warnings
        spec = importlib.util.spec_from_file_location("_msda_reference_func", STAGED)
        mod = importlib.util.module_from_spec(spec)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")               # torch.cuda.amp.custom_fwd deprecation in the decorators
            spec.loader.exec_module(mod)
    finally:
        if had is not None:
            sys.modules[name] = had
        else:
            del sys.modules[name]
    _cached = mod.ms_deform_attn_core_pytorch
    return _cached
