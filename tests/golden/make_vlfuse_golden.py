#!/usr/bin/env python
"""Regenerate tests/golden/reference/vlfuse_*.npz: the reference's own BiAttentionBlockForCheckpoint
(fuse_helper.py:142-179) on the CPU, in eval mode, on the cases of tests/vlfuse_case.py.  Needs a reference checkout;
the tests themselves do not.

    python tests/golden/make_vlfuse_golden.py

fuse_helper.py is copied verbatim into the git-ignored oracle/_ref/vlfuse/.  Written here, not copied: a stub of the one
name it imports from timm (``DropPath``, unused at drop_path = 0) and the cfg namespace that carries the three fusion
flags at the reference config's defaults (STABLE_SOFTMAX_2D False, both clamps True).
"""
import importlib.util
import os
import shutil
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refpy import REFERENCE  # noqa: E402
from tests import vlfuse_case as vc  # noqa: E402

SRC = os.path.join(REFERENCE, "projects/UNINEXT/uninext/models/deformable_detr/fuse_helper.py")
DEST = os.path.join(ROOT, "oracle", "_ref", "vlfuse")
OUT = os.path.join(ROOT, "tests", "golden", "reference")


def _reference_module():
    os.makedirs(DEST, exist_ok=True)
    shutil.copyfile(SRC, os.path.join(DEST, "fuse_helper.py"))
    timm = types.ModuleType("timm")
    timm.models = types.ModuleType("timm.models")
    timm.models.layers = types.ModuleType("timm.models.layers")

    class DropPath(torch.nn.Module):
        def __init__(self, p=0.0):
            super().__init__()
            raise NotImplementedError("DropPath stub: the fusion block is built with drop_path = 0")

    timm.models.layers.DropPath = DropPath
    sys.modules.update({"timm": timm, "timm.models": timm.models, "timm.models.layers": timm.models.layers})
    spec = importlib.util.spec_from_file_location("ref_fuse_helper", os.path.join(DEST, "fuse_helper.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _cfg():
    fuse = types.SimpleNamespace(STABLE_SOFTMAX_2D=False, CLAMP_MIN_FOR_UNDERFLOW=True, CLAMP_MAX_FOR_OVERFLOW=True)
    return types.SimpleNamespace(MODEL=types.SimpleNamespace(DYHEAD=types.SimpleNamespace(FUSE_CONFIG=fuse)))


def main():
    ref = _reference_module()
    torch.set_num_threads(os.cpu_count() or 1)
    for name in vc.CASES:
        block = ref.BiAttentionBlockForCheckpoint(vc.V_DIM, vc.L_DIM, vc.EMBED, vc.HEADS, dropout=0.1, drop_path=0.0,
                                                  init_values=1.0 / 6, cfg=_cfg())
        rec = vc.run(block, name, "cpu")
        rec["state_dict_keys"] = np.array(sorted(block.state_dict().keys()))
        np.savez_compressed(os.path.join(OUT, f"vlfuse_{name}.npz"), **rec)
        print("written", name, {k: v.shape for k, v in rec.items() if not k.startswith("grad.attn")})


if __name__ == "__main__":
    main()
