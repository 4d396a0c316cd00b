#!/usr/bin/env python
"""Regenerate tests/golden/reference/*.npz: the results of the reference's own classes and functions on the inputs the
tests build from fixed seeds, computed on the CPU with the reference's own ``ms_deform_attn_core_pytorch`` standing in
for its compiled extension.  Needs a reference checkout (staged by tests/stage_reference.py); the tests themselves do not.

    MSDA_RECORD_REFERENCE=1 python tests/golden/make_reference_golden.py
"""
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
assert os.environ.get("MSDA_RECORD_REFERENCE") == "1", "run with MSDA_RECORD_REFERENCE=1"

import torch  # noqa: E402

from tests import stage_reference  # noqa: E402


class _CpuKernels:
    """The reference pybind module's two entry points, computed with the reference's own CPU function."""
    core = None

    @classmethod
    def ms_deform_attn_forward(cls, value, shapes, lsi, loc, attn, im2col_step):
        with torch.no_grad():
            return cls.core(value, shapes, loc, attn)

    @classmethod
    def ms_deform_attn_backward(cls, value, shapes, lsi, loc, attn, grad_output, im2col_step):
        with torch.enable_grad():
            v, lo, at = (t.detach().clone().requires_grad_(True) for t in (value, loc, attn))
            return list(torch.autograd.grad(cls.core(v, shapes, lo, at), (v, lo, at), grad_output))


def main():
    assert stage_reference.stage(), "no reference checkout to stage from"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        func_mod = stage_reference.import_reference()[0]
    _CpuKernels.core = staticmethod(func_mod.ms_deform_attn_core_pytorch)
    func_mod.MSDA = _CpuKernels
    torch.set_default_dtype(torch.float32)
    from tests import test_gpu_reference_dropin as t
    for which in (0, 1):
        t.test_reference_module_and_encoder_layer_on_dropin(which)
        t.test_reference_decoder_layer_on_dropin(which)
    t.test_reference_reid_head_on_dropin()
    for refine in (True, False):
        t.test_reference_decoder_loop_on_dropin(refine, False)
    t.test_geometry_kernels_match_reference_functions()
    from tests import test_gpu_condinst as c
    for factor in (2, 4):
        for shape in c.BILINEAR_SHAPES:
            c.test_aligned_bilinear_matches_reference(factor, shape)
    for rel_coord in (True, False):
        for case in c.MASK_CASES:
            c.test_dynamic_mask_head_matches_reference(rel_coord, *case)
    from tests import test_reference_mirrors as m
    m.record()
    from tests import test_bench_cli as b
    b.test_reference_file_and_port_agree()
    print("written:", sorted(os.listdir(os.path.join(ROOT, "tests", "golden", "reference"))))


if __name__ == "__main__":
    main()
