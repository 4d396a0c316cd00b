"""CPU tests of the host-side mirror of the reference interface (no GPU, no compute calls)."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_args():
    shapes = torch.tensor([[2, 2]])
    return (torch.zeros(1, 4, 1, 2), shapes, torch.tensor([0]), torch.zeros(1, 1, 1, 1, 1, 2),
            torch.zeros(1, 1, 1, 1, 1))


def test_dropin_exports_reference_names_and_refuses_cpu():
    from uninext_b200.dropin import MultiScaleDeformableAttention as M
    assert set(M.__all__) == {"ms_deform_attn_forward", "ms_deform_attn_backward"}      # vision.cpp:13-16
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):               # ms_deform_attn.h:38
        M.ms_deform_attn_forward(*_cpu_args(), 64)
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        M.ms_deform_attn_backward(*_cpu_args(), torch.zeros(1, 1, 2), 64)
    v = torch.zeros(1, 4, 1, 4)[..., ::2]                       # same shape as value, not contiguous
    with pytest.raises(RuntimeError, match="contiguous"):                               # cu:28
        M.ms_deform_attn_forward(v, *_cpu_args()[1:], 64)


def test_shape_cross_checks_reject_inconsistent_tensors():
    """The reference reads sizes from each tensor without cross-checking (cu:40-48); the drop-in refuses instead."""
    from uninext_b200.dropin import MultiScaleDeformableAttention as M
    v, ss, lsi, loc, at = _cpu_args()
    M._check_shapes(v, ss, lsi, loc, at)                                    # consistent: passes
    M._check_shapes(v, ss, lsi, loc, at, torch.zeros(1, 1, 2))
    bad = [
        (v[0], ss, lsi, loc, at, None, "value must be"),
        (v, ss.view(-1), lsi, loc, at, None, "spatial_shapes must be"),
        (v, ss, torch.tensor([0, 4]), loc, at, None, "level_start_index must be"),
        (v, ss, lsi, torch.zeros(1, 1, 2, 1, 1, 2), at, None, "sampling_loc must be"),       # heads differ from value
        (v, ss, lsi, torch.zeros(1, 1, 1, 2, 1, 2), at, None, "sampling_loc must be"),       # levels differ
        (v, ss, lsi, loc, torch.zeros(1, 1, 1, 1, 3), None, "attn_weight must be"),
        (v, ss, lsi, loc, at, torch.zeros(1, 2, 2), "grad_output must be"),
    ]
    for *args, go, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            M._check_shapes(*args, go)


def test_function_signature_matches_reference():
    from uninext_b200.functions import MSDeformAttnFunction
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        MSDeformAttnFunction.apply(*_cpu_args(), 64)


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under uninext_b200/ may import, load or mention it."""
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "uninext_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle|libmsda_oracle|msda_oracle|grid_sample", text, flags=re.M):
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_module_matches_reference_parameters_and_location_math():
    from uninext_b200.modules import MSDeformAttn
    m = MSDeformAttn(256, 4, 8, 4)
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {
        "sampling_offsets.weight": (256, 256), "sampling_offsets.bias": (256,),
        "attention_weights.weight": (128, 256), "attention_weights.bias": (128,),
        "value_proj.weight": (256, 256), "value_proj.bias": (256,),
        "output_proj.weight": (256, 256), "output_proj.bias": (256,)}                  # SURVEY.md section 5
    # ring initialisation: head 0 points along +x, point p at distance p+1 (ms_deform_attn.py:64-70)
    b = sd["sampling_offsets.bias"].view(8, 4, 4, 2)
    assert torch.allclose(b[0, :, :, 0], torch.tensor([1.0, 2.0, 3.0, 4.0]).expand(4, 4))
    assert torch.allclose(b[0, :, :, 1], torch.zeros(4, 4), atol=1e-6)
    assert torch.allclose(b[2, 0, 1], torch.tensor([0.0, 2.0]), atol=1e-6)
    shapes = torch.tensor([[4, 8], [2, 4]])
    off = torch.randn(1, 3, 8, 2, 4, 2)
    ref2 = torch.rand(1, 3, 2, 2)
    loc = MSDeformAttn(256, 2, 8, 4).sampling_locations(off, ref2, shapes)
    want = ref2[:, :, None, :, None, :] + off / torch.tensor([[8.0, 4.0], [4.0, 2.0]])[None, None, None, :, None, :]
    assert torch.allclose(loc, want)                                                    # ms_deform_attn.py:103-106
    ref4 = torch.rand(1, 3, 2, 4)
    loc4 = MSDeformAttn(256, 2, 8, 4).sampling_locations(off, ref4, shapes)
    want4 = ref4[:, :, None, :, None, :2] + off / 4 * ref4[:, :, None, :, None, 2:] * 0.5
    assert torch.allclose(loc4, want4)                                                  # ms_deform_attn.py:107-109
    with pytest.raises(ValueError):
        MSDeformAttn(256, 2, 8, 4).sampling_locations(off, torch.rand(1, 3, 2, 3), shapes)
    with pytest.raises(ValueError):
        MSDeformAttn(250, 4, 8, 4)


def test_workload_shapes_match_survey_table():
    from uninext_b200.workloads import CONFIGS, algorithmic_bytes
    c2 = CONFIGS["cfg2"]
    assert c2.shapes == [(100, 168), (50, 84), (25, 42), (13, 21)] and c2.S == 22323
    assert c2.samples("enc") == 5714688 and c2.samples("dec") == 76800
    assert CONFIGS["cfg1"].S == 2125 and CONFIGS["cfg3"].S == 32640 and CONFIGS["cfg4"].S == 5100
    assert algorithmic_bytes(c2, "enc", 4, "fwd") == 160011264            # 28 B / sample
    assert algorithmic_bytes(c2, "enc", 4, "bwd") == 320022528            # 56 B / sample


def test_level_table_is_validated_once_per_distinct_table():
    """`MSDeformAttn` keeps the reference's `(H_l * W_l).sum() == Len_in` assertion (ms_deform_attn.py:91) but pays its
    device->host read once per distinct table: cached on (storage, version), re-checked after an in-place change."""
    from uninext_b200.modules import ms_deform_attn as mod
    ss = torch.tensor([[4, 5], [2, 3]])
    lsi = torch.tensor([0, 20])
    mod._LEVELS_OK.clear()
    mod.check_levels(ss, lsi, 26)
    assert len(mod._LEVELS_OK) == 1
    mod.check_levels(ss, lsi, 26)                                           # cache hit: no new entry
    assert len(mod._LEVELS_OK) == 1
    with pytest.raises(AssertionError, match="Len_in"):
        mod.check_levels(ss, lsi, 27)                                       # same table, other flattened length
    with pytest.raises(AssertionError, match="level_start_index"):
        mod.check_levels(ss, torch.tensor([0, 19]), 26)
    with pytest.raises(AssertionError, match="positive"):
        mod.check_levels(torch.tensor([[4, 5], [0, 3]]), None, 20)          # an empty level would index row -1
    ss[1, 1] = 4                                                            # in-place edit bumps the version counter
    with pytest.raises(AssertionError, match="Len_in"):
        mod.check_levels(ss, lsi, 26)
    mod.check_levels(ss, lsi, 28)
