"""GPU tests (-m gpu) of the CondInst dynamic mask head (uninext_b200/modules/dynamic_mask_head.py, kernels in
csrc/msda_condinst.cuh) against stored results of the REFERENCE functions -- ``DDETRSegmUni.dynamic_mask_with_coords`` /
``mask_heads_forward`` / ``parse_dynamic_params`` / ``aligned_bilinear`` / ``compute_locations`` of
uninext/models/ddetrs.py, run in fp32 with grouped convolutions (tests/golden/reference/, tests/refgolden.py): forward and
every gradient (mask features, dynamic parameters, reference points), 2e-4 of scale."""
import types
import warnings

import pytest
import torch

from tests import refgolden

pytestmark = pytest.mark.gpu

DEV = "cpu" if refgolden.RECORDING else "cuda"
if torch.cuda.is_available() or refgolden.RECORDING:
    from uninext_b200.modules.dynamic_mask_head import (CondInstMaskHead, aligned_bilinear, dynamic_mask_with_coords,
                                                        dynamic_param_counts)


def _ddetrs():
    from tests import stage_reference
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return stage_reference.import_ddetrs()


def _holder(ddetrs, rel_coord, mask_out_stride):
    """An object with exactly the attributes the reference method reads (ddetrs.py:45-70)."""
    h = types.SimpleNamespace(dynamic_mask_channels=8, mask_out_stride=mask_out_stride, use_raft=False)
    h.weight_nums, h.bias_nums = dynamic_param_counts(3, rel_coord)
    h.mask_heads_forward = lambda *a: ddetrs.DDETRSegmUni.mask_heads_forward(h, *a)
    return h


BILINEAR_SHAPES = [(3, 5, 7), (2, 1, 1), (1, 13, 21), (5, 40, 66)]
MASK_CASES = [([5, 3], (12, 20), 4), ([0, 7], (9, 11), 4), ([37, 21, 1], (25, 42), 8), ([300], (32, 40), 4),
              ([30, 17], (100, 168), 4), ([3], (7, 9), 2)]


@pytest.mark.parametrize("factor", [2, 4])
@pytest.mark.parametrize("shape", BILINEAR_SHAPES)
def test_aligned_bilinear_matches_reference(factor, shape):
    group = f"aligned_bilinear_{factor}_{'x'.join(map(str, shape))}"
    g = torch.Generator().manual_seed(1)
    x = torch.randn(*shape, generator=g).to(DEV)
    a = x.clone().requires_grad_(True)
    if refgolden.RECORDING:
        out = _ddetrs().aligned_bilinear(a[None], factor)[0]
    else:
        out = aligned_bilinear(a, factor)
    go = torch.randn(out.shape, generator=g).to(DEV)
    out.backward(go)
    if refgolden.RECORDING:
        refgolden.put(group, "out", out)
        refgolden.put(group, "grad", a.grad)
        refgolden.flush(group)
        return
    want = refgolden.load(group)
    assert refgolden.rel(out, want, "out", group) < 1e-6
    assert refgolden.rel(a.grad, want, "grad", group) < 1e-5


@pytest.mark.parametrize("rel_coord", [True, False])
@pytest.mark.parametrize("num_insts,hw,mask_out_stride", MASK_CASES)
def test_dynamic_mask_head_matches_reference(rel_coord, num_insts, hw, mask_out_stride):
    case = MASK_CASES.index((num_insts, hw, mask_out_stride))
    group = f"dynamic_mask_{int(rel_coord)}_{case}"
    g = torch.Generator().manual_seed(2)
    n, (h, w), total = len(num_insts), hw, sum(num_insts)
    npar = sum(sum(x) for x in dynamic_param_counts(3, rel_coord))
    feats = torch.randn(n, 8, h, w, generator=g).to(DEV)
    refs = (torch.rand(1, total, 2, generator=g) * torch.tensor([w * 8.0, h * 8.0])).to(DEV)
    params = (torch.randn(1, total, npar, generator=g) * 0.3).to(DEV)
    f, r, p = (t.clone().requires_grad_(True) for t in (feats, refs, params))
    if refgolden.RECORDING:
        ddetrs = _ddetrs()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = ddetrs.DDETRSegmUni.dynamic_mask_with_coords(_holder(ddetrs, rel_coord, mask_out_stride), f, r, p,
                                                               num_insts=num_insts, mask_feat_stride=8, rel_coord=rel_coord)
    else:
        from uninext_b200 import _cabi
        lib = _cabi.load()
        before = lib.msda_launch_count()
        out = dynamic_mask_with_coords(f, r, p, num_insts, 8, rel_coord, mask_out_stride)
        assert lib.msda_launch_count() > before
    go = torch.randn(out.shape, generator=g).to(DEV)
    out.backward(go)
    if refgolden.RECORDING:
        for k, t in (("out", out), ("feats", f.grad), ("params", p.grad), ("refs", r.grad)):
            refgolden.put(group, k, t if t is not None else torch.zeros(0))
        refgolden.flush(group)
        return
    want = refgolden.load(group)
    assert refgolden.rel(out, want, "out", group) < 2e-4
    assert refgolden.rel(f.grad, want, "feats", group) < 2e-4
    assert refgolden.rel(p.grad, want, "params", group) < 2e-4
    if rel_coord:
        assert refgolden.rel(r.grad, want, "refs", group) < 1e-3     # piecewise-linear through two ReLUs: sums of many signed terms


def test_condinst_module_parameter_names_and_forward():
    torch.manual_seed(3)
    head = CondInstMaskHead(256).to(DEV)
    assert set(head.state_dict()) == {f"controller.layers.{i}.{k}" for i in range(3) for k in ("weight", "bias")}
    assert head.num_gen_params == 169 and head.controller.layers[2].out_features == 169
    hs = torch.randn(2, 30, 256, device=DEV)
    feats = torch.randn(2, 8, 10, 16, device=DEV, requires_grad=True)
    refs = torch.rand(2, 30, 2, device=DEV) * 100
    sel = [torch.tensor([1, 5, 7], device=DEV), torch.tensor([0, 29], device=DEV)]
    out = head(hs, feats, refs, sel)
    assert out.shape == (1, 5, 20, 32)
    out.square().mean().backward()
    assert feats.grad is not None and all(p.grad is not None and torch.isfinite(p.grad).all() for p in head.parameters())
