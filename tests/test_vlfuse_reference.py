"""The early-fusion block against the reference's own BiAttentionBlockForCheckpoint (tests/golden/reference/vlfuse_*.npz,
recorded by tests/golden/make_vlfuse_golden.py): the torch composition on the CPU, the fused module on the GPU."""
import os

import numpy as np
import pytest
import torch

from tests import vlfuse_case as vc
from uninext_b200.modules.vl_fusion import BiAttentionBlock

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")


def _block():
    return BiAttentionBlock(vc.V_DIM, vc.L_DIM, vc.EMBED, vc.HEADS, dropout=0.1, drop_path=0.0, init_values=1.0 / 6)


def _compare(name, device, tol):
    want = dict(np.load(os.path.join(GOLDEN, f"vlfuse_{name}.npz")))
    keys = list(want.pop("state_dict_keys"))
    block = _block()
    assert sorted(block.state_dict().keys()) == keys
    got = vc.run(block, name, device)
    assert set(got) == set(want)
    for k, w in want.items():
        err = np.abs(got[k].astype(np.float64) - w).max() / max(np.abs(w).max(), 1e-30)
        assert err < tol, (name, k, err)


@pytest.mark.parametrize("name", sorted(vc.CASES))
def test_torch_composition_matches_reference_block(name):
    torch.manual_seed(0)
    _compare(name, "cpu", 2e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(vc.CASES))
def test_fused_module_matches_reference_block(name):
    _compare(name, "cuda", 2e-4)
