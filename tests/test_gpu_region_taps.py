"""GPU tests (-m gpu): the region backward's grad_loc / grad_attn come from msda_bwd_tiled's own tap code, so they are
bit-identical to the msda_bwd_tiled route (MSDA_KNOB_REGION_BWD = 0) -- with TMA-staged taps (L*P % 4 == 0, the bench's
cfg2 encoder call) and with __ldg taps (L*P % 4 != 0).  grad_value is summed in another order and is compared within
the suite's tolerance."""
import pytest
import torch

from tests.test_gpu_region_bwd import TOL, _bwd, _check_vs_oracle, _encoder_inputs, _region_bwd, lib  # noqa: F401

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.workloads import CONFIGS, make_inputs


def _tiled_bwd(lib, inp):  # noqa: F811
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    try:
        return _bwd(inp)
    finally:
        lib.msda_set_knob(_cabi.KNOB_REGION_BWD, -1)


def _check_bit_identical(lib, got, inp):  # noqa: F811
    tv, tl, ta = _tiled_bwd(lib, inp)
    gv, gl, ga = got
    assert torch.equal(gl, tl) and torch.equal(ga, ta)
    assert (gv - tv).abs().max().item() <= TOL * tv.abs().max().item()


@pytest.mark.parametrize("P", [3, 5])
def test_ldg_tap_pass_matches_tiled(lib, P):  # noqa: F811
    """Three levels and P = 3 or 5: L*P = 9 or 15 taps, not a multiple of 4, so the tap pass reads them with __ldg."""
    shapes = [(48, 48), (24, 24), (12, 12)]
    inp = _encoder_inputs(shapes, 1, P=P, seed=51, wild_fraction=0.05)
    assert (len(shapes) * P) % 4 != 0
    _check_bit_identical(lib, _check_vs_oracle(inp), inp)


def test_cfg2_matches_tiled_bit_for_bit(lib):  # noqa: F811
    """The bench's first cfg2 encoder call (TMA-staged taps)."""
    inp = make_inputs(CONFIGS["cfg2"], "enc", "cuda", seed=1000)
    _check_bit_identical(lib, _region_bwd(inp), inp)
