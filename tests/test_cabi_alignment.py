"""CPU test: the C-ABI entry points whose kernels use vector loads / stores reject pointers without the alignment those
accesses need (MSDA_E_BADARG) before they touch the device.  A contiguous view with a storage offset is only 4-byte
aligned; a float4 access through it is a misaligned-address fault, so the check has to happen on the host.

The calls use fake device addresses and valid sizes.  Without a GPU an aligned call gets past the argument check and
then fails in the CUDA runtime (any code but MSDA_E_BADARG); a misaligned one must stop at the check.  On a machine with
a GPU the aligned calls would launch kernels on the fake addresses, so the file is skipped there
(tests/test_gpu_unaligned_operands.py makes the same checks with real buffers)."""
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="calls with fake device addresses; the GPU variant is test_gpu_unaligned_operands.py")

BADARG = -1                                     # MSDA_E_BADARG
BASE = 0x7F0000000000                           # fake, 4 KiB-aligned device addresses, one 1 MiB slot per operand


def _fake_ptrs(names, bad=None, off=4):
    return {n: BASE + (i << 20) + (off if n == bad else 0) for i, n in enumerate(names)}


# name -> (pointer operands in argument order, alignment each guarded operand needs, build the argument list)
R, M, L, P, ROWS, COLS = 6, 2, 2, 3, 10, 256
CASES = {
    "msda_prologue_forward_f32": (
        ("proj", "ref", "shapes", "loc", "attn"), {"loc": 8},
        lambda p: (p["proj"], p["ref"], p["shapes"], R, M, L, P, 2, p["loc"], p["attn"], None)),
    "msda_prologue_backward_f32": (
        ("grad_loc", "grad_attn", "attn", "ref", "shapes", "grad_proj"), {"grad_loc": 8},
        lambda p: (p["grad_loc"], p["grad_attn"], p["attn"], p["ref"], p["shapes"], R, M, L, P, 4, p["grad_proj"], None)),
    "msda_colsum_f32": (
        ("x", "out"), {"x": 16, "out": 16},
        lambda p: (p["x"], ROWS, COLS, p["out"], None)),
    "msda_relu_backward_colsum_f32": (
        ("g", "y", "g2", "colsum"), {"g": 16, "y": 16, "g2": 16, "colsum": 16},
        lambda p: (p["g"], p["y"], ROWS, COLS, p["g2"], p["colsum"], None)),
    "msda_add_layernorm_forward_f32": (
        ("a", "b", "gamma", "beta", "z", "y", "mean", "rstd"),
        {"a": 16, "b": 16, "gamma": 16, "beta": 16, "z": 16, "y": 16},
        lambda p: (p["a"], p["b"], p["gamma"], p["beta"], ROWS, COLS, 1e-5, p["z"], p["y"], p["mean"], p["rstd"], None)),
    "msda_layernorm_backward_f32": (
        ("dy", "z", "gamma", "mean", "rstd", "dz", "dgamma", "dbeta"),
        {"dy": 16, "z": 16, "gamma": 16, "dz": 16, "dgamma": 16, "dbeta": 16},
        lambda p: (p["dy"], p["z"], p["gamma"], p["mean"], p["rstd"], ROWS, COLS, p["dz"], p["dgamma"], p["dbeta"], None)),
}
GUARDED = [(fn, op) for fn, (_, need, _) in CASES.items() for op in need]


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    return _cabi.load(build.build())


@pytest.mark.parametrize("fn", sorted(CASES))
def test_aligned_call_passes_the_argument_check(lib, fn):
    names, _, args = CASES[fn]
    assert getattr(lib, fn)(*args(_fake_ptrs(names))) != BADARG


@pytest.mark.parametrize("fn,operand", GUARDED)
def test_misaligned_operand_is_rejected(lib, fn, operand):
    names, need, args = CASES[fn]
    assert getattr(lib, fn)(*args(_fake_ptrs(names, bad=operand, off=4))) == BADARG, f"{fn}: {operand} 4 bytes off"
    if need[operand] == 16:                     # 8 bytes off a 16-byte boundary is still misaligned for a float4
        assert getattr(lib, fn)(*args(_fake_ptrs(names, bad=operand, off=8))) == BADARG, f"{fn}: {operand} 8 bytes off"
    else:                                       # a float2 needs 8 bytes, not 16
        assert getattr(lib, fn)(*args(_fake_ptrs(names, bad=operand, off=8))) != BADARG, f"{fn}: {operand} 8 bytes off"


def test_add_layernorm_forward_checks_b_and_z_only_when_given(lib):
    fn = lib.msda_add_layernorm_forward_f32
    p = _fake_ptrs(("a", "gamma", "beta", "y", "mean", "rstd", "z"))
    call = lambda a, z: fn(a, None, p["gamma"], p["beta"], ROWS, COLS, 1e-5, z, p["y"], p["mean"], p["rstd"], None)
    assert call(p["a"], None) != BADARG                         # no b, no z: nothing else to check
    assert call(p["a"], p["z"]) != BADARG                       # z without b is written too (it equals a) ...
    assert call(p["a"], p["z"] + 4) == BADARG                   # ... so it must be aligned as well
    assert call(p["a"] + 4, None) == BADARG
