"""GPU tests (-m gpu) of the region backward as two kernels (uninext_b200/csrc/msda_region.cuh): msda_bwd_region, the tap
pass (grad_loc / grad_attn), and msda_region_grad_value_pass, the grad_value pass, launched as a PDL secondary of the
tap kernel, which waits for the zero-fill as its last statement.

For a cfg2 encoder input and a level table that does not tile [0, S) (linear chunks, no window):
  - both kernels run, and nothing else of the op's kernel families;
  - grad_value, grad_loc and grad_attn match the CPU oracle and the msda_bwd_tiled route (MSDA_KNOB_REGION_BWD = 0);
    grad_loc and grad_attn bit for bit;
  - the same holds for every zero-fill mode (memset, fill kernel, fill kernel as PDL primary) and in a captured CUDA
    graph, whose replays run the kernels in plain stream order;
  - one backward counts the two launches."""
import numpy as np
import pytest
import torch

from oracle import msda_oracle
from tests.test_gpu_region_bwd import _encoder_inputs, _kernel_names

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA
    from uninext_b200.workloads import CONFIGS, make_inputs

DEV = "cuda"
TOL = 1e-4
TAP, GV = "msda_bwd_region<8, 2>", "msda_region_grad_value_pass<8, 2>"


@pytest.fixture
def lib():
    lib = _cabi.load()
    saved = {k: lib.msda_set_knob(k, -1000000) for k in (_cabi.KNOB_REGION_BWD, _cabi.KNOB_ZERO_FILL)}
    yield lib
    for k, v in saved.items():
        lib.msda_set_knob(k, v)


def _args(inp):
    return (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
            inp["attention_weights"])


def _bwd(inp):
    g = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)
    torch.cuda.synchronize()
    return g


def _maxerr(got, want):
    got = got.detach().double().cpu().numpy()
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _cfg2():
    return make_inputs(CONFIGS["cfg2"], "enc", DEV, seed=1000)


def _linear():
    return _encoder_inputs([(20, 20), (10, 10)], 2, seed=31, S=520, wild_fraction=0.05)


CASES = {"cfg2": _cfg2, "linear": _linear}


def _region_run(inp):
    """The default backward, checking that exactly the two region kernels of the op ran."""
    res = []

    def run():
        res[:] = _bwd(inp)

    names = _kernel_names(run)
    ours = {n for n in names if "msda_" in n and "zero_fill" not in n}
    assert any(TAP in n for n in ours) and any(GV in n for n in ours), ours
    assert all(TAP in n or GV in n for n in ours), ours
    return res


@pytest.mark.parametrize("case", sorted(CASES))
def test_two_kernels_match_oracle_and_tiled_route(lib, case):
    inp = CASES[case]()
    gv, gl, ga = _region_run(inp)
    n = lambda t: t.detach().cpu().numpy()
    f64 = lambda t: t.detach().double().cpu().numpy()
    a = _args(inp)
    gv_t, _, ga_t = msda_oracle.backward(f64(inp["grad_output"]), f64(a[0]), n(a[1]), n(a[2]), f64(a[3]), f64(a[4]))
    _, gl32, _ = msda_oracle.backward(n(inp["grad_output"]), n(a[0]), n(a[1]), n(a[2]), n(a[3]), n(a[4]))
    assert _maxerr(gv, gv_t) < TOL
    assert _maxerr(ga, ga_t) < TOL
    assert _maxerr(gl, gl32.astype(np.float64)) < 2 * TOL
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    want = _bwd(inp)
    assert (gv - want[0]).abs().max().item() <= TOL * want[0].abs().max().item()
    assert torch.equal(gl, want[1]) and torch.equal(ga, want[2])


@pytest.mark.parametrize("case", sorted(CASES))
def test_zero_fill_modes_and_graph_capture(lib, case):
    inp = CASES[case]()
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    ref = _bwd(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, -1)
    scale = ref[0].abs().max().item()
    for mode in (0, 1, 2):
        lib.msda_set_knob(_cabi.KNOB_ZERO_FILL, mode)
        for _ in range(3):
            junk = torch.full((inp["value"].numel() + 64,), 7.0, device=DEV)      # dirty the allocator's blocks
            del junk
            gv, gl, ga = _bwd(inp)
            assert (gv - ref[0]).abs().max().item() <= TOL * scale, mode
            assert torch.equal(gl, ref[1]) and torch.equal(ga, ref[2]), mode
    lib.msda_set_knob(_cabi.KNOB_ZERO_FILL, 2)
    _bwd(inp)                                          # warm-up outside the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)
    for _ in range(3):
        for t in got:
            t.fill_(3.0)
        g.replay()
        torch.cuda.synchronize()
        assert (got[0] - ref[0]).abs().max().item() <= TOL * scale
        assert torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])


def test_backward_counts_both_launches(lib):
    inp = _cfg2()
    _bwd(inp)
    before = lib.msda_launch_count()
    _bwd(inp)
    assert lib.msda_launch_count() - before == 2
