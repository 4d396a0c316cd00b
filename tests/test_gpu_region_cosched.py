"""GPU tests (-m gpu) of the region backward's launch chain (uninext_b200/csrc/msda_region.cuh): zero-fill -> grad_value
kernel -> tap kernel, chained by PDL, with grids sized so that 2 grad_value CTAs and 1 tap CTA share each SM.

At the cfg2 encoder shape (the bench's first encoder input) and on a ragged pyramid:
  - grad_loc / grad_attn are bit-identical to msda_bwd_tiled's (MSDA_KNOB_REGION_BWD = 0): each pair is one group's work
    in a fixed FMA order, whatever the grid;
  - grad_value matches the fp64 oracle within tests/test_gpu_region_bwd.py's tolerance;
  - a CUDA graph of the backward (captured without the PDL pairings) replays to the eager results;
  - one region backward counts two launches (msda_launch_count; the fill is not counted)."""
import numpy as np
import pytest
import torch

from oracle import msda_oracle

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA
    from uninext_b200.workloads import CONFIGS, make_inputs
    from tests.test_gpu_region_bwd import _encoder_inputs

DEV = "cuda"
TOL = 1e-4                  # tests/test_gpu_region_bwd.py
GV_REORDER = 2e-5           # grad_value of two runs: the same sums, reds in another order


@pytest.fixture
def lib():
    lib = _cabi.load()
    saved = {k: lib.msda_set_knob(k, -1000000) for k in (_cabi.KNOB_REGION_BWD, _cabi.KNOB_ZERO_FILL)}
    yield lib
    for k, v in saved.items():
        lib.msda_set_knob(k, v)


def _case(name):
    if name == "cfg2":
        return make_inputs(CONFIGS["cfg2"], "enc", DEV, seed=1000)
    # 1 x W, H x 1 and 1 x 1 levels next to a small 2-D one
    return _encoder_inputs([(1, 150), (60, 1), (1, 1), (12, 10)], 4, seed=31, wild_fraction=0.05)


def _args(inp):
    return (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
            inp["attention_weights"])


def _bwd(inp):
    g = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)
    torch.cuda.synchronize()
    return g


def _c_backward(inp, outs):
    v, ss, lsi, loc, at = _args(inp)
    N, S, M, D = v.shape
    gv, gl, ga = outs
    return _cabi.load().msda_backward_f32(inp["grad_output"].data_ptr(), v.data_ptr(), ss.data_ptr(), lsi.data_ptr(),
                                          loc.data_ptr(), at.data_ptr(), N, S, M, D, ss.shape[0], loc.shape[1],
                                          loc.shape[4], gv.data_ptr(), gl.data_ptr(), ga.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("case", ["cfg2", "ragged"])
def test_tap_outputs_bit_identical_to_tiled_and_grad_value_matches_oracle(lib, case):
    inp = _case(case)
    v, ss, lsi, loc, at = _args(inp)
    assert lib.msda_uses_fast_path(4, 32, ss.shape[0], loc.shape[4]) == 1
    gv, gl, ga = _bwd(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    _, gl_t, ga_t = _bwd(inp)
    assert torch.equal(gl, gl_t) and torch.equal(ga, ga_t)
    f64 = lambda t: t.detach().double().cpu().numpy()
    n = lambda t: t.detach().cpu().numpy()
    want, _, _ = msda_oracle.backward(f64(inp["grad_output"]), f64(v), n(ss), n(lsi), f64(loc), f64(at))
    err = float(np.abs(f64(gv) - want).max() / max(np.abs(want).max(), 1e-30))
    assert err < TOL, err


@pytest.mark.parametrize("case", ["cfg2", "ragged"])
def test_graph_capture_replays_to_eager(lib, case):
    inp = _case(case)
    eager = _bwd(inp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)
    scale = eager[0].abs().max().item()
    for _ in range(2):
        for t in captured:
            t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert (captured[0] - eager[0]).abs().max().item() <= GV_REORDER * scale
        assert torch.equal(captured[1], eager[1]) and torch.equal(captured[2], eager[2])


@pytest.mark.parametrize("case", ["cfg2", "ragged"])
def test_region_backward_counts_two_launches(lib, case):
    inp = _case(case)
    outs = (torch.empty_like(inp["value"]), torch.empty_like(inp["sampling_locations"]),
            torch.empty_like(inp["attention_weights"]))
    assert _c_backward(inp, outs) == 0                    # first call: per-device set-up outside the count
    torch.cuda.synchronize()
    before = lib.msda_launch_count()
    assert _c_backward(inp, outs) == 0
    torch.cuda.synchronize()
    assert lib.msda_launch_count() == before + 2
    want = _bwd(inp)
    assert torch.equal(outs[1], want[1]) and torch.equal(outs[2], want[2])
