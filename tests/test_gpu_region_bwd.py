"""GPU tests (-m gpu) of the region backward (uninext_b200/csrc/msda_region.cuh), the default fp32 backward of encoder
self-attention (D = 32, L*P <= 16, Lq == S, large launches).  Every path of the kernel is compared with the CPU oracle:
in-window corners summed on chip, corners outside the window (wide offsets, wild taps), queries past the stash, in-window
levels that are not staged, and a level table that does not tile [0, S) (linear order, no window); each comparison
also checks that msda_bwd_region ran.  tests/test_gpu_region_halo.py holds the cases chosen for one window layout each.
MSDA_KNOB_REGION_BWD = 0 selects msda_bwd_tiled for the A/B comparisons."""
import time

import numpy as np
import pytest
import torch

from oracle import msda_oracle

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA
    from uninext_b200.workloads import CONFIGS, encoder_reference_points, make_inputs, ring_offsets

DEV = "cuda"
TOL = 1e-4


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
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else got
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _check_vs_oracle(inp):
    n = lambda t: t.detach().cpu().numpy()
    f64 = lambda t: t.detach().double().cpu().numpy()
    a = _args(inp)
    gv_t, _, ga_t = msda_oracle.backward(f64(inp["grad_output"]), f64(a[0]), n(a[1]), n(a[2]), f64(a[3]), f64(a[4]))
    _, gl32, _ = msda_oracle.backward(n(inp["grad_output"]), n(a[0]), n(a[1]), n(a[2]), n(a[3]), n(a[4]))
    gv, gl, ga = _region_bwd(inp)
    assert _maxerr(gv, gv_t) < TOL
    assert _maxerr(ga, ga_t) < TOL
    assert _maxerr(gl, gl32.astype(np.float64)) < 2 * TOL        # same rounding sequence for the pixel coordinate
    return gv, gl, ga


def _kernel_names(fn):
    """Names of the events recorded while fn runs.  Now and then the profiler records a window's launches but delivers
    none of its kernel records, so a window without any msda kernel is profiled again, up to four times (every fn given
    here launches one)."""
    for _ in range(4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=DEV).add_(1)          # the profiler can also lose the first kernels of its window
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        if any("msda_" in n for n in names):
            break
        time.sleep(0.5)
    return names


def _region_bwd(inp):
    """_bwd, checking that msda_bwd_region ran.  _kernel_names may run the backward again when the profiler drops a
    window's kernel records; the gradients returned are those of the last run."""
    res = []

    def run():
        res[:] = _bwd(inp)

    names = _kernel_names(run)
    assert any("msda_bwd_region" in k for k in names), names
    return res


def _encoder_inputs(shapes, N, M=8, D=32, P=4, seed=0, jitter_px=2.0, wild_fraction=0.0, S=None, lsi=None,
                    dtype=torch.float32):
    """Encoder self-attention inputs (query i = pixel i, ring offsets + jitter) for an arbitrary level table; `dtype` is
    that of value and grad_output (locations and weights are fp64 with fp64 values, fp32 otherwise)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    L = len(shapes)
    ss = torch.tensor(shapes, dtype=torch.long, device=DEV)
    if lsi is None:
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    else:
        lsi = torch.tensor(lsi, dtype=torch.long, device=DEV)
    npix = sum(h * w for h, w in shapes)
    S = npix if S is None else S
    ref = encoder_reference_points(shapes, DEV)
    if S > npix:                                   # extra rows past the pyramid: queries anywhere
        ref = torch.cat((ref, torch.rand(S - npix, 2, generator=g, device=DEV)), 0)
    wh = torch.tensor([(w, h) for h, w in shapes], device=DEV, dtype=torch.float32)
    off = ring_offsets(M, L, P, DEV) + jitter_px * torch.randn(N, S, M, L, P, 2, generator=g, device=DEV)
    loc = ref.view(1, S, 1, 1, 1, 2) + off / wh.view(1, 1, 1, L, 1, 2)
    if wild_fraction > 0:
        wild = torch.rand(loc.shape[:-1], generator=g, device=DEV) < wild_fraction
        loc = torch.where(wild[..., None], torch.rand(loc.shape, generator=g, device=DEV) * 2.0 - 0.5, loc)
    attn = torch.softmax(torch.randn(N, S, M, L * P, generator=g, device=DEV), -1).view(N, S, M, L, P)
    aux = torch.float64 if dtype == torch.float64 else torch.float32
    return dict(value=torch.randn(N, S, M, D, generator=g, device=DEV).to(dtype), spatial_shapes=ss,
                level_start_index=lsi, sampling_locations=loc.to(aux).contiguous(),
                attention_weights=attn.to(aux).contiguous(),
                grad_output=torch.randn(N, S, M * D, generator=g, device=DEV).to(dtype))


@pytest.mark.parametrize("cfg", ["cfg1", "cfg4"])
@pytest.mark.parametrize("variant", ["bench", "wild", "wide"])
def test_region_backward_vs_oracle(lib, cfg, variant):
    kw = {"bench": {}, "wild": {"wild_fraction": 0.1}, "wide": {"jitter_px": 20.0}}[variant]
    inp = make_inputs(CONFIGS[cfg], "enc", DEV, seed=21, **kw)
    _check_vs_oracle(inp)


def test_region_kernel_is_the_default_for_encoder_fp32(lib):
    inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=22)
    names = _kernel_names(lambda: _bwd(inp))
    assert any("msda_bwd_region" in n for n in names), names
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    names = _kernel_names(lambda: _bwd(inp))
    assert not any("msda_bwd_region" in n for n in names) and any("msda_bwd_tiled" in n for n in names), names


# 1 x W, H x 1 and 1 x 1 levels; four equal-size levels (256 queries per inner tile, past the 96-query stash; level 0,
# and in the inner tiles level 1 too, in the window but not staged); five equal-size levels, P = 3 (320 queries per
# tile; levels 0 and 1 in the window but not staged)
@pytest.mark.parametrize("shapes,N", [([(1, 150), (60, 1), (1, 1), (12, 10)], 4), ([(24, 24)] * 4, 1),
                                      ([(16, 20)] * 5, 1)])
def test_region_backward_ragged_level_tables(lib, shapes, N):
    P = 4 if len(shapes) <= 4 else 3
    inp = _encoder_inputs(shapes, N, P=P, seed=23, wild_fraction=0.05)
    assert _cabi.load().msda_uses_fast_path(4, 32, len(shapes), P) == 1
    _check_vs_oracle(inp)


def test_region_backward_table_not_tiling_rows(lib):
    """Lq == S, but S has rows past the pyramid: the kernel runs linear chunks of pairs with no window."""
    inp = _encoder_inputs([(20, 20), (10, 10)], 2, seed=24, S=520)
    _check_vs_oracle(inp)
    inp = _encoder_inputs([(20, 20), (10, 10)], 2, seed=25, lsi=[100, 0])        # levels out of order
    _check_vs_oracle(inp)


def test_region_backward_writes_every_tap_once(lib):
    """grad_loc / grad_attn pre-filled with NaN through the C ABI: every tap is overwritten."""
    inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=26, wild_fraction=0.1)
    v, ss, lsi, loc, at = _args(inp)
    go = inp["grad_output"]
    N, S, M, D = v.shape
    gv = torch.full_like(v, float("nan"))
    gl = torch.full_like(loc, float("nan"))
    ga = torch.full_like(at, float("nan"))
    code = _cabi.load().msda_backward_f32(go.data_ptr(), v.data_ptr(), ss.data_ptr(), lsi.data_ptr(), loc.data_ptr(),
                                         at.data_ptr(), N, S, M, D, ss.shape[0], loc.shape[1], loc.shape[4], gv.data_ptr(),
                                         gl.data_ptr(), ga.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert code == 0
    assert not gv.isnan().any() and not gl.isnan().any() and not ga.isnan().any()
    want = _region_bwd(inp)
    assert torch.equal(gl, want[1]) and torch.equal(ga, want[2])


def test_region_matches_tiled_at_cfg2(lib):
    inp = make_inputs(CONFIGS["cfg2"], "enc", DEV, seed=1000)
    got = _region_bwd(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    want = _bwd(inp)
    for g, w in zip(got, want):
        assert (g - w).abs().max().item() <= TOL * w.abs().max().item()


def test_region_zero_fill_modes_and_graph_capture(lib):
    inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=27, wild_fraction=0.05)
    lib.msda_set_knob(_cabi.KNOB_ZERO_FILL, 0)
    ref = _region_bwd(inp)
    scale = ref[0].abs().max().item()
    for mode in (1, 2):
        lib.msda_set_knob(_cabi.KNOB_ZERO_FILL, mode)
        for _ in range(3):
            junk = torch.full((inp["value"].numel() + 64,), 7.0, device=DEV)      # dirty the allocator's blocks
            del junk
            gv, gl, ga = _bwd(inp)
            assert (gv - ref[0]).abs().max().item() <= 2e-5 * scale, mode
            assert torch.equal(gl, ref[1]) and torch.equal(ga, ref[2]), mode
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64)
    for _ in range(3):
        got[0].fill_(3.0)
        g.replay()
    torch.cuda.synchronize()
    assert (got[0] - ref[0]).abs().max().item() <= 2e-5 * scale
    assert torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])
