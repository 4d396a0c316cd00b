"""GPU tests (-m gpu) of msda_bwd_region (uninext_b200/csrc/msda_region.cuh) at the shipped window halo.

The halo sets how far a tile's window reaches past its region on every level, and with it which levels fit the window-row
budget and which are staged in shared memory.  _window_layout restates the kernel's tile geometry at the shipped
kRegionEdge / kRegionHalo and confirms each case's premise first: a tile whose window reaches the window-row budget, so
a level reds directly; the cfg2 pyramid, whose windows are staged whole in every tile; wild and wide offsets, whose
corners fall outside the window.  Every case is compared with the CPU oracle and with msda_bwd_tiled (MSDA_KNOB_REGION_BWD = 0), which reads the
same corner values in the same FMA order: grad_loc and grad_attn must be bit-identical to it."""
import pytest
import torch

from tests.test_gpu_region_bwd import TOL, _bwd, _check_vs_oracle, _encoder_inputs, lib  # noqa: F401

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.workloads import CONFIGS, make_inputs

R, HALO, WIN_ROWS, STAGE_ROWS = 8, 2, 1024, 384          # kRegionEdge, kRegionHalo, kRegionWinRows, kRegionStageRows


def _window_layout(shapes):
    """[(rows per level, staged per level)] over the tiles of a level table that tiles [0, S), as the kernel lays them out."""
    href, wref = max(h for h, _ in shapes), max(w for _, w in shapes)
    out = []
    for ry in range(-(-href // R)):
        for rx in range(-(-wref // R)):
            rows, nw = [], 0
            for h, w in shapes:
                wy0, wy1 = max(0, ry * R * h // href - HALO), min(h, -(-(ry + 1) * R * h // href) + HALO)
                wx0, wx1 = max(0, rx * R * w // wref - HALO), min(w, -(-(rx + 1) * R * w // wref) + HALO)
                n = (wy1 - wy0) * (wx1 - wx0)
                n = 0 if nw + n > WIN_ROWS else n
                rows.append(n)
                nw += n
            staged, tail = [False] * len(shapes), 0
            for lvl in reversed(range(len(shapes))):
                if tail + rows[lvl] > STAGE_ROWS:
                    break
                tail += rows[lvl]
                staged[lvl] = True
            out.append((rows, staged))
    return out


def _check_vs_tiled(lib, inp):  # noqa: F811
    gv, gl, ga = _check_vs_oracle(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    tv, tl, ta = _bwd(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, -1)
    assert torch.equal(gl, tl) and torch.equal(ga, ta)
    assert (gv - tv).abs().max().item() <= TOL * tv.abs().max().item()


def test_window_reaches_the_row_budget(lib):  # noqa: F811
    """Eight equal-size levels: an inner tile's windows fill the 1024-row budget after seven levels, so the eighth level
    gets no window rows and reds directly; the seven levels before it are in the window, the last two of them staged."""
    shapes = [(32, 32)] * 8
    lay = _window_layout(shapes)
    assert any(r[7] == 0 and all(r[:7]) and s == [False] * 5 + [True] * 3 for r, s in lay)
    _check_vs_tiled(lib, _encoder_inputs(shapes, 1, P=2, seed=41, wild_fraction=0.05))


def test_cfg2_staged_level_layout(lib):  # noqa: F811
    """The cfg2 pyramid: every tile stages the window of all four levels, so every in-window corner is read from shared
    memory."""
    shapes = [tuple(s) for s in CONFIGS["cfg2"].shapes]
    lay = _window_layout(shapes)
    assert all(all(r) and all(s) for r, s in lay)
    _check_vs_tiled(lib, _encoder_inputs(shapes, 1, seed=42))


@pytest.mark.parametrize("variant", ["wild", "wide"])
def test_wild_and_wide_offsets(lib, variant):  # noqa: F811
    """Taps anywhere in the image (wild) or far from the query (wide): many corners fall outside the narrower window and
    red directly, next to the entries of the in-window corners."""
    kw = {"wild": {"wild_fraction": 0.2}, "wide": {"jitter_px": 12.0}}[variant]
    _check_vs_tiled(lib, make_inputs(CONFIGS["cfg1"], "enc", "cuda", seed=43, **kw))
