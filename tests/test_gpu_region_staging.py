"""GPU tests (-m gpu) of the staged value window of msda_bwd_region (uninext_b200/csrc/msda_region.cuh).

Per tile the kernel copies the window rows of its last levels into shared memory, from the last level down while they fit
kRegionStageRows, and reads in-window corners of those levels from there.  Each case below is chosen for one path, which
_window_layout (the kernel's tile geometry restated) confirms first: a staged level, an in-window level that is not
staged because it is over the staging budget, a level over the window-row budget, and the linear-chunk mode with no window.
Every case is compared with the CPU oracle and with msda_bwd_tiled (MSDA_KNOB_REGION_BWD = 0): the corner values are the
same wherever they are read from, so grad_loc and grad_attn must be bit-identical to the tiled kernel's."""
import pytest
import torch

from tests.test_gpu_region_bwd import TOL, _bwd, _check_vs_oracle, _encoder_inputs, lib  # noqa: F401

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi

R, HALO, WIN_ROWS, STAGE_ROWS = 8, 4, 1024, 384          # kRegionEdge, kRegionHalo, kRegionWinRows, kRegionStageRows


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


def test_staged_and_unstaged_in_window_levels(lib):  # noqa: F811
    """Inner tiles stage levels 1-3 and leave level 0 over the staging budget (the cfg2 layout, scaled down); corner
    tiles stage every level."""
    shapes = [(40, 64), (20, 32), (10, 16), (5, 8)]
    lay = _window_layout(shapes)
    assert any(s == [False, True, True, True] and r[0] > 0 for r, s in lay) and any(all(s) for _, s in lay)
    _check_vs_tiled(lib, _encoder_inputs(shapes, 2, seed=31, wild_fraction=0.05))


def test_only_the_last_level_fits_the_staging_budget(lib):  # noqa: F811
    """Four equal-size levels: the last level's 256 rows are staged, the third would take the tile past the budget."""
    shapes = [(24, 24)] * 4
    lay = _window_layout(shapes)
    assert any(s == [False, False, False, True] and r[2] > 0 for r, s in lay)
    _check_vs_tiled(lib, _encoder_inputs(shapes, 1, seed=32, jitter_px=4.0))


def test_level_over_the_window_budget_with_staging(lib):  # noqa: F811
    """Five equal-size levels: inner tiles give the last level no window rows (window-row budget) and stage the level
    before it."""
    shapes = [(24, 24)] * 5
    lay = _window_layout(shapes)
    assert any(r[4] == 0 and s == [False, False, False, True, True] and r[3] > 0 for r, s in lay)
    _check_vs_tiled(lib, _encoder_inputs(shapes, 1, P=3, seed=33, wild_fraction=0.05))


def test_linear_chunks_have_no_staged_window(lib):  # noqa: F811
    """Rows past the pyramid: the kernel runs linear chunks of pairs with no window and no staging."""
    _check_vs_tiled(lib, _encoder_inputs([(20, 20), (10, 10)], 2, seed=34, S=520))
