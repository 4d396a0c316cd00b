"""Tests of msda_bwd_region (uninext_b200/csrc/msda_region.cuh) at the shipped window halo and budgets.

The halo sets how far a tile's window reaches past its region on every level, and with it which levels fit the window-row
budget and which are staged in shared memory.  Each case below is chosen for one path of the kernel: a tile whose window
reaches the window-row budget, so a level reds directly; staged levels next to an in-window level that is not staged;
the cfg2 pyramid, whose windows are staged whole in every tile; the linear-chunk mode with no window; wild and wide
offsets, whose corners fall outside the window.

A case's premise is checked on the CPU against tests/region_layout.py, which reads the kernel's constants from its
header: when a change of the halo or the budgets makes a case miss its path, the premise test fails on any machine.
On the GPU every case is compared with the CPU oracle and with msda_bwd_tiled (MSDA_KNOB_REGION_BWD = 0), which reads the
same corner values in the same FMA order: grad_loc and grad_attn must be bit-identical to it."""
import pytest
import torch

from tests.region_layout import region_constants, window_layout
from tests.test_gpu_region_bwd import TOL, _bwd, _check_vs_oracle, _encoder_inputs, lib  # noqa: F401
from uninext_b200.workloads import CONFIGS

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.workloads import make_inputs


def _budget_premise(lay):
    """An inner tile's windows fill the window-row budget after seven levels: the eighth level gets no window rows and
    reds directly; of the seven levels before it the last two are staged."""
    return any(r[7] == 0 and all(r[:7]) and s == [False] * 5 + [True] * 3 for r, s, _ in lay)


def _staged_and_unstaged_premise(lay):
    """Inner tiles stage levels 1-3 and leave level 0 in the window but over the staging budget; corner tiles stage every
    level."""
    return any(s == [False, True, True, True] and r[0] > 0 for r, s, _ in lay) and any(all(s) for _, s, _ in lay)


def _two_levels_staged_premise(lay):
    """A tile stages only its last two levels and reads the first two, in the window, from global memory.  Staging only the
    last level cannot happen at this halo: a level has at most (kRegionEdge + 2 kRegionHalo)^2 = 144 window rows, so any
    two levels fit the 384-row staging budget."""
    return any(s == [False, False, True, True] and r[0] > 0 and r[1] > 0 for r, s, _ in lay)


def _all_staged_premise(lay):
    """Every tile stages the window of every level, so every in-window corner is read from shared memory."""
    return all(all(r) and all(s) for r, s, _ in lay)


# name -> (level table, premise on its window layout, encoder-input arguments)
CASES = {
    "window_budget": ([(32, 32)] * 8, _budget_premise, dict(N=1, P=2, seed=41, wild_fraction=0.05)),
    "staged_and_unstaged": ([(48, 48), (48, 48), (36, 36), (36, 36)], _staged_and_unstaged_premise,
                            dict(N=1, seed=31, wild_fraction=0.05)),
    "two_levels_staged": ([(24, 24)] * 4, _two_levels_staged_premise, dict(N=1, seed=32, jitter_px=4.0)),
    "cfg2_all_staged": ([tuple(s) for s in CONFIGS["cfg2"].shapes], _all_staged_premise, dict(N=1, seed=42)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_region_case_premise(name):
    shapes, premise, _ = CASES[name]
    assert premise(window_layout(shapes)), (name, region_constants(), premise.__doc__)


def test_two_levels_always_fit_the_staging_budget():
    """The reason _two_levels_staged_premise gives for not testing a tile that stages only its last level."""
    c = region_constants()
    assert 2 * (c["kRegionEdge"] + 2 * c["kRegionHalo"]) ** 2 <= c["kRegionStageRows"]


def _check_vs_tiled(lib, inp):  # noqa: F811
    gv, gl, ga = _check_vs_oracle(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, 0)
    tv, tl, ta = _bwd(inp)
    lib.msda_set_knob(_cabi.KNOB_REGION_BWD, -1)
    assert torch.equal(gl, tl) and torch.equal(ga, ta)
    assert (gv - tv).abs().max().item() <= TOL * tv.abs().max().item()


def _check_case(lib, name):  # noqa: F811
    shapes, premise, kw = CASES[name]
    assert premise(window_layout(shapes)), (name, region_constants())
    _check_vs_tiled(lib, _encoder_inputs(shapes, **kw))


@pytest.mark.gpu
def test_window_reaches_the_row_budget(lib):  # noqa: F811
    _check_case(lib, "window_budget")


@pytest.mark.gpu
def test_staged_and_unstaged_in_window_levels(lib):  # noqa: F811
    _check_case(lib, "staged_and_unstaged")


@pytest.mark.gpu
def test_last_two_levels_staged(lib):  # noqa: F811
    _check_case(lib, "two_levels_staged")


@pytest.mark.gpu
def test_cfg2_staged_level_layout(lib):  # noqa: F811
    _check_case(lib, "cfg2_all_staged")


@pytest.mark.gpu
def test_linear_chunks_have_no_staged_window(lib):  # noqa: F811
    """Lq == S, but S has rows past the pyramid: the kernel runs linear chunks of pairs with no window and no staging."""
    _check_vs_tiled(lib, _encoder_inputs([(20, 20), (10, 10)], 2, seed=34, S=520))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["wild", "wide"])
def test_wild_and_wide_offsets(lib, variant):  # noqa: F811
    """Taps anywhere in the image (wild) or far from the query (wide): many corners fall outside the window and red
    directly, next to the entries of the in-window corners."""
    kw = {"wild": {"wild_fraction": 0.2}, "wide": {"jitter_px": 12.0}}[variant]
    _check_vs_tiled(lib, make_inputs(CONFIGS["cfg1"], "enc", "cuda", seed=43, **kw))
