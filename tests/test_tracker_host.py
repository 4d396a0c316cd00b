"""CPU tests of the IDOL tracker's host side: the restatement of tests/tracker_case.py reproduces the reference's goldens
(tests/golden/tracker/, made by tests/golden/make_tracker_golden.py) exactly; include/msda_tracker.h, the ctypes table
and the library's exports agree; msda_idol_workspace / msda_idol_match_f32 reject bad arguments before they touch a
pointer or the device; IDOLTracker's constructor and inputs are checked."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from tests import tracker_case as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "msda_tracker.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "tracker")
BADARG = -1


@pytest.mark.parametrize("flag_index", range(len(tc.FLAG_SETS)))
def test_restatement_reproduces_the_reference_goldens(flag_index):
    flags = tc.FLAG_SETS[flag_index]
    z = np.load(os.path.join(GOLDEN, "lm{}_fw{}_tw{}.npz".format(*(int(x) for x in flags))))
    seq = tc.golden_sequence(flag_index)
    assert str(z["checksum"]) == tc.checksum(seq) and int(z["frames"]) == len(seq) >= 14
    ref = tc.Restated(**tc.settings(flags))
    seen = set()
    for f, (scores, masks, embeds) in enumerate(seq):
        assert scores.shape[0] <= 48 and masks.shape[2:] == (40, 72)
        keep, ids = ref.step(scores, masks[:, 0], embeds, f)
        assert keep == z[f"{f}/keep"].tolist() and ids == z[f"{f}/ids"].tolist(), f
        assert [3 * r + 7 for r in keep] == z[f"{f}/indices"].tolist()
        cols = sorted(ref.tracks)
        assert cols == z[f"{f}/track_ids"].tolist()
        for c, k in enumerate(cols):
            v = ref.tracks[k]
            ln = len(v["long_embed"])
            assert (v["last_frame"], v["exist_frame"], ln) == (z[f"{f}/last_frame"][c], z[f"{f}/exist_frame"][c],
                                                               z[f"{f}/ring_len"][c])
            assert np.array_equal(v["embed"].numpy(), z[f"{f}/embed"][c])
            assert np.array_equal(torch.stack(v["long_embed"]).numpy(), z[f"{f}/long_embed"][c, :ln])
            assert np.array_equal(torch.stack(v["long_score"]).numpy(), z[f"{f}/long_score"][c, :ln])
            seen.add(("ring full", ln == 3))
        seen.update(("id", min(i, 0)) for i in ids)
        seen.add(("empty", not cols))
    # the sequences reach matches / new ids, backdrops, rows left at -2, full rings, expiry of every tracklet, and both
    # sides of the frame-weight branch
    assert {("id", 0), ("id", -1), ("id", -2), ("ring full", True), ("empty", True)} <= seen
    assert min(ref.margins) >= 1e-4
    if flags[1]:
        assert ref.weighted_rows >= 1


def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): len([a for a in m.group(2).split(",") if a.strip()])
            for m in re.finditer(r"\bint\s+(msda_\w+)\s*\(([^;{]*)\)\s*;", text)}


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.tracker()


def test_header_ctypes_table_and_exports_agree(lib):
    from uninext_b200 import _cabi
    decl = _declared()
    assert set(decl) == set(_cabi.TRACKER_SIGNATURES) and len(decl) == 2
    assert not set(decl) & (set(_cabi.SIGNATURES) | set(_cabi.TRACKPOST_SIGNATURES))
    for name, nargs in decl.items():
        assert len(_cabi.TRACKER_SIGNATURES[name][1]) == nargs, name
        assert _cabi.entry(name).argtypes == _cabi.TRACKER_SIGNATURES[name][1], name
    text = open(HEADER).read()
    consts = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+MSDA_IDOL_(\w+)\s+(\d+)\b", text)}
    assert consts["LONG_MATCH"] == _cabi.IDOL_LONG_MATCH and consts["FRAME_WEIGHT"] == _cabi.IDOL_FRAME_WEIGHT
    assert consts["TEMPORAL_WEIGHT"] == _cabi.IDOL_TEMPORAL_WEIGHT and consts["STATE_FLAGS"] == 2
    assert consts["OVERFLOW"] == _cabi.IDOL_OVERFLOW and consts["BAD_ROW"] == _cabi.IDOL_BAD_ROW
    assert lib.msda_abi_version() == 11 == _cabi.ABI_VERSION                       # msda_b200.h is unchanged


# (n_cap, max_tracklets, dim, h, w)
BAD_SIZES = [(0, 8, 32, 40, 72), (1025, 8, 32, 40, 72), (10, 0, 32, 40, 72), (10, 1025, 32, 40, 72),
             (10, 8, 0, 40, 72), (10, 8, 32, 0, 72), (10, 8, 32, 40, 0), (10, 8, 32, 4096, 4096)]


def _args(dims=(10, 8, 32, 40, 72), ws_bytes=1 << 40, null=None, ws=256, memory_len=3, frames=10, flags=7, n_src=10):
    """Pointer slots in order: masks, embeds, scores, rows, count (0-4), temporal_weights (5), state, embed, ring_embed,
    ring_score, ids, tracked, tracked_count (6-12), workspace (13).  Fake addresses: never dereferenced when a check
    fails."""
    n_cap, T, dim, h, w = dims
    p = [ctypes.c_void_p(256)] * 14
    p[13] = ctypes.c_void_p(ws)
    if null is not None:
        p[null] = None
    return (*p[:5], n_src, n_cap, h, w, dim, 0.5, 0.05, 0.2, 0.2, 0.5, 0.8, frames, memory_len, flags, p[5], 0, T,
            *p[6:13], p[13], ws_bytes, None)


@pytest.mark.parametrize("dims", BAD_SIZES)
def test_sizes_are_checked_before_any_launch(lib, dims):
    from uninext_b200 import _cabi
    n = ctypes.c_int64(-5)
    assert _cabi.entry("msda_idol_workspace")(*dims, ctypes.byref(n)) == BADARG and n.value == -5
    assert _cabi.entry("msda_idol_match_f32")(*_args(dims)) == BADARG


def test_workspace_query_and_argument_checks(lib):
    from uninext_b200 import _cabi
    ws_query, f32 = _cabi.entry("msda_idol_workspace"), _cabi.entry("msda_idol_match_f32")
    n = ctypes.c_int64(0)
    assert ws_query(10, 8, 32, 40, 72, None) == BADARG
    assert ws_query(10, 8, 32, 40, 72, ctypes.byref(n)) == 0
    assert n.value >= 10 * 92 * 4 + 8 * 32 * 4 + 10 * 8 * 4           # mask bits, memo embeddings, feats
    small = n.value
    assert f32(*_args(ws_bytes=small - 1)) == BADARG                   # workspace too small
    assert f32(*_args(ws_bytes=small, ws=264)) == BADARG               # workspace not 16-byte aligned
    for i in range(14):
        assert f32(*_args(ws_bytes=small, null=i)) == BADARG, i
    for bad in (dict(memory_len=0), dict(memory_len=65), dict(frames=0), dict(flags=8), dict(n_src=0)):
        assert f32(*_args(ws_bytes=small, **bad)) == BADARG, bad


def test_constructor_and_input_errors():
    from uninext_b200.modules.tracker import IDOLTracker, temporal_weights
    for bad in (dict(match_metric="softmax"), dict(match_metric="cosine"), dict(memory_len=0), dict(memory_len=65),
                dict(memo_momentum=1.5), dict(memo_tracklet_frames=0), dict(max_tracklets=0),
                dict(max_tracklets=1025), dict(match_score_thr=-0.1)):
        with pytest.raises(ValueError):
            IDOLTracker(**dict(tc.VIS_SETTINGS, **bad))
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        IDOLTracker(**tc.VIS_SETTINGS, device="cpu")
    with pytest.raises(ValueError, match="torch.range"):
        temporal_weights(93)                                # torch.range(0, 1, 1/93) does not have 94 elements
    tw = temporal_weights(64)
    assert tw.shape == (64, 64) and tw[2, :3].tolist() == pytest.approx([1 / 3, 2 / 3, 1.0])
    with pytest.raises(ValueError, match="memory_len"):
        IDOLTracker(**dict(tc.VIS_SETTINGS, memory_len=93))


def test_cpu_inputs_and_empty_frames_raise():
    from uninext_b200.modules.tracker import IDOLTracker
    tr = IDOLTracker.__new__(IDOLTracker)                    # no device needed to reach the input checks
    tr.device = torch.device("cuda")
    with pytest.raises(ValueError, match="no detections"):
        tr.match(torch.zeros(0, 5), torch.zeros(0), torch.zeros(0, 1, 4, 4), torch.zeros(0, 8), 0, [])
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        tr.match(torch.zeros(2, 5), torch.zeros(2), torch.zeros(2, 1, 4, 4), torch.zeros(2, 8), 0, [0, 1])
