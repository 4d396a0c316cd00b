"""CPU tests of the QuasiDense tracker's host side: the restatement of tests/qdtrack_case.py reproduces the reference's
goldens (tests/golden/qdtrack/, made by tests/golden/make_qdtrack_golden.py) exactly; include/msda_qdtrack.h, the
ctypes table and the library's exports agree; msda_qdtrack_workspace / msda_qdtrack_match_f32 reject bad arguments
before they touch a pointer or the device; QuasiDenseTracker's constructor and inputs are checked."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests import qdtrack_case as qc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "msda_qdtrack.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "qdtrack")
BADARG = -1


@pytest.mark.parametrize("name", sorted(qc.SETTINGS))
def test_restatement_reproduces_the_reference_goldens(name):
    z = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    seq = qc.golden_sequence(name)
    assert str(z["checksum"]) == qc.checksum(seq) and int(z["frames"]) == len(seq) == 20
    ref = qc.Restated(**qc.SETTINGS[name])
    unsorted = 0
    for f, (boxes, scores, labels, embeds) in enumerate(seq):
        n = scores.shape[0]
        assert n <= 40 and embeds.shape[1] == 256 and int(labels.max()) < 8
        order, keep, ids = ref.step(boxes, scores, labels, embeds, f)
        unsorted += order != list(range(n))
        assert [order[p] for p in keep] == z[f"{f}/rows"].tolist() and ids == z[f"{f}/ids"].tolist(), f
        assert [3 * p + 7 for p in keep] == z[f"{f}/indices"].tolist()          # the sorted mask on unsorted indices
        tids = sorted(ref.tracks)
        assert tids == z[f"{f}/track_ids"].tolist()
        for c, t in enumerate(tids):
            v = ref.tracks[t]
            assert (v["last_frame"], v["label"]) == (z[f"{f}/last_frame"][c], z[f"{f}/label"][c])
            assert np.array_equal(v["embed"].numpy(), z[f"{f}/embed"][c])
        back_l = ref.backdrops[0].tolist() if ref.backdrops is not None else []
        assert back_l == z[f"{f}/back_labels"].tolist()
        if back_l:
            assert np.array_equal(ref.backdrops[1].numpy(), z[f"{f}/back_embeds"])
    assert unsorted == 1
    want = {"dup_class", "dup_backdrop", "dup_via_removed", "suppressed", "left", "category_decides", "new", "empty"}
    if qc.SETTINGS[name]["memo_backdrop_frames"]:
        want.add("best_is_backdrop")
    assert want <= ref.seen, want - ref.seen
    assert min(ref.margins) >= 1e-4


def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): len([a for a in m.group(2).split(",") if a.strip()])
            for m in re.finditer(r"\bint\s+(msda_\w+)\s*\(([^;{]*)\)\s*;", text)}


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.qdtrack()


def test_header_ctypes_table_and_exports_agree(lib):
    from uninext_b200 import _cabi
    decl = _declared()
    assert set(decl) == set(_cabi.QDTRACK_SIGNATURES) and len(decl) == 2
    others = set(_cabi.SIGNATURES) | set(_cabi.TRACKPOST_SIGNATURES) | set(_cabi.TRACKER_SIGNATURES)
    assert not set(decl) & others
    for name, nargs in decl.items():
        assert len(_cabi.QDTRACK_SIGNATURES[name][1]) == nargs, name
        assert _cabi.entry(name).argtypes == _cabi.QDTRACK_SIGNATURES[name][1], name
    text = open(HEADER).read()
    consts = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+MSDA_QD_(\w+)\s+(\d+)\b", text)}
    assert consts == {"BACKDROPS": _cabi.QD_BACKDROPS, "MAX_BACKDROPS": _cabi.QD_MAX_BACKDROPS, "STATE_LIVE": 0,
                      "STATE_NEXT_ID": 1, "STATE_FLAGS": 2, "STATE_BACKDROPS": 3, "OVERFLOW": _cabi.QD_OVERFLOW,
                      "BAD_ROW": _cabi.QD_BAD_ROW}
    assert (_cabi.QD_OVERFLOW, _cabi.QD_BAD_ROW) == (_cabi.IDOL_OVERFLOW, _cabi.IDOL_BAD_ROW)   # one error reader
    assert re.search(r"MSDA_QD_STATE_INTS\(max_tracklets\) \(4 \+ 4 \* \(max_tracklets\) \+ 1024\)", text)
    assert lib.msda_abi_version() == 11 == _cabi.ABI_VERSION                       # msda_b200.h is unchanged


def test_library_without_the_entry_points_raises_only_for_them(tmp_path):
    from uninext_b200 import _cabi
    src = tmp_path / "stub.c"
    body = ["int msda_abi_version(void) { return %d; }" % _cabi.ABI_VERSION]
    body += [f"int {n}(void) {{ return 0; }}" for n in _cabi.SIGNATURES if n != "msda_abi_version"]
    src.write_text("\n".join(body) + "\n")
    so = tmp_path / "libstub.so"
    try:
        subprocess.run(["gcc", "-shared", "-fPIC", "-o", str(so), str(src)], check=True, capture_output=True)
    except (OSError, subprocess.CalledProcessError) as exc:
        pytest.skip(f"no C compiler: {exc}")
    assert _cabi.load(str(so)).msda_abi_version() == _cabi.ABI_VERSION
    with pytest.raises(_cabi.MSDALibraryError, match="msda_qdtrack_"):
        _cabi.qdtrack(str(so))
    for name in _cabi.QDTRACK_SIGNATURES:
        with pytest.raises(_cabi.MSDALibraryError, match=name):
            _cabi.entry(name, str(so))


# (n_cap, max_tracklets, dim)
BAD_SIZES = [(0, 8, 32), (1025, 8, 32), (10, 0, 32), (10, 1025, 32), (10, 8, 0)]


def _args(dims=(10, 8, 32), ws_bytes=1 << 40, null=None, ws=256, frames=10, flags=1, n_src=10):
    """Pointer slots in order: boxes, scores, labels, embeds, rows, count (0-5), state, embed, backdrop_embed, order,
    ids, tracked, tracked_count (6-12), workspace (13).  Fake addresses: never dereferenced when a check fails."""
    n_cap, T, dim = dims
    p = [ctypes.c_void_p(256)] * 14
    p[13] = ctypes.c_void_p(ws)
    if null is not None:
        p[null] = None
    return (*p[:6], n_src, n_cap, dim, 0.5, 0.3, 0.5, 0.5, 0.3, 0.7, 1.0, frames, flags, 0, T, *p[6:13], p[13],
            ws_bytes, None)


@pytest.mark.parametrize("dims", BAD_SIZES)
def test_sizes_are_checked_before_any_launch(lib, dims):
    from uninext_b200 import _cabi
    n = ctypes.c_int64(-5)
    assert _cabi.entry("msda_qdtrack_workspace")(*dims, ctypes.byref(n)) == BADARG and n.value == -5
    assert _cabi.entry("msda_qdtrack_match_f32")(*_args(dims)) == BADARG


def test_workspace_query_and_argument_checks(lib):
    from uninext_b200 import _cabi
    ws_query, f32 = _cabi.entry("msda_qdtrack_workspace"), _cabi.entry("msda_qdtrack_match_f32")
    n = ctypes.c_int64(0)
    assert ws_query(10, 8, 32, None) == BADARG
    assert ws_query(10, 8, 32, ctypes.byref(n)) == 0
    assert n.value >= (8 + 1024) * 32 * 4 + 10 * (8 + 1024) * 4           # memo embeddings, feats
    small = n.value
    assert f32(*_args(ws_bytes=small - 1)) == BADARG                   # workspace too small
    assert f32(*_args(ws_bytes=small, ws=264)) == BADARG               # workspace not 16-byte aligned
    for i in range(14):
        assert f32(*_args(ws_bytes=small, null=i)) == BADARG, i
    for bad in (dict(frames=0), dict(flags=2), dict(flags=-1), dict(n_src=0)):
        assert f32(*_args(ws_bytes=small, **bad)) == BADARG, bad


def test_constructor_and_input_errors():
    from uninext_b200.modules.tracker import QuasiDenseTracker
    for bad in (dict(match_metric="softmax"), dict(match_metric="cosine"), dict(with_cats=False),
                dict(memo_backdrop_frames=2), dict(memo_momentum=1.5), dict(memo_momentum=-0.1),
                dict(memo_tracklet_frames=0), dict(max_tracklets=0), dict(max_tracklets=1025),
                dict(match_score_thr=-0.1)):
        with pytest.raises(ValueError):
            QuasiDenseTracker(**dict(qc.BDD, **bad))
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        QuasiDenseTracker(**qc.BDD, device="cpu")


def test_cpu_inputs_and_empty_frames_raise():
    from uninext_b200.modules.tracker import QuasiDenseTracker
    tr = QuasiDenseTracker.__new__(QuasiDenseTracker)          # no device needed to reach the input checks
    tr.device = torch.device("cuda")
    with pytest.raises(ValueError, match="no detections"):
        tr.match(torch.zeros(0, 5), torch.zeros(0), torch.zeros(0, 8), 0, [])
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        tr.match(torch.zeros(2, 5), torch.zeros(2), torch.zeros(2, 8), 0, [0, 1])
