"""CPU tests of the video trackers' detection selection's host side (include/msda_trackpost.h,
select_track_detections): the header, the ctypes table and the library's exports agree; a library without the entry
points still loads and only the new API raises; msda_trackpost_workspace / msda_trackpost_f32 reject bad sizes, pointers
and formats with MSDA_E_BADARG before they touch a pointer or the device; CPU tensors raise."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from uninext_b200.modules.detection_postprocess import select_track_detections

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "msda_trackpost.h")
BADARG = -1


def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): len([a for a in m.group(2).split(",") if a.strip()])
            for m in re.finditer(r"\bint\s+(msda_\w+)\s*\(([^;{]*)\)\s*;", text)}


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.trackpost()


def test_header_ctypes_table_and_exports_agree(lib):
    from uninext_b200 import _cabi
    decl = _declared()
    assert set(decl) == set(_cabi.TRACKPOST_SIGNATURES) and len(decl) == 2
    assert not set(decl) & (set(_cabi.SIGNATURES) | set(_cabi.TWOSTAGE_SIGNATURES) | set(_cabi.FLATTEN_SIGNATURES))
    for name, nargs in decl.items():
        assert len(_cabi.TRACKPOST_SIGNATURES[name][1]) == nargs, name
        assert _cabi.entry(name).argtypes == _cabi.TRACKPOST_SIGNATURES[name][1], name
    text = open(HEADER).read()
    formats = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+MSDA_TRACKPOST_(\w+)\s+(\d+)\b", text)}
    assert formats == {"CXCYWH": _cabi.TRACKPOST_CXCYWH, "XYXY_PIXELS": _cabi.TRACKPOST_XYXY_PIXELS}
    assert lib.msda_abi_version() == 11 == _cabi.ABI_VERSION                       # msda_b200.h is unchanged


def test_library_without_the_entry_points_raises_only_for_them(tmp_path):
    """A library that exports msda_b200.h only loads for the rest of the package; the trackers' entry points raise
    MSDALibraryError."""
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
    stub = _cabi.load(str(so))
    assert stub.msda_abi_version() == _cabi.ABI_VERSION
    with pytest.raises(_cabi.MSDALibraryError, match="msda_trackpost_"):
        _cabi.trackpost(str(so))
    for name in _cabi.TRACKPOST_SIGNATURES:
        with pytest.raises(_cabi.MSDALibraryError, match=name):
            _cabi.entry(name, str(so))


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        select_track_detections(torch.zeros(1, 10, 256), torch.zeros(1, 10, 4), {1: [0]}, score_thres=0.1,
                                nms_iou=0.7, box_format="cxcywh")


# (B, Q, T, C)
BAD_SIZES = [
    (-1, 900, 256, 8),
    (65536, 900, 256, 8),
    (1, 0, 256, 8),
    (1, 1025, 256, 8),                                  # Q past 1024
    (1, 900, 0, 8),
    (1, 900, 257, 8),                                   # T past 256
    (1, 900, 256, 0),
    (1, 900, 256, 4097),
]


def _args(dims=(1, 900, 256, 40), ws_bytes=1 << 40, fmt=1, null=None, ws=256, boxes=256):
    """Pointer slots in order: box_cls, box_pred, iou_pred, class_start, tokens, ori_sizes (0-5), then scores, labels,
    query_index, boxes, count, workspace (6-11).  Fake addresses: never dereferenced when a check fails."""
    p = [ctypes.c_void_p(256)] * 12
    p[9], p[11] = ctypes.c_void_p(boxes), ctypes.c_void_p(ws)
    if null is not None:
        p[null] = None
    return (*p[:6], *dims, 0.1, 0.7, fmt, *p[6:12], ws_bytes, None)


@pytest.mark.parametrize("dims", BAD_SIZES)
def test_sizes_are_checked_before_any_launch(lib, dims):
    from uninext_b200 import _cabi
    n = ctypes.c_int64(-5)
    assert _cabi.entry("msda_trackpost_workspace")(*dims, ctypes.byref(n)) == BADARG and n.value == -5
    assert _cabi.entry("msda_trackpost_f32")(*_args(dims)) == BADARG


def test_workspace_query_and_its_checks(lib):
    from uninext_b200 import _cabi
    ws_query, f32 = _cabi.entry("msda_trackpost_workspace"), _cabi.entry("msda_trackpost_f32")
    n = ctypes.c_int64(0)
    assert ws_query(1, 900, 256, 40, None) == BADARG
    assert ws_query(1, 900, 256, 40, ctypes.byref(n)) == 0
    assert n.value >= 900 * 40 * 4 + 900 * 8                # prob [B, Q, C] and the per-query maxima
    small = n.value
    assert ws_query(2, 900, 256, 40, ctypes.byref(n)) == 0 and n.value >= 2 * (900 * 40 * 4 + 900 * 8)
    assert ws_query(0, 900, 256, 40, ctypes.byref(n)) == 0
    assert f32(*_args(ws_bytes=small - 1)) == BADARG                            # workspace too small
    assert f32(*_args(ws_bytes=small, ws=264)) == BADARG                        # workspace not 16-byte aligned
    assert f32(*_args(ws_bytes=small, boxes=260)) == BADARG                     # boxes not 16-byte aligned
    for fmt in (-1, 2):
        assert f32(*_args(ws_bytes=small, fmt=fmt)) == BADARG                   # unknown box_format
    for i in (0, 1, 3, 4, 5, 6, 7, 8, 9, 10, 11):          # every pointer but iou_pred (and ori_sizes for cxcywh)
        assert f32(*_args(ws_bytes=small, null=i)) == BADARG, i
    assert f32(*_args((0, 900, 256, 40), ws_bytes=small, null=2)) == 0          # B = 0: checks pass, nothing runs
    assert f32(*_args((0, 900, 256, 40), ws_bytes=small, fmt=0, null=5)) == 0   # cxcywh reads no ori_sizes
