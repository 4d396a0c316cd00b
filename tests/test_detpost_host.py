"""CPU tests of detection post-processing's host side: the positive map -> CSR conversion and its rejections, CPU tensors
raise (there is no CPU implementation), and msda_detpost_workspace / msda_detpost_f32 reject bad sizes with
MSDA_E_BADARG before they touch a pointer or the device."""
import ctypes

import pytest
import torch

from uninext_b200.modules.detection_postprocess import positive_map_to_csr, postprocess_detections

BADARG = -1


def test_csr_follows_labels_and_token_order():
    start, tokens = positive_map_to_csr({2: [7], 1: [3, 1, 2], 3: [0, 5]}, 256, "cpu")
    assert start.dtype == tokens.dtype == torch.int32
    assert start.tolist() == [0, 3, 4, 6]
    assert tokens.tolist() == [3, 1, 2, 7, 0, 5]


def test_csr_is_cached_per_content():
    a = positive_map_to_csr({1: [0, 1], 2: [4]}, 256, "cpu")
    b = positive_map_to_csr({2: [4], 1: [0, 1]}, 256, "cpu")
    assert a[0] is b[0] and a[1] is b[1]
    c = positive_map_to_csr({1: [0, 1], 2: [5]}, 256, "cpu")
    assert c[1] is not a[1]


@pytest.mark.parametrize("pmap, match", [
    ({2: [0], 3: [1]}, "exactly 1..C"),                 # the reference raises IndexError for label C + 1
    ({1: [0], 3: [1]}, "exactly 1..C"),                 # a gap: the reference would leave a zero column
    ({0: [0], 1: [1]}, "exactly 1..C"),
    ({}, "exactly 1..C"),
    ({1: [0], 2: []}, "no tokens"),                     # the reference's mean over no tokens is NaN
    ({1: [0, 256]}, "outside"),
    ({1: [-1]}, "outside"),
])
def test_csr_rejections(pmap, match):
    with pytest.raises(ValueError, match=match):
        positive_map_to_csr(pmap, 256, "cpu")


def test_token_outside_the_call_T_raises():
    with pytest.raises(ValueError, match="outside"):
        positive_map_to_csr({1: [0], 2: [200]}, 128, "cpu")


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        postprocess_detections(torch.zeros(1, 10, 256), torch.zeros(1, 10, 4), {1: [0]}, [(480, 640)])


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.load()


# (B, Q, T, C, max_num_inst)
BAD_SIZES = [
    (-1, 900, 256, 80, 100),
    (65536, 900, 256, 80, 100),
    (1, 0, 256, 80, 100),
    (1, 1025, 256, 80, 100),                            # Q past 1024
    (1, 900, 0, 80, 100),
    (1, 900, 257, 80, 100),                             # T past 256
    (1, 900, 256, 0, 100),
    (1, 900, 256, 4097, 100),
    (1, 900, 256, 80, 0),
    (1, 10, 256, 1, 11),                                # max_num_inst past Q*C
]


@pytest.mark.parametrize("dims", BAD_SIZES)
def test_sizes_are_checked_before_any_launch(lib, dims):
    n = ctypes.c_int64(-5)
    assert lib.msda_detpost_workspace(*dims, ctypes.byref(n)) == BADARG and n.value == -5
    fake = ctypes.c_void_p(256)                         # never dereferenced: the sizes are checked first
    b, q, t, c, k = dims
    assert lib.msda_detpost_f32(*[fake] * 6, b, q, t, c, 1, 0.7, k, *[fake] * 6, 1 << 40, None) == BADARG


def test_workspace_query_and_its_checks(lib):
    n = ctypes.c_int64(0)
    assert lib.msda_detpost_workspace(1, 900, 256, 80, 100, None) == BADARG
    assert lib.msda_detpost_workspace(1, 900, 256, 80, 100, ctypes.byref(n)) == 0
    assert n.value >= 900 * 80 * 4 + 900 * 8                # prob [B, Q, C] and the per-query maxima
    small = n.value
    assert lib.msda_detpost_workspace(1, 900, 256, 80, 900 * 80, ctypes.byref(n)) == 0
    assert n.value >= small + 131072 * 8                    # a sort buffer once max_num_inst passes 2048
    assert lib.msda_detpost_workspace(0, 900, 256, 80, 100, ctypes.byref(n)) == 0
    fake = ctypes.c_void_p(256)
    args = lambda ws_bytes, ws=fake, boxes=fake: (*[fake] * 6, 1, 900, 256, 80, 1, 0.7, 100, fake, fake, fake, boxes,
                                                  fake, ws, ws_bytes, None)
    assert lib.msda_detpost_f32(*args(small - 1)) == BADARG                       # workspace too small
    assert lib.msda_detpost_f32(*args(small, ws=ctypes.c_void_p(264))) == BADARG   # workspace not 16-byte aligned
    assert lib.msda_detpost_f32(*args(small, boxes=ctypes.c_void_p(260))) == BADARG
    nulls = list(args(small))
    for i in (0, 1, 3, 4, 5, 13, 14, 15, 16, 17, 18):      # every pointer but iou_pred is required
        a = list(nulls)
        a[i] = None
        assert lib.msda_detpost_f32(*a) == BADARG, i
