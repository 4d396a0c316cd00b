"""CPU tests of COCO run-length encoding (DESIGN.md section 3.14): the restatement in tests/coco_rle.py gives the known
answers and round-trips, its numpy form agrees with it, CPU tensors raise (there is no CPU implementation), and the
msda_mask_rle_* entries reject bad sizes with MSDA_E_BADARG / MSDA_E_TOOLARGE before they touch a pointer or the device."""
import ctypes

import numpy as np
import pytest
import torch

from tests.coco_rle import counts_np, counts_of, from_string, string_np, to_string
from uninext_b200.modules.mask_postprocess import encode_masks_rle, paste_masks_rle

BADARG, TOOLARGE = -1, -2


@pytest.mark.parametrize("mask, counts, string", [
    (np.zeros((2, 2)), [4], b"4"),
    (np.ones((2, 2)), [0, 4], b"04"),
    (np.array([[0, 1], [1, 0]]), [1, 2, 1], b"121"),
])
def test_known_masks(mask, counts, string):
    assert counts_of(mask) == counts == counts_np(mask).tolist()
    assert to_string(counts) == string == string_np(counts)


@pytest.mark.parametrize("counts, string", [([100], b"T3"), ([5, 3, 1, 4], b"5311"), ([576000000], b"PPTZUa0")])
def test_known_counts(counts, string):
    assert to_string(counts) == string == string_np(counts)
    assert from_string(string) == counts


def test_round_trip_on_random_masks():
    rng = np.random.default_rng(0)
    for _ in range(300):
        h, w = rng.integers(1, 40, size=2)
        m = rng.random((h, w)) < rng.random()
        c = counts_of(m)
        assert sum(c) == h * w and all(v > 0 for v in c[1:])
        assert c == counts_np(m).tolist()
        s = to_string(c)
        assert s == string_np(c) and from_string(s) == c


def test_large_count_differences():
    rng = np.random.default_rng(1)
    for _ in range(50):
        c = [0] + rng.integers(1, 2 ** 32 - 1, size=rng.integers(1, 20)).tolist()  # differences span +-2^32
        s = to_string(c)
        assert s == string_np(c) and from_string(s) == c


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        paste_masks_rle(torch.zeros(2, 1, 10, 12), (40, 48), (20, 24))
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        encode_masks_rle(torch.zeros(2, 20, 24, dtype=torch.bool))


def test_threshold_must_be_a_number():
    with pytest.raises(ValueError, match="binary"):
        paste_masks_rle(torch.zeros(2, 1, 10, 12), (40, 48), (20, 24), threshold=None)


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.load()


# (I, out_h, out_w, expected), common to every entry
SIZES = [
    (-1, 20, 24, BADARG),
    (2, 0, 24, BADARG),
    (2, 20, -3, BADARG),
    (2, 65536, 65536, TOOLARGE),                     # 2^32 pixels: past the COCO API's 32-bit counts
    (2, 1, 1 << 30, TOOLARGE),
    (1 << 31, 20, 24, TOOLARGE),
]


@pytest.mark.parametrize("args", SIZES)
def test_sizes_are_checked_before_any_launch(lib, args):
    i, h, w, want = args
    n = ctypes.c_int64(-5)
    assert lib.msda_mask_rle_workspace(i, h, w, ctypes.byref(n)) == want and n.value == -5
    fake = ctypes.c_void_p(256)                      # never dereferenced: the sizes are checked first
    assert lib.msda_mask_rle_count_u8(fake, i, h, w, fake, 1 << 40, None) == want
    assert lib.msda_mask_rle_encode(i, h, w, 0, fake, 1 << 40, fake, fake, fake, None) == want
    if h <= 65535 * 16:
        assert lib.msda_mask_rle_count_f32(fake, i, 10, 12, 4, 40, 48, h, w, 0.5, fake, 1 << 40, None) == want


def test_pixel_limit_is_2_32_minus_1(lib):
    fake = ctypes.c_void_p(256)
    assert lib.msda_mask_rle_encode(1, 65536, 65537, 0, fake, 0, fake, fake, fake, None) == TOOLARGE
    assert lib.msda_mask_rle_encode(1, 65536, 65536, 0, fake, 0, fake, fake, fake, None) == TOOLARGE
    # 65535 x 65537 = 2^32 - 1 pixels passes the size checks; the boundary bound is checked against it
    assert lib.msda_mask_rle_encode(1, 65535, 65537, 2 ** 32, fake, 0, fake, fake, fake, None) == BADARG


# msda_mask_paste_f32's own limits, on the logits entry: (I, Hs, Ws, stride, crop_h, crop_w, out_h, out_w, expected)
PASTE_SIZES = [
    (2, 10, 12, 4, 41, 48, 20, 24, BADARG),          # crop taller than the padded input
    (2, 10, 12, 4, 40, 0, 20, 24, BADARG),
    (2, 10, 12, 0, 40, 48, 20, 24, BADARG),
    (2, 1 << 29, 12, 4, 40, 48, 20, 24, BADARG),     # stride * Hs past int32
    (2, 10, 12, 4, 40, 48, 65535 * 16 + 1, 24, TOOLARGE),
    (0, 10, 12, 4, 40, 48, 20, 24, 0),               # no instances: nothing to launch
]


@pytest.mark.parametrize("args", PASTE_SIZES)
def test_paste_limits_apply_to_the_logits_entry(lib, args):
    *dims, want = args
    fake = ctypes.c_void_p(256)
    assert lib.msda_mask_rle_count_f32(fake, *dims, 0.5, fake, 1 << 40, None) == want


def test_null_and_misaligned_pointers(lib):
    fake, odd = ctypes.c_void_p(256), ctypes.c_void_p(264)
    assert lib.msda_mask_rle_workspace(2, 20, 24, None) == BADARG
    assert lib.msda_mask_rle_count_u8(None, 2, 20, 24, fake, 1 << 40, None) == BADARG
    assert lib.msda_mask_rle_count_u8(fake, 2, 20, 24, None, 1 << 40, None) == BADARG
    assert lib.msda_mask_rle_count_u8(fake, 2, 20, 24, odd, 1 << 40, None) == BADARG      # workspace not 16-aligned
    assert lib.msda_mask_rle_count_f32(None, 2, 10, 12, 4, 40, 48, 20, 24, 0.5, fake, 1 << 40, None) == BADARG
    enc = lambda b, pos, offs, chars: lib.msda_mask_rle_encode(2, 20, 24, b, fake, 1 << 40, pos, offs, chars, None)
    assert enc(5, None, fake, fake) == BADARG                                            # positions needed when B > 0
    assert enc(5, fake, None, fake) == BADARG
    assert enc(5, fake, fake, None) == BADARG
    assert enc(5, fake, ctypes.c_void_p(260), fake) == BADARG                            # offsets not 8-aligned
    assert enc(-1, fake, fake, fake) == BADARG
    assert enc(2 * 20 * 24 + 1, fake, fake, fake) == BADARG                              # more boundaries than pixels
