"""CPU tests of mask pasting's host side: CPU tensors raise (there is no CPU implementation), and msda_mask_paste_f32
rejects bad sizes (MSDA_E_BADARG / MSDA_E_TOOLARGE) before it touches a pointer or the device."""
import ctypes

import pytest
import torch

from uninext_b200.modules.mask_postprocess import paste_masks

BADARG, TOOLARGE = -1, -2


def test_cpu_tensor_raises():
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        paste_masks(torch.zeros(2, 1, 10, 12), (40, 48), (20, 24))


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.load()


# (I, Hs, Ws, stride, crop_h, crop_w, out_h, out_w, expected)
SIZES = [
    (-1, 10, 12, 4, 40, 48, 20, 24, BADARG),
    (2, 0, 12, 4, 1, 48, 20, 24, BADARG),
    (2, 10, 12, 0, 40, 48, 20, 24, BADARG),
    (2, 10, 12, 4, 41, 48, 20, 24, BADARG),          # crop taller than the padded input
    (2, 10, 12, 4, 40, 49, 20, 24, BADARG),
    (2, 10, 12, 4, 0, 48, 20, 24, BADARG),
    (2, 10, 12, 4, 40, 48, 0, 24, BADARG),
    (2, 10, 12, 4, 40, 48, 20, -3, BADARG),
    (2, 1 << 29, 12, 4, 40, 48, 20, 24, BADARG),     # stride * Hs past int32
    (2, 10, 12, 4, 40, 48, 1 << 30, 24, TOOLARGE),
    (2, 10, 12, 4, 40, 48, 20, 1 << 30, TOOLARGE),
    (0, 10, 12, 4, 40, 48, 20, 24, 0),                # no instances: nothing to launch
]


@pytest.mark.parametrize("args", SIZES)
def test_sizes_are_checked_before_any_launch(lib, args):
    *dims, want = args
    fake = ctypes.c_void_p(256)                      # never dereferenced: the sizes are checked first
    assert lib.msda_mask_paste_f32(fake, *dims, 0.5, 1, fake, None) == want
    assert lib.msda_mask_paste_f32(None, *dims, 0.5, 1, fake, None) == BADARG
