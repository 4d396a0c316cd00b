"""CPU test: the COCO RLE kernels (msda_maskrle.cuh) are in the compiler's report in uninext_b200/lib/build.log without
register spills or a stack frame, and mask_paste, whose pixel expression they share through mp_prob, keeps the register
counts it had before mp_prob existed.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
RLE_KERNELS = ["rle_bits_logits", "rle_bits_u8ILb0E", "rle_bits_u8ILb1E", "rle_boundaries", "rle_tile_bytes",
               "rle_scan_tiles", "rle_write"]
# mask_paste<BINARY, VEC> with nvcc 12.9 for sm_90a, as built before its expression moved into mp_prob
MASK_PASTE_REGISTERS = {("0", "0"): 80, ("0", "1"): 102, ("1", "0"): 80, ("1", "1"): 94}


def _reports():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    return re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", text)


def test_rle_kernels_are_built_without_spills():
    reports = _reports()
    for k in RLE_KERNELS:
        found = [r for r in reports if k in r[0]]
        assert found, f"{LOG}: no ptxas report for {k}"
        for name, stack, st, ld, _ in found:
            assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, \
                f"{name}: {stack} bytes stack, {st} bytes spill stores, {ld} bytes spill loads"


def test_mask_paste_register_counts_are_unchanged():
    got = {re.search(r"ILb([01])ELb([01])E", n).groups(): int(regs)
           for n, _, _, _, regs in _reports() if "10mask_paste" in n}
    assert got == MASK_PASTE_REGISTERS
