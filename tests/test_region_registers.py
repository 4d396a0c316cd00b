"""CPU test: the region backward (msda_bwd_region) fits the register budget of 2 CTAs/SM, and the grad_value pass it
calls does not spill.

uninext_b200/build.py compiles the library with -Xptxas -v and keeps the compiler's report in uninext_b200/lib/build.log.
The kernel is launched with 256 threads and two resident CTAs per SM (kRegionMinCtas): 65536 registers / 512 threads
allows at most 128 registers per thread.  The grad_value pass is a separate (non-inlined) device function, so its own
report line is checked here too.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
MAX_REGS = 65536 // (256 * 2)


def _log():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        return fh.read()


def test_region_kernel_fits_two_ctas_per_sm():
    found = re.findall(r"Function properties for (\S*msda_bwd_region\S*)\s*\n[^\n]*\n\s*ptxas info\s*: Used (\d+) registers",
                       _log())
    assert found, f"{LOG} has no register report for msda_bwd_region"
    for name, regs in found:
        assert int(regs) <= MAX_REGS, f"{name}: {regs} registers, more than {MAX_REGS} (2 CTAs/SM)"


def test_region_grad_value_pass_does_not_spill():
    found = re.findall(r"Function properties for (\S*region_grad_value_pass\S*)\s*\n\s*(\d+) bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", _log())
    assert found, f"{LOG} has no ptxas report for region_grad_value_pass"
    for name, _, st, ld in found:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
