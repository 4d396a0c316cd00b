"""CPU test: the video trackers' selection kernel (msda_detpost.cuh: trackpost_select, after detpost_scores) is in the
compiler's report in uninext_b200/lib/build.log without register spills.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def test_trackpost_kernel_is_built_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*trackpost_select\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert reports, f"{LOG}: no ptxas report of trackpost_select"
    for name, stack, st, ld in reports:
        assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, f"{name}: {stack} bytes stack, {st} / {ld} spills"
