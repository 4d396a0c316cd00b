"""CPU test: the detection post-processing kernels (msda_detpost.cuh: the score kernel and both instantiations of the
per-image select kernel, with and without NMS) are in the compiler's report in uninext_b200/lib/build.log without
register spills.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def test_detpost_kernels_are_built_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*detpost_(?:scores|select)\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    built = {("scores",) if "scores" in n else ("select", re.search(r"ILb([01])E", n).group(1)) for n, *_ in reports}
    want = {("scores",), ("select", "0"), ("select", "1")}
    assert want <= built, f"{LOG}: missing ptxas reports, got {built}"
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
