"""CPU test: the deterministic backward's kernels (msda_det.cuh) compile without register spills.

uninext_b200/build.py compiles the library with -Xptxas -v and keeps the compiler's report in uninext_b200/lib/build.log.
The ordered accumulate keeps a round of grad_out rows in registers while earlier adds retire; a spill would put local
memory traffic on that serial chain.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def test_deterministic_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*msda_det_\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    names = {re.match(r"[a-z0-9_]+", n.split("msda_det_", 1)[1]).group(0) for n, *_ in reports}
    assert {"keys", "bounds", "accumulate", "accumulate_v4"} <= names, f"{LOG}: missing ptxas reports, got {names}"
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
