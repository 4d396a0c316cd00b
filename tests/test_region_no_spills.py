"""CPU test: the region backward (msda_bwd_region) compiles without register spills.

uninext_b200/build.py compiles the library with -Xptxas -v and keeps the compiler's report in uninext_b200/lib/build.log.
Local-memory spills in that kernel's gather loop compete with the gathers for the SM's L1, so a change that brings them
back fails here.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def _region_reports(text):
    """[(function, stack bytes, spill store bytes, spill load bytes)] for every compiled msda_bwd_region instance."""
    out = []
    for m in re.finditer(r"Function properties for (\S*msda_bwd_region\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text):
        out.append((m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))))
    return out


def test_region_backward_does_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        reports = _region_reports(fh.read())
    assert reports, f"{LOG} has no ptxas report for msda_bwd_region"
    for name, stack, st, ld in reports:
        assert st == 0 and ld == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
