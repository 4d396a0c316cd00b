"""CPU test: the fused image-text attention kernels (msda_vlfuse.cuh) compile without register spills.

uninext_b200/build.py compiles the library with -Xptxas -v and keeps the compiler's report in uninext_b200/lib/build.log.
Each kernel keeps a register tile of logits (and, on the column side, two gradient accumulators) live across its loop;
a spill would put local-memory traffic inside every product.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def test_vlfuse_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*vlf_\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    names = {re.search(r"vlf_[a-z_]+", n).group(0) for n, *_ in reports}
    assert {"vlf_fwd_rows", "vlf_fwd_cols", "vlf_colstats", "vlf_reduce", "vlf_bwd_delta", "vlf_bwd_rows",
            "vlf_bwd_cols", "vlf_dropout_mask"} <= names, f"{LOG}: missing ptxas reports, got {names}"
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
