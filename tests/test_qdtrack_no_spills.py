"""CPU test: the QuasiDense tracker's kernels (msda_qdtrack.cuh: qd_sort, qd_iou, qd_dedup, qd_memo, qd_assign,
qd_update; idol_feats and idol_softmax_stats are shared with the IDOL tracker) are in the compiler's report in
uninext_b200/lib/build.log without a stack frame or register spills.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
KERNELS = ["qd_sort", "qd_iou", "qd_dedup", "qd_memo", "qd_assign", "qd_update", "idol_feats", "idol_softmax_stats"]


def test_qdtrack_kernels_are_built_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (_ZN4msda\d+(?:qd|idol)_\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    found = {k for k in KERNELS for name, *_ in reports if re.search(rf"\d{k}E", name)}
    assert found == set(KERNELS), f"{LOG}: no ptxas report of {sorted(set(KERNELS) - found)}"
    for name, stack, st, ld in reports:
        assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, f"{name}: {stack} bytes stack, {st} / {ld} spills"
