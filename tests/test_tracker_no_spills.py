"""CPU test: the IDOL tracker's kernels (msda_tracker.cuh: idol_pack, idol_iou, idol_nms, idol_memo, idol_feats,
idol_softmax_stats, idol_assign, idol_update) are in the compiler's report in uninext_b200/lib/build.log without a stack
frame or register spills.  Skipped when the library has not been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
KERNELS = ["idol_pack", "idol_iou", "idol_nms", "idol_memo", "idol_feats", "idol_softmax_stats", "idol_assign",
           "idol_update"]


def test_tracker_kernels_are_built_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*idol_\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    found = {k for k in KERNELS for name, *_ in reports if re.search(rf"\d{k}E", name)}
    assert found == set(KERNELS), f"{LOG}: no ptxas report of {sorted(set(KERNELS) - found)}"
    for name, stack, st, ld in reports:
        assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, f"{name}: {stack} bytes stack, {st} / {ld} spills"
