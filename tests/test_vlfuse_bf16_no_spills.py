"""CPU test: the bf16 tensor-core kernels of the fused image-text attention (msda_vlfuse_bf16.cuh) are in the compiler's
report in uninext_b200/lib/build.log, for both head sizes, without register spills.  Skipped when the library has not
been built."""
import os
import re

import pytest

from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")


def test_vlfuse_bf16_kernels_are_built_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        text = fh.read()
    reports = re.findall(r"Function properties for (\S*vlf_bf16_\S*)\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    built = {(re.search(r"vlf_bf16_[a-z_]+", n).group(0), re.search(r"ILi(\d+)E", n).group(1)) for n, *_ in reports}
    want = {(k, d) for k in ("vlf_bf16_fwd_rows", "vlf_bf16_fwd_cols", "vlf_bf16_bwd_rows", "vlf_bf16_bwd_cols")
            for d in ("128", "256")}
    assert want <= built, f"{LOG}: missing ptxas reports, got {built}"
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"
