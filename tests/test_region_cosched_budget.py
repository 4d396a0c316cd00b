"""CPU test: 2 grad_value CTAs (msda_region_grad_value_pass) and 1 tap CTA (msda_bwd_region) fit one H100 SM together.

The region backward launches the two kernels so that they run side by side (uninext_b200/csrc/msda_region.cuh,
region_grids): the tap pass is bound by its gathers, the grad_value pass by latency.  The block scheduler can only place
them together while, per SM:
  - registers, allocated per warp in units of 256: 2 x 8 warps x roundup(32 x r_gv, 256) + 8 warps x roundup(32 x r_tap,
    256) <= 65536;
  - shared memory: 2 x (static + dynamic + 1 KB reserved) of the grad_value kernel + the same for the tap kernel
    <= 228 KB;
  - threads: 3 x 256 <= 2048.
Registers and static shared memory come from the ptxas report in uninext_b200/lib/build.log (uninext_b200/build.py
compiles with -Xptxas -v); the dynamic sizes are restated from the header's constants.  A register or shared-memory
increase that would serialise the two kernels again fails here.  Skipped when the library has not been built."""
import os
import re

import pytest

from tests.region_layout import HEADER
from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
REGS_PER_SM = 65536                  # H100 (sm_90)
SMEM_PER_SM = 228 * 1024
THREADS_PER_SM = 2048
RESERVED_PER_CTA = 1024              # shared memory the SM reserves per resident CTA
THREADS = 256                        # kTiledThreads: both kernels
GV_CTAS, TAP_CTAS = 2, 1


def _header():
    with open(HEADER) as fh:
        return fh.read()


def _constants(text):
    return {k: int(v) for k, v in re.findall(r"constexpr int (k\w+) = (\d+);", text)}


def _gv_dynamic_smem(text):
    """region_gv_smem_bytes(): per entry position (slot, tap, corner) a coefficient (f32), a window row (u16) and a
    sorted index (u16); one 128-byte grad_out row per stash slot; one int count per window row."""
    body = re.search(r"constexpr size_t region_gv_smem_bytes\(\) \{(.*?)\n\}", text, re.S)
    assert body, f"{HEADER} has no region_gv_smem_bytes()"
    assert re.search(r"kRegionEntries \* \(4 \+ 2 \+ 2\) \+ \(size_t\)kRegionSlots \* 128 \+ \(size_t\)kRegionWinRows \* 4",
                     body.group(1)), "region_gv_smem_bytes() changed: update the restatement here"
    c = _constants(text)
    return c["kRegionSlots"] * 16 * 4 * (4 + 2 + 2) + c["kRegionSlots"] * 128 + c["kRegionWinRows"] * 4


def _tap_dynamic_smem(text):
    """region_tap_smem_bytes(): one TapStage<4, 16, true> per warp, a double buffer of 4 groups x 16 taps x (x, y, a)."""
    assert re.search(r"using RegionTapStage = TapStage<4, 16, true>;", text), "RegionTapStage changed: update here"
    assert re.search(r"region_tap_smem_bytes\(\) \{ return \(size_t\)kTiledWarps \* RegionTapStage::kBytes; \}", text), \
        "region_tap_smem_bytes() changed: update the restatement here"
    return (THREADS // 32) * 2 * (4 * 16 * 8 + 4 * 16 * 4)


def _reports(kernel):
    """[(mangled name, registers, spill store bytes, spill load bytes, static smem bytes)] of a kernel."""
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        log = fh.read()
    found = re.findall(r"Function properties for (\S*" + kernel + r"I\S*)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads\s*\n\s*ptxas info\s*: Used (\d+) registers, [^\n]*?(\d+) bytes smem",
                       log)
    assert found, f"{LOG} has no ptxas report for {kernel}"
    return [(name, int(regs), int(st), int(ld), int(smem)) for name, st, ld, regs, smem in found]


def _cta_registers(regs):
    return (THREADS // 32) * ((regs * 32 + 255) // 256 * 256)


def test_two_grad_value_ctas_and_one_tap_cta_fit_one_sm():
    text = _header()
    gv_dyn, tap_dyn = _gv_dynamic_smem(text), _tap_dynamic_smem(text)
    for gname, gregs, gst, gld, gstatic in _reports("msda_region_grad_value_pass"):
        for tname, tregs, tst, tld, tstatic in _reports("msda_bwd_region"):
            assert gst == gld == tst == tld == 0, (gname, tname, "spills")
            regs = GV_CTAS * _cta_registers(gregs) + TAP_CTAS * _cta_registers(tregs)
            assert regs <= REGS_PER_SM, f"{gname} ({gregs}) x {GV_CTAS} + {tname} ({tregs}): {regs} registers per SM"
            smem = GV_CTAS * (gstatic + gv_dyn + RESERVED_PER_CTA) + TAP_CTAS * (tstatic + tap_dyn + RESERVED_PER_CTA)
            assert smem <= SMEM_PER_SM, f"{gname} x {GV_CTAS} + {tname}: {smem} bytes of shared memory per SM"
            assert (GV_CTAS + TAP_CTAS) * THREADS <= THREADS_PER_SM

