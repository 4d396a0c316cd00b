"""CPU test: the region backward's grad_value kernel (msda_region_grad_value_pass, uninext_b200/csrc/msda_region.cuh)
fits the number of CTAs per SM its __launch_bounds__ asks for.

The kernel is latency-bound, so its speed rests on how many of its 256-thread CTAs are resident.  With k = the
minimum-CTAs argument of its __launch_bounds__:
  - registers: at most 65536 / (256 k) per thread, and no spills (ptxas report in uninext_b200/lib/build.log, which
    uninext_b200/build.py writes with -Xptxas -v);
  - shared memory: static (ptxas report) + dynamic (region_gv_smem_bytes(), restated here from the header's constants)
    + the 1 KB the SM reserves per CTA, k times, within the H100's 228 KB of shared memory per SM.
Skipped when the library has not been built."""
import os
import re

import pytest

from tests.region_layout import HEADER
from uninext_b200 import build as b

LOG = os.path.join(b.LIB_DIR, "build.log")
SMEM_PER_SM = 228 * 1024             # H100 (sm_90): shared memory per SM
RESERVED_PER_CTA = 1024              # shared memory the SM reserves per resident CTA
KERNEL = "msda_region_grad_value_pass"


def _header():
    with open(HEADER) as fh:
        return fh.read()


def _constants(text):
    return {k: int(v) for k, v in re.findall(r"constexpr int (k\w+) = (\d+);", text)}


def _min_ctas(text):
    m = re.search(r"__launch_bounds__\(kTiledThreads, (\w+)\)\s*\n\s*" + KERNEL + r"\(", text)
    assert m, f"{HEADER}: no __launch_bounds__ on {KERNEL}"
    arg = m.group(1)
    return int(arg) if arg.isdigit() else _constants(text)[arg]


def _dynamic_smem(text):
    """region_gv_smem_bytes(): per entry position (slot, tap, corner) a coefficient (f32), a window row (u16) and a
    sorted index (u16); one 128-byte grad_out row per stash slot; one int count per window row."""
    c = _constants(text)
    body = re.search(r"constexpr size_t region_gv_smem_bytes\(\) \{(.*?)\n\}", text, re.S)
    assert body, f"{HEADER} has no region_gv_smem_bytes()"
    assert re.search(r"kRegionEntries \* \(4 \+ 2 \+ 2\) \+ \(size_t\)kRegionSlots \* 128 \+ \(size_t\)kRegionWinRows \* 4",
                     body.group(1)), "region_gv_smem_bytes() changed: update the restatement here"
    entries = c["kRegionSlots"] * 16 * 4
    return entries * (4 + 2 + 2) + c["kRegionSlots"] * 128 + c["kRegionWinRows"] * 4


def _reports():
    """[(mangled name, registers, spill store bytes, spill load bytes, static smem bytes)] of the kernel."""
    if not os.path.exists(LOG):
        pytest.skip("library not built: no build.log")
    with open(LOG) as fh:
        log = fh.read()
    found = re.findall(r"Function properties for (\S*" + KERNEL + r"\S*)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads\s*\n\s*ptxas info\s*: Used (\d+) registers, [^\n]*?(\d+) bytes smem",
                       log)
    assert found, f"{LOG} has no ptxas report for {KERNEL}"
    return [(name, int(regs), int(st), int(ld), int(smem)) for name, st, ld, regs, smem in found]


def test_grad_value_kernel_registers_fit_its_ctas_per_sm():
    k = _min_ctas(_header())
    for name, regs, st, ld, _ in _reports():
        assert regs <= 65536 // (256 * k), f"{name}: {regs} registers, more than {65536 // (256 * k)} ({k} CTAs/SM)"
        assert st == 0 and ld == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"


def test_grad_value_kernel_shared_memory_fits_its_ctas_per_sm():
    text = _header()
    k, dyn = _min_ctas(text), _dynamic_smem(text)
    share = SMEM_PER_SM // k - RESERVED_PER_CTA
    for name, _, _, _, static in _reports():
        assert static + dyn <= share, f"{name}: {static} + {dyn} bytes of shared memory, more than {share} ({k} CTAs/SM)"


def test_grad_value_kernel_keeps_three_ctas_per_sm():
    assert _min_ctas(_header()) >= 3
