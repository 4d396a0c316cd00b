"""Tile geometry of msda_bwd_region (uninext_b200/csrc/msda_region.cuh), restated in Python for the region tests.

The constants are read from the kernel header, so a change of the shipped halo or budgets changes the layouts the tests
check their premises against; a premise that no longer holds then fails on any machine, GPU or not."""
import os
import re

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "uninext_b200", "csrc",
                      "msda_region.cuh")
NAMES = ("kRegionEdge", "kRegionHalo", "kRegionWinRows", "kRegionStageRows", "kRegionSlots")


def region_constants():
    """{name: value} of the region kernel's tile constants, as msda_region.cuh defines them."""
    with open(HEADER) as fh:
        text = fh.read()
    found = dict(re.findall(r"constexpr int (kRegion\w+) = (\d+);", text))
    missing = [n for n in NAMES if n not in found]
    assert not missing, f"{HEADER} does not define {missing}"
    return {n: int(found[n]) for n in NAMES}


def window_layout(shapes):
    """[(window rows per level, staged per level, queries)] over the tiles of a level table that tiles [0, S), as the
    kernel lays them out: each level's window is the tile's region scaled to the level plus the halo; a level that would
    take the window past kRegionWinRows gets no rows; whole levels are staged from the last one down while they fit
    kRegionStageRows."""
    c = region_constants()
    R, halo, win_rows, stage_rows = c["kRegionEdge"], c["kRegionHalo"], c["kRegionWinRows"], c["kRegionStageRows"]
    href, wref = max(h for h, _ in shapes), max(w for _, w in shapes)
    def first(i, n, ref):              # region_first: the first pixel of a level whose centre lies in region i
        num = 2 * i * n * R - ref
        return 0 if num <= 0 else min(n, -(-num // (2 * ref)))
    out = []
    for ry in range(-(-href // R)):
        for rx in range(-(-wref // R)):
            rows, nw, nq = [], 0, 0
            for h, w in shapes:
                nq += (first(ry + 1, h, href) - first(ry, h, href)) * (first(rx + 1, w, wref) - first(rx, w, wref))
                wy0, wy1 = max(0, ry * R * h // href - halo), min(h, -(-(ry + 1) * R * h // href) + halo)
                wx0, wx1 = max(0, rx * R * w // wref - halo), min(w, -(-(rx + 1) * R * w // wref) + halo)
                n = (wy1 - wy0) * (wx1 - wx0)
                n = 0 if nw + n > win_rows else n
                rows.append(n)
                nw += n
            staged, tail = [False] * len(shapes), 0
            for lvl in reversed(range(len(shapes))):
                if tail + rows[lvl] > stage_rows:
                    break
                tail += rows[lvl]
                staged[lvl] = True
            out.append((rows, staged, nq))
    return out
