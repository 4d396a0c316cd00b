#!/usr/bin/env python
"""The early-fusion block (BiAttentionBlock, DESIGN.md section 3.11): fused kernels against the torch composition of the
same maths (the reference's order of operations), in one process.

    python tools/vlfuse_bench.py [--rounds 3] [--iters 5] [--out DIR]

UNINEXT dims (v 256, l 768, embed 2048, 8 heads), B = 2, S = 22323 (cfg2), T = 256 and T = 32, training mode
(dropout 0.1).  For each T and each path: forward, and forward + backward, timed with CUDA events over `iters` calls,
the two paths alternating `rounds` times; medians and the spread of the round medians; peak memory of one forward +
backward above the inputs and parameters.  Prints the card's name and power limit, read in the same run; writes a
JSON copy under --out when given."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.det_bench import card  # noqa: E402
from uninext_b200.modules import vl_fusion as vf  # noqa: E402


def run(blk, v, l, mask, fused, backward):
    """One call of the block; fused=False runs the same module on the torch composition."""
    if fused:
        out_v, out_l = blk(v, l, mask)
    else:
        orig = vf.fused_supported
        vf.fused_supported = lambda *a, **k: False
        try:
            out_v, out_l = blk(v, l, mask)
        finally:
            vf.fused_supported = orig
    if backward:
        (out_v.sum() + out_l.sum()).backward()


def time_it(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--S", type=int, default=22323)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vlfuse_bench needs a CUDA device"
    torch.manual_seed(0)
    results = {"device": card(), "S": a.S, "B": 2}
    blk = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6).cuda().train()
    for T in (256, 32):
        v = torch.randn(2, a.S, 256, device="cuda", requires_grad=True)
        l = torch.randn(2, T, 768, device="cuda", requires_grad=True)
        mask = torch.ones(2, T, dtype=torch.int64, device="cuda")
        mask[1, T // 2:] = 0
        for backward in (False, True):
            times = {True: [], False: []}
            for _ in range(a.rounds):
                for fused in (True, False):
                    times[fused].append(time_it(lambda: run(blk, v, l, mask, fused, backward), a.iters))
            for fused in (True, False):
                key = f"T{T}_{'fwd_bwd' if backward else 'fwd'}_{'fused' if fused else 'torch'}_ms"
                results[key] = round(statistics.median(times[fused]), 3)
                results[key + "_spread"] = [round(min(times[fused]), 3), round(max(times[fused]), 3)]
        for fused in (True, False):
            blk.zero_grad(set_to_none=True)
            v.grad = l.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            run(blk, v, l, mask, fused, True)
            torch.cuda.synchronize()
            results[f"T{T}_peak_MiB_{'fused' if fused else 'torch'}"] = round(
                (torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        del v, l
    print(json.dumps(results, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vlfuse_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
