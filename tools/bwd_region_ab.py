#!/usr/bin/env python
"""A/B of the fp32 encoder backward: MSDA_KNOB_REGION_BWD = 0 (msda_bwd_tiled) against -1 (auto: msda_bwd_region), in one
process, on cfg2 encoder inputs (the bench's first encoder call, seed 1000).

    python tools/bwd_region_ab.py [--rounds 5] [--iters 30] [--config cfg2]

The two settings alternate `rounds` times; each round times `iters` L2-flushed calls of the backward (grad_value zero-fill
included, as in bench.py's enc_bwd_ms) with CUDA events.  Prints the median and spread (min..max of the round medians)
of each setting and the largest difference of grad_value, grad_loc and grad_attn between them, relative to each tensor's
largest magnitude."""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200 import _cabi  # noqa: E402
from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA  # noqa: E402
from uninext_b200.workloads import CONFIGS, make_inputs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--config", default="cfg2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bwd_region_ab.py needs a CUDA device")
    lib = _cabi.load()
    inp = make_inputs(CONFIGS[args.config], "enc", "cuda", seed=1000)
    a = (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"], inp["attention_weights"])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def call():
        return MSDA.ms_deform_attn_backward(*a, inp["grad_output"], 64)

    def round_ms(setting):
        lib.msda_set_knob(_cabi.KNOB_REGION_BWD, setting)
        xs = []
        for i in range(args.iters + 3):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                xs.append(e0.elapsed_time(e1))
        return statistics.median(xs)

    was = lib.msda_set_knob(_cabi.KNOB_REGION_BWD, -1000000)
    try:
        res = {0: [], -1: []}
        for _ in range(args.rounds):
            for s in (0, -1):
                res[s].append(round_ms(s))
        outs = {}
        for s in (0, -1):
            lib.msda_set_knob(_cabi.KNOB_REGION_BWD, s)
            outs[s] = [t.double() for t in call()]
        torch.cuda.synchronize()
    finally:
        lib.msda_set_knob(_cabi.KNOB_REGION_BWD, was)

    props = torch.cuda.get_device_properties(0)
    print(f"device: {props.name}, {props.multi_processor_count} SMs; {args.config} encoder backward, "
          f"{args.rounds} rounds x {args.iters} L2-flushed calls")
    for s, name in ((0, "tiled  (knob 0)"), (-1, "region (knob -1)")):
        xs = res[s]
        print(f"{name}: enc_bwd median {statistics.median(xs):.4f} ms, spread {min(xs):.4f} .. {max(xs):.4f} ms")
    print(f"speed-up: {statistics.median(res[0]) / statistics.median(res[-1]):.3f}x")
    for name, t0, t1 in zip(("grad_value", "grad_loc", "grad_attn"), outs[0], outs[-1]):
        print(f"{name}: max |region - tiled| / max |tiled| = {(t1 - t0).abs().max().item() / t0.abs().max().item():.3e}")


if __name__ == "__main__":
    main()
