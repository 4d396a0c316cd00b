#!/usr/bin/env python
"""Cost of the deterministic backward (msda_backward_det_*, DESIGN.md section 3.10) against the default one, in one process.

    python tools/det_bench.py [--rounds 5] [--iters 20] [--steps 5] [--config cfg2]

On the bench's inputs (first encoder call seed 1000, first decoder call seed 1100; bench.py build_calls), for fp32 and
bf16:
  * one call's backward, default vs deterministic: the two modes alternate `rounds` times, each round times `iters`
    L2-flushed calls with CUDA events (grad_value zero-fill, workspace query and allocation included);
  * the 12-call step (6 encoder + 6 decoder calls, forward and backward) in both modes, alternating, `steps` timed steps
    per round;
  * the workspace each call uses, and the largest |deterministic - default| of grad_value relative to its largest
    magnitude.
Prints medians and spread (min..max of the round medians), and the card's name and power limit read in the same run."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200 import _cabi  # noqa: E402
from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA  # noqa: E402
from uninext_b200.workloads import CONFIGS, make_inputs  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = f"{float(q.stdout.strip().splitlines()[0]):.0f} W"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        watts = "unknown"
    return f"{name}, power limit {watts}"


def args_of(c):
    return (c["value"], c["spatial_shapes"], c["level_start_index"], c["sampling_locations"], c["attention_weights"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--config", default="cfg2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("det_bench.py needs a CUDA device")
    lib = _cabi.load()
    cfg = CONFIGS[a.config]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print(f"device: {card()}; {a.config}, {a.rounds} rounds")

    for dtype in (torch.float32, torch.bfloat16):
        tag = "fp32" if dtype == torch.float32 else "bf16"
        calls = [make_inputs(cfg, "enc", "cuda", dtype=dtype, seed=1000 + i) for i in range(6)]
        calls += [make_inputs(cfg, "dec", "cuda", dtype=dtype, seed=1100 + i) for i in range(6)]

        def bwd(c, det):
            return MSDA.ms_deform_attn_backward(*args_of(c), c["grad_output"], 64, deterministic=det)

        def call_ms(c, det):
            xs = []
            for i in range(a.iters + 3):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                bwd(c, det)
                e1.record()
                torch.cuda.synchronize()
                if i >= 3:
                    xs.append(e0.elapsed_time(e1))
            return statistics.median(xs)

        def step_ms(det):
            def step():
                for c in calls:
                    MSDA.ms_deform_attn_forward(*args_of(c), 64)
                    bwd(c, det)
            step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / a.steps

        for kind, c in (("enc", calls[0]), ("dec", calls[6])):
            res = {False: [], True: []}
            for _ in range(a.rounds):
                for det in (False, True):
                    res[det].append(call_ms(c, det))
            n, s, m, d = c["value"].shape
            dims = (n, s, m, d, c["spatial_shapes"].shape[0], c["sampling_locations"].shape[1],
                    c["sampling_locations"].shape[4])
            ws = MSDA._det_workspace(lib, c["value"], dims).numel()
            g0 = bwd(c, False)[0].double()
            g1 = bwd(c, True)[0].double()
            diff = (g1 - g0).abs().max().item() / g0.abs().max().item()
            med0, med1 = statistics.median(res[False]), statistics.median(res[True])
            print(f"{tag} {kind} backward: default {med0:.4f} ms ({min(res[False]):.4f} .. {max(res[False]):.4f}), "
                  f"deterministic {med1:.4f} ms ({min(res[True]):.4f} .. {max(res[True]):.4f}), x{med1 / med0:.2f}; "
                  f"workspace {ws / 2**20:.1f} MiB; grad_value max |det - default| / scale {diff:.2e}")

        res = {False: [], True: []}
        for _ in range(a.rounds):
            for det in (False, True):
                res[det].append(step_ms(det))
        med0, med1 = statistics.median(res[False]), statistics.median(res[True])
        print(f"{tag} 12-call step: default {med0:.3f} ms ({min(res[False]):.3f} .. {max(res[False]):.3f}), "
              f"deterministic {med1:.3f} ms ({min(res[True]):.3f} .. {max(res[True]):.3f}), x{med1 / med0:.2f}")
        del calls
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
