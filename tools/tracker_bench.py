#!/usr/bin/env python
"""The IDOL tracker's association step (``IDOLTracker.match``, msda_idol_match_f32, DESIGN.md section 3.18) against the
reference's host-driven chain (models/tracker.py:17-298, restated in tests/tracker_case.py ReferenceChain) on CUDA, in
one process on one GPU.

    python tools/tracker_bench.py [--rounds 3] [--frames 20]

Cases: n in {25, 100, 250} detections per frame at YTVIS (120 x 216) and OVIS (180 x 320) stride-4 mask sizes, D = 64,
the VIS settings with (long_match, frame_weight, temporal_weight) = (T, T, T).  Each round runs a fresh tracker of each
arm over the same 20-frame sequence (after a warm-up sequence), both ending every frame with the ids on the host, and
times the whole sequence with CUDA events; the arms alternate `rounds` times.  Prints the per-frame median over the
rounds with the spread (min..max), whether the ids agreed on every frame, the card's name and power limit read in the
same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import tracker_case as tc  # noqa: E402
from uninext_b200.modules.tracker import IDOLTracker  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = f"{float(q.stdout.strip().splitlines()[0]):.0f} W"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        watts = "unknown"
    return f"{name}, power limit {watts}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tracker_bench.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}; {a.rounds} rounds x {a.frames} frames")
    flags = (True, True, True)
    for size, (h, w) in (("YTVIS", (120, 216)), ("OVIS", (180, 320))):
        for n in (25, 100, 250):
            seq = [tuple(t.cuda() for t in fr) for fr in tc.random_sequence(n, n, h, w, frames=a.frames)]
            warm = [tuple(t.cuda() for t in fr) for fr in tc.random_sequence(n + 1, n, h, w, frames=2)]
            boxes = [torch.cat((torch.rand(s.shape[0], 4, device="cuda"), s[:, None]), 1) for s, _, _ in seq]

            def fused(frames, bxs=None):
                tr = IDOLTracker(**tc.settings(flags))
                out = []
                for f, (s, m, e) in enumerate(frames):
                    b = bxs[f] if bxs else torch.cat((torch.zeros(s.shape[0], 4, device="cuda"), s[:, None]), 1)
                    _, _, ids, idx = tr.match(b, s, m, e, f, list(range(s.shape[0])))
                    out.append((idx, ids.tolist()))
                return out

            def chain(frames, bxs=None):
                ref = tc.ReferenceChain(**tc.settings(flags))
                return [ref.step(s, m, e, f) for f, (s, m, e) in enumerate(frames)]

            arms = {"fused": fused, "reference": chain}
            for fn in arms.values():
                fn(warm)
            torch.cuda.synchronize()
            res = {k: [] for k in arms}
            outs = {}
            for _ in range(a.rounds):
                for k, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    outs[k] = fn(seq, boxes)
                    e1.record()
                    torch.cuda.synchronize()
                    res[k].append(e0.elapsed_time(e1) / len(seq))
            agree = outs["fused"] == outs["reference"]
            med = {k: statistics.median(v) for k, v in res.items()}
            name = f"{size} {h}x{w}, n={n}"
            print(f"{name}: fused {med['fused']:.3f} ms/frame ({min(res['fused']):.3f} .. {max(res['fused']):.3f}), "
                  f"reference {med['reference']:.2f} ms/frame ({min(res['reference']):.2f} .. "
                  f"{max(res['reference']):.2f}), x{med['reference'] / med['fused']:.0f}; ids "
                  f"{'agree on every frame' if agree else 'DIFFER'}")
            print(json.dumps({"case": name, "fused_ms": med["fused"], "reference_ms": med["reference"],
                              "fused_spread_ms": [min(res["fused"]), max(res["fused"])],
                              "reference_spread_ms": [min(res["reference"]), max(res["reference"])], "agree": agree,
                              "device": dev}))


if __name__ == "__main__":
    main()
