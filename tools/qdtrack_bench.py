#!/usr/bin/env python
"""The QuasiDense tracker's association step (``QuasiDenseTracker.match``, msda_qdtrack_match_f32, DESIGN.md section
3.19) against the reference's host-driven chain (models/tracker.py:304-503, restated in tests/qdtrack_case.py
ReferenceChain) on CUDA, in one process on one GPU.

    python tools/qdtrack_bench.py [--rounds 5] [--frames 20]

Cases: n in {25, 100, 250} detections per frame, D = 256, the BDD settings, sequences of tests/qdtrack_case.py's
random generator with about 100 live tracklets (plus last frame's backdrops).  Each round runs a fresh tracker of each
arm over the same sequence (after a warm-up sequence), both ending every frame with the ids on the host; every frame is
timed with CUDA events between two synchronisations, and the arms alternate `rounds` times.  Prints the per-frame
median over all frames and rounds with the spread (min..max of the round medians), whether the ids agreed on every
frame, the card's name and power limit read in the same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import qdtrack_case as qc  # noqa: E402
from uninext_b200.modules.tracker import QuasiDenseTracker  # noqa: E402


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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qdtrack_bench.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}; {a.rounds} rounds x {a.frames} frames")
    for n in (25, 100, 250):
        seq = [tuple(t.cuda() for t in fr) for fr in qc.random_sequence(n, max(n, 124), frames=a.frames, dim=qc.DIM)]
        seq = [tuple(t[:n] for t in fr) for fr in seq]
        warm = [tuple(t[:n].cuda() for t in fr) for fr in qc.random_sequence(n + 1, max(n, 124), frames=3, dim=qc.DIM)]

        def fused(frames, times):
            tr = QuasiDenseTracker(**qc.BDD)
            out = []
            for f, (b, s, l, e) in enumerate(frames):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                _, _, ids, idx = tr.match(torch.cat((b, s[:, None]), 1), l, e, f, list(range(s.shape[0])))
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                out.append((idx, ids.tolist(), len(tr.tracklets()) if f == len(frames) - 1 else None))
            return out

        def chain(frames, times):
            ref = qc.ReferenceChain(**qc.BDD)
            out = []
            for f, (b, s, l, e) in enumerate(frames):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                order, keep, ids = ref.step(b, s, l, e, f)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                out.append(([p for p in keep], ids, len(ref.tracks) if f == len(frames) - 1 else None))
            return out

        arms = {"fused": fused, "reference": chain}
        for fn in arms.values():
            fn(warm, [])
        per_round = {k: [] for k in arms}
        every = {k: [] for k in arms}
        outs = {}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                times = []
                outs[k] = fn(seq, times)
                every[k] += times
                per_round[k].append(statistics.median(times))
        agree = outs["fused"] == outs["reference"]
        med = {k: statistics.median(v) for k, v in every.items()}
        live = outs["fused"][-1][2]
        name = f"n={n}, D={qc.DIM}, {live} live tracklets at the end"
        print(f"{name}: fused {med['fused']:.3f} ms/frame ({min(per_round['fused']):.3f} .. "
              f"{max(per_round['fused']):.3f}), reference {med['reference']:.2f} ms/frame "
              f"({min(per_round['reference']):.2f} .. {max(per_round['reference']):.2f}), "
              f"x{med['reference'] / med['fused']:.1f}; ids {'agree on every frame' if agree else 'DIFFER'}")
        print(json.dumps({"case": name, "fused_ms": med["fused"], "reference_ms": med["reference"],
                          "fused_round_medians_ms": per_round["fused"],
                          "reference_round_medians_ms": per_round["reference"], "agree": agree, "device": dev}))


if __name__ == "__main__":
    main()
