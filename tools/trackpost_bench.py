#!/usr/bin/env python
"""The video trackers' per-frame detection selection (``select_track_detections``, msda_trackpost_f32, DESIGN.md
section 3.17) against the reference's chains (uninext_vid.py:1224-1250 inference_mot, :1380-1415 inference_vis, restated
line for line in tests/trackpost_case.py), in one process on one GPU.

    python tools/trackpost_bench.py [--rounds 5] [--iters 20]

Cases: one frame (B = 1), Q = 900 and 300, T = 256; the YTVIS (40 classes), OVIS (25) and BDD (8) prompt maps; MOT
(NMS 0.7, xyxy boxes in pixels) on BDD and VIS (NMS 0.9, normalised cxcywh) on YTVIS and OVIS, each with and without
the IoU branch; and a frame where no query passes the threshold (the top-1 fallback).  The inputs are tie-free and
shifted so that about a sixth of the queries pass the threshold (0.1 for MOT, 0.05 for VIS).  Both arms end where the
reference hands over to the tracker, with the kept count known on the host: the fused arm includes its one host read,
``int(count[0])``.  The two arms alternate `rounds` times; a round times `iters` calls, each between CUDA events
followed by a synchronise, and takes their median.  Prints medians, spread (min..max of the round medians), whether
the arms agree bitwise (queries, labels, scores, boxes), the card's name and power limit read in the same run, and one
JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import trackpost_case as tc  # noqa: E402
from uninext_b200.modules.detection_postprocess import select_track_detections  # noqa: E402

NMS = {"mot": 0.7, "vis": 0.9}
THRES = {"mot": 0.1, "vis": 0.05}
FORMAT = {"mot": "xyxy_pixels", "vis": "cxcywh"}


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
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trackpost_bench.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}; {a.rounds} rounds x {a.iters} calls")
    sizes = [(720, 1280)]
    # (name, path, Q, map, IoU branch, logit shift); the shifts leave about a sixth of the queries above the threshold
    shifts = {("mot", True): -8.0, ("mot", False): -6.1, ("vis", True): -9.6, ("vis", False): -6.9}
    cases = [(f"{p.upper()} {m.upper()} Q={q}{', IoU branch' if iou else ''}", p, q, m, iou, shifts[p, iou])
             for q in (900, 300) for p, m in (("mot", "bdd"), ("vis", "ytvis"), ("vis", "ovis")) for iou in (True, False)]
    cases += [("MOT BDD Q=900, IoU branch, no query passes", "mot", 900, "bdd", True, -12.0),
              ("VIS YTVIS Q=300, no query passes", "vis", 300, "ytvis", False, -12.0)]
    for seed, (name, path, Q, mname, iou, shift) in enumerate(cases):
        pmap = tc.MAPS[mname]()
        box_cls, box_pred, iou_pred = tc.make_inputs(1, Q, pmap, 256, iou, seed=seed, logit_shift=shift)
        thr = THRES[path]

        def fused():
            d = select_track_detections(box_cls, box_pred, pmap, iou_pred, score_thres=thr, nms_iou=NMS[path],
                                        box_format=FORMAT[path], ori_sizes=sizes)
            n = int(d.count[0])                             # the one host read per frame
            return d, n

        arms = {"fused": fused, "torch": lambda: tc.chain(path, box_cls, box_pred, pmap, iou_pred, thr, sizes)}

        def run_ms(fn):
            times = []
            for _ in range(a.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            return statistics.median(times)

        for fn in arms.values():                               # warm-up
            fn()
        torch.cuda.synchronize()
        res = {arm: [] for arm in arms}
        for _ in range(a.rounds):
            for arm, fn in arms.items():
                res[arm].append(run_ms(fn))
        (got, n), want = arms["fused"](), arms["torch"]()[0]
        agree = (n == want["query"].numel() and torch.equal(got.query_index[0, :n].long(), want["query"]) and
                 torch.equal(got.labels[0, :n].long(), want["labels"]) and
                 torch.equal(got.scores[0, :n], want["scores"]) and torch.equal(got.boxes[0, :n], want["boxes"]))
        prob = tc.convert_grounding_to_od_logits(box_cls, len(pmap), pmap)[0].sigmoid()
        if iou_pred is not None:
            prob = torch.sqrt(prob * iou_pred[0].sigmoid())
        cand = int((prob.max(1)[0] > thr).sum())
        med = {arm: statistics.median(v) for arm, v in res.items()}
        print(f"{name}: {cand} candidates, {n} kept; fused {med['fused']:.3f} ms "
              f"({min(res['fused']):.3f} .. {max(res['fused']):.3f}), torch {med['torch']:.3f} ms "
              f"({min(res['torch']):.3f} .. {max(res['torch']):.3f}), x{med['torch'] / med['fused']:.1f}; "
              f"{'agree' if agree else 'DIFFER'}")
        print(json.dumps({"case": name, "candidates": cand, "kept": n, "fused_ms": med["fused"],
                          "torch_ms": med["torch"], "fused_spread_ms": [min(res["fused"]), max(res["fused"])],
                          "torch_spread_ms": [min(res["torch"]), max(res["torch"])], "agree": agree, "device": dev}))


if __name__ == "__main__":
    main()
