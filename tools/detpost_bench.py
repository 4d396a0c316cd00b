#!/usr/bin/env python
"""Detection post-processing (``postprocess_detections``, msda_detpost_f32, DESIGN.md section 3.13) against the
reference's chain (uninext_img.py:389-472: convert_grounding_to_od_logits, sigmoid / sqrt, torchvision batched_nms,
topk, cxcywh -> xyxy, Boxes.scale), in one process on one GPU.

    python tools/detpost_bench.py [--rounds 5] [--iters 20]

Cases: B = 1, Q = 900, T = 256 with an 80-class COCO-shaped positive map and the IoU branch, with and without NMS;
B = 1, Q = 900 grounding ({1: [0]}, max_num_inst = 1); B = 8, Q = 300 (COCO map, NMS).  The two arms alternate `rounds`
times; a round times `iters` calls, each between CUDA events followed by a synchronise, and takes their median.  Prints
medians, spread (min..max of the round medians), whether the arms agree, the card's name and power limit read in the
same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torchvision

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200.modules.detection_postprocess import postprocess_detections  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = f"{float(q.stdout.strip().splitlines()[0]):.0f} W"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        watts = "unknown"
    return f"{name}, power limit {watts}"


def coco_like_map():
    pmap, t = {}, 1
    for c in range(80):
        n = 1 + (c % 7 == 3) + (c % 11 == 5)
        pmap[c + 1] = list(range(t, t + n))
        t += n + 1
    return pmap


def convert_grounding_to_od_logits(logits, num_classes, positive_map):
    """uninext_img.py:598-613 (MEAN)."""
    scores = torch.zeros(logits.shape[0], logits.shape[1], num_classes).to(logits.device)
    for label_j in positive_map:
        scores[:, :, label_j - 1] = logits[:, :, torch.LongTensor(positive_map[label_j])].mean(-1)
    return scores


def box_cxcywh_to_xyxy(x):
    x_c, y_c, w, h = x.unbind(-1)
    return torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)


def chain(box_cls, box_pred, pmap, image_sizes, iou_pred, nms_iou, max_num_inst):
    """uninext_img.py:389-472 per image, as the reference writes it (masks aside)."""
    C = len(pmap)
    out = []
    for i in range(box_cls.shape[0]):
        logits = convert_grounding_to_od_logits(box_cls[i].unsqueeze(0), C, pmap)[0]
        prob = logits.sigmoid()
        if iou_pred is not None:
            prob = torch.sqrt(prob * iou_pred[i].sigmoid())
        bp = box_pred[i]
        if nms_iou is not None:
            nms_scores, idxs = torch.max(prob, 1)
            keep = torchvision.ops.batched_nms(box_cxcywh_to_xyxy(bp), nms_scores, idxs, nms_iou)
            prob, bp = prob[keep], bp[keep]
        num_inst = min(max_num_inst, len(prob.view(-1)))
        v, ix = torch.topk(prob.view(-1), num_inst, dim=0)
        rows = torch.div(ix, C, rounding_mode='floor')
        boxes = box_cxcywh_to_xyxy(bp[rows])
        boxes[:, 0::2] *= image_sizes[i][1]
        boxes[:, 1::2] *= image_sizes[i][0]
        out.append((v, ix % C, boxes))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detpost_bench.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}; {a.rounds} rounds x {a.iters} calls")
    g = torch.Generator(device="cuda").manual_seed(0)
    coco = coco_like_map()

    def inputs(B, Q):
        return (torch.randn(B, Q, 256, device="cuda", generator=g) * 3,
                torch.cat((torch.rand(B, Q, 2, device="cuda", generator=g),
                           torch.rand(B, Q, 2, device="cuda", generator=g) * 0.4 + 0.02), -1),
                torch.randn(B, Q, 1, device="cuda", generator=g))

    cases = [("B=1 Q=900 COCO, IoU branch, NMS 0.7, top 100", 1, 900, coco, 0.7, 100),
             ("B=1 Q=900 COCO, IoU branch, no NMS, top 100", 1, 900, coco, None, 100),
             ("B=1 Q=900 grounding {1: [0]}, NMS 0.7, top 1", 1, 900, {1: [0]}, 0.7, 1),
             ("B=8 Q=300 COCO, IoU branch, NMS 0.7, top 100", 8, 300, coco, 0.7, 100)]
    for name, B, Q, pmap, nms, k in cases:
        box_cls, box_pred, iou_pred = inputs(B, Q)
        sizes = [(800, 1333)] * B
        arms = {"fused": lambda: postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, nms, k),
                "torch": lambda: chain(box_cls, box_pred, pmap, sizes, iou_pred, nms, k)}

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
        got, want = arms["fused"](), arms["torch"]()
        agree = all(torch.equal(got.labels[b, :int(got.count[b])].long(), want[b][1]) and
                    torch.equal(got.boxes[b, :int(got.count[b])], want[b][2]) for b in range(B))
        med = {arm: statistics.median(v) for arm, v in res.items()}
        print(f"{name}: fused {med['fused']:.3f} ms ({min(res['fused']):.3f} .. {max(res['fused']):.3f}), "
              f"torch {med['torch']:.3f} ms ({min(res['torch']):.3f} .. {max(res['torch']):.3f}), "
              f"x{med['torch'] / med['fused']:.1f}; labels and boxes {'agree' if agree else 'DIFFER'}")
        print(json.dumps({"case": name, "fused_ms": med["fused"], "torch_ms": med["torch"],
                          "fused_spread_ms": [min(res["fused"]), max(res["fused"])],
                          "torch_spread_ms": [min(res["torch"]), max(res["torch"])], "agree": agree, "device": dev}))


if __name__ == "__main__":
    main()
