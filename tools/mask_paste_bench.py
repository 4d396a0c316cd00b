#!/usr/bin/env python
"""Mask pasting (``paste_masks``, msda_mask_paste_f32, DESIGN.md section 3.12) against the reference's torch chain, in one
process on one GPU.

    python tools/mask_paste_bench.py [--rounds 5] [--iters 10]

Cases: 100 and 300 instances of 200x336 stride-4 logits, crop 800x1333 (COCO's padded 800x1344 input), output 480x640 and
1080x1920, binary masks (uninext_img.py:474-479 + ddetrs.py:1060-1064); and the video shape, one track of 90x160 logits
(360x640 input) pasted to 720x1280 with `> 0.5` (uninext_vid.py:1264-1266), `--tracks` calls of one instance each.
The two arms alternate `rounds` times; a round times `iters` calls with CUDA events and takes their median.  Also
reported: each arm's peak allocation during one call above what was allocated before it, and how many output pixels
differ between the arms (all of them must lie within 1e-6 of the threshold in probability).  Prints medians, spread
(min..max of the round medians), the card's name and power limit read in the same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200.modules.mask_postprocess import paste_masks  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = f"{float(q.stdout.strip().splitlines()[0]):.0f} W"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        watts = "unknown"
    return f"{name}, power limit {watts}"


def chain_image(mask_pred_i, image_size, height, width, mask_stride=4, mask_thres=0.5):
    """uninext_img.py:474-479, then segmentation_postprocess (ddetrs.py:1060-1064), as the reference writes them."""
    N, C, H, W = mask_pred_i.shape
    mask = F.interpolate(mask_pred_i, size=(H*mask_stride, W*mask_stride), mode='bilinear', align_corners=False)
    mask = mask.sigmoid() > mask_thres
    mask = mask[:,:,:image_size[0],:image_size[1]]
    mask = F.interpolate(mask.float(), size=(height, width), mode='nearest')
    mask = mask.squeeze(1).byte()
    return mask


def chain_video(track_masks, image_size, ori_size, output_h, output_w):
    """uninext_vid.py:1264-1266 on the GPU (the reference moves the probabilities to merge_device first)."""
    track_masks = F.interpolate(track_masks,  size=(output_h*4, output_w*4) ,mode="bilinear", align_corners=False).sigmoid()
    track_masks = track_masks[:, :, :image_size[0],:image_size[1]] # crop the padding area
    track_masks = F.interpolate(track_masks, size=(ori_size[0], ori_size[1]), mode='nearest') # (1, 1, H, W)
    track_masks = (track_masks[:, 0] > 0.5)
    return track_masks


def probs(x, crop, outs):
    m = F.interpolate(x, size=(x.shape[2] * 4, x.shape[3] * 4), mode="bilinear", align_corners=False).sigmoid()
    return F.interpolate(m[:, :, :crop[0], :crop[1]], size=outs, mode="nearest")[:, 0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--tracks", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_paste_bench.py needs a CUDA device")
    print(f"device: {card()}; {a.rounds} rounds x {a.iters} calls")
    g = torch.Generator(device="cuda").manual_seed(0)

    cases = []
    for n in (100, 300):
        for outs in ((480, 640), (1080, 1920)):
            x = torch.rand(n, 1, 200, 336, device="cuda", generator=g) * 60 - 30
            cases.append((f"image I={n} 200x336 -> crop 800x1333 -> {outs[0]}x{outs[1]}", [x], (800, 1333), outs,
                          lambda xs, c=(800, 1333), o=outs: [chain_image(xs[0], c, *o)]))
    tracks = [torch.rand(1, 1, 90, 160, device="cuda", generator=g) * 60 - 30 for _ in range(a.tracks)]
    cases.append((f"video {a.tracks} tracks x (I=1 90x160 -> crop 360x640 -> 720x1280)", tracks, (360, 640), (720, 1280),
                  lambda xs: [chain_video(t, (360, 640), (720, 1280), 90, 160) for t in xs]))

    for name, xs, crop, outs, chain in cases:
        arms = {"fused": lambda xs, crop=crop, outs=outs: [paste_masks(t, crop, outs) for t in xs], "torch": chain}

        def run_ms(fn):
            times = []
            for _ in range(a.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(xs)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            return statistics.median(times)

        peak = {}
        for arm, fn in arms.items():                                 # warm-up, peak memory
            fn(xs)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = fn(xs)
            torch.cuda.synchronize()
            peak[arm] = torch.cuda.max_memory_allocated() - base
            del out
        res = {arm: [] for arm in arms}
        for _ in range(a.rounds):
            for arm, fn in arms.items():
                res[arm].append(run_ms(fn))
        got, want = arms["fused"](xs), chain(xs)
        differ = near = 0
        for t, gb, wb in zip(xs, got, want):
            d = gb != wb.bool()
            differ += int(d.sum())
            near += int((d & ((probs(t, crop, outs) - 0.5).abs() <= 1e-6)).sum())
        med = {arm: statistics.median(v) for arm, v in res.items()}
        print(f"{name}: fused {med['fused']:.3f} ms ({min(res['fused']):.3f} .. {max(res['fused']):.3f}), "
              f"torch {med['torch']:.3f} ms ({min(res['torch']):.3f} .. {max(res['torch']):.3f}), "
              f"x{med['torch'] / med['fused']:.1f}; peak {peak['fused'] / 2**20:.1f} MiB against "
              f"{peak['torch'] / 2**20:.1f} MiB; {differ} pixels differ, {near} of them within 1e-6 of the threshold")
        print(json.dumps({"case": name, "fused_ms": med["fused"], "torch_ms": med["torch"],
                          "fused_spread_ms": [min(res["fused"]), max(res["fused"])],
                          "torch_spread_ms": [min(res["torch"]), max(res["torch"])],
                          "fused_peak_bytes": peak["fused"], "torch_peak_bytes": peak["torch"],
                          "pixels_differ": differ, "pixels_differ_near_threshold": near, "device": card()}))
        del got, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
