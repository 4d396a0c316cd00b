#!/usr/bin/env python
"""COCO RLE of instance masks (``paste_masks_rle`` / ``encode_masks_rle``, DESIGN.md section 3.14) against the reference
path, in one process on one GPU.

    python tools/mask_rle_bench.py [--rounds 5] [--iters 5]

Arms, each from the same logits to the list of ``{"size", "counts"}`` dicts:
  fused      paste_masks_rle (logits -> strings, no full-resolution mask);
  two-step   paste_masks, then encode_masks_rle on the device masks;
  reference  the reference's torch chain (bilinear, sigmoid, crop, nearest, > 0.5), ``.cpu()``, and per instance
             pycocotools.mask.encode when pycocotools imports, otherwise the numpy encoder of tests/coco_rle.py
             (the JSON line names the one that ran).
Cases: 100 instances to 480x640 (COCO evaluation), 300 to 1080x1920, and 10 video tracks of 90x160 logits (crop 360x640)
to 720x1280.  The logits are mask-like: a few smooth blobs per instance.  The arms alternate `rounds` times; a round
times `iters` calls with a host clock around work that ends in a synchronisation (every arm returns host bytes) and takes
their median.  Also reported: each arm's peak device allocation above what was allocated before the call, and whether
all strings are equal.  Prints medians, spread (min..max of the round medians), the card's name and power limit read in
the same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from uninext_b200.modules.mask_postprocess import encode_masks_rle, paste_masks, paste_masks_rle  # noqa: E402

try:
    from pycocotools import mask as mask_util
    ENCODER = "pycocotools"
except ImportError:
    mask_util = None
    ENCODER = "numpy (tests/coco_rle.py)"
    from tests.coco_rle import encode_np  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        watts = f"{float(q.stdout.strip().splitlines()[0]):.0f} W"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        watts = "unknown"
    return f"{name}, power limit {watts}"


def blob_logits(i, hs, ws, gen):
    """A few smooth blobs per instance: positive inside, negative outside."""
    yy, xx = torch.meshgrid(torch.arange(hs, device="cuda", dtype=torch.float32),
                            torch.arange(ws, device="cuda", dtype=torch.float32), indexing="ij")
    out = torch.full((i, 1, hs, ws), -8.0, device="cuda")
    for k in range(i):
        for _ in range(int(torch.randint(1, 4, (1,), generator=gen))):
            cy, cx = float(torch.rand(1, generator=gen)) * hs, float(torch.rand(1, generator=gen)) * ws
            r = 3 + float(torch.rand(1, generator=gen)) * hs / 4
            out[k, 0] = torch.maximum(out[k, 0], 8.0 * (1 - ((yy - cy) ** 2 + (xx - cx) ** 2) / r ** 2))
    return out


def reference(x, crop, outs):
    """uninext_vid.py:1425-1432 for all instances at once (the chain of paste_masks), then the host encoder."""
    m = F.interpolate(x, size=(x.shape[2] * 4, x.shape[3] * 4), mode="bilinear", align_corners=False).sigmoid()
    m = m[:, :, :crop[0], :crop[1]]
    m = F.interpolate(m, size=outs, mode="nearest")[:, 0] > 0.5
    host = m.cpu().numpy()
    if mask_util is not None:
        return [mask_util.encode(np.array(host[k][:, :, None], order="F", dtype="uint8"))[0] for k in range(len(host))]
    return [encode_np(host[k]) for k in range(len(host))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_rle_bench.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}; reference encoder: {ENCODER}; {a.rounds} rounds x {a.iters} calls")
    gen = torch.Generator().manual_seed(0)
    cases = [("image I=100 200x336 -> crop 800x1333 -> 480x640", [blob_logits(100, 200, 336, gen)], (800, 1333),
              (480, 640)),
             ("image I=300 200x336 -> crop 800x1333 -> 1080x1920", [blob_logits(300, 200, 336, gen)], (800, 1333),
              (1080, 1920)),
             ("video 10 tracks x (I=1 90x160 -> crop 360x640 -> 720x1280)",
              [blob_logits(1, 90, 160, gen) for _ in range(10)], (360, 640), (720, 1280))]

    for name, xs, crop, outs in cases:
        arms = {"fused": lambda: [r for x in xs for r in paste_masks_rle(x, crop, outs)],
                "two_step": lambda: [r for x in xs for r in encode_masks_rle(paste_masks(x, crop, outs))],
                "reference": lambda: [r for x in xs for r in reference(x, crop, outs)]}

        def run_ms(fn):
            times = []
            for _ in range(a.iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times.append((time.perf_counter() - t0) * 1e3)
            return statistics.median(times)

        peak, result = {}, {}
        for arm, fn in arms.items():                                 # warm-up, peak memory, results
            fn()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            result[arm] = fn()
            torch.cuda.synchronize()
            peak[arm] = torch.cuda.max_memory_allocated() - base
        res = {arm: [] for arm in arms}
        for _ in range(a.rounds):
            for arm, fn in arms.items():
                res[arm].append(run_ms(fn))
        want = [(list(r["size"]), r["counts"]) for r in result["reference"]]
        equal = all([(list(r["size"]), r["counts"]) for r in result[arm]] == want for arm in ("fused", "two_step"))
        med = {arm: statistics.median(v) for arm, v in res.items()}
        print(f"{name}: " + ", ".join(f"{arm} {med[arm]:.2f} ms ({min(v):.2f} .. {max(v):.2f}), peak "
                                      f"{peak[arm] / 2**20:.1f} MiB" for arm, v in res.items()) +
              f"; reference / fused x{med['reference'] / med['fused']:.1f}; all strings equal: {equal}")
        print(json.dumps({"case": name, "ms": med, "spread_ms": {k: [min(v), max(v)] for k, v in res.items()},
                          "peak_bytes": peak, "strings_equal": equal, "reference_encoder": ENCODER,
                          "string_bytes_per_instance": statistics.mean(len(r["counts"]) for r in result["fused"]),
                          "device": dev}))
        del result
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
