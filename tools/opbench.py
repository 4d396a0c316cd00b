#!/usr/bin/env python
"""Micro-benchmark of single MSDeformAttn calls (CUDA events, L2 flushed between iterations).
    python tools/opbench.py --config cfg2 --kind enc --dtype fp32 --iters 20
Also a short command to run under a profiler."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA  # noqa: E402
from uninext_b200.workloads import CONFIGS, algorithmic_bytes, make_inputs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--config", default="cfg2")
ap.add_argument("--kind", default="enc")
ap.add_argument("--dtype", default="fp32")
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--jitter", type=float, default=2.0)
ap.add_argument("--no-flush", action="store_true")
ap.add_argument("--ref", action="store_true", help="time the reference's own CUDA kernels (oracle/_ref) instead")
a = ap.parse_args()

cfg = CONFIGS[a.config]
dt = torch.float32 if a.dtype == "fp32" else torch.bfloat16
inp = make_inputs(cfg, a.kind, "cuda", dtype=dt, seed=0, jitter_px=a.jitter)
args = (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"], inp["attention_weights"])
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
if a.ref:
    from oracle import refcuda
    assert refcuda.available() and a.dtype == "fp32"
    ref_out = torch.empty_like(inp["grad_output"])
    ref_g = (torch.empty_like(args[0]), torch.empty_like(args[3]), torch.empty_like(args[4]))

    class MSDA:  # noqa: F811  (same call shape; at::zeros / zeros_like of the reference wrapper are included)
        @staticmethod
        def ms_deform_attn_forward(v, ss, lsi, loc, attn, step):
            return refcuda.forward(v, ss, lsi, loc, attn)

        @staticmethod
        def ms_deform_attn_backward(v, ss, lsi, loc, attn, go, step):
            return refcuda.backward(v, ss, lsi, loc, attn, go, outs=ref_g)
fw, bw = [], []
for i in range(a.warmup + a.iters):
    if not a.no_flush:
        flush.zero_()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    out = MSDA.ms_deform_attn_forward(*args, 64)
    e[1].record()
    g = MSDA.ms_deform_attn_backward(*args, inp["grad_output"], 64)
    e[2].record()
    torch.cuda.synchronize()
    if i >= a.warmup:
        fw.append(e[0].elapsed_time(e[1])); bw.append(e[1].elapsed_time(e[2]))
fw.sort(); bw.sort()
mf, mb = fw[len(fw) // 2], bw[len(bw) // 2]
smp = cfg.samples(a.kind)
el = 4 if a.dtype == "fp32" else 2
print(json.dumps({"impl": "reference-cuda" if a.ref else "b200", "config": cfg.name, "kind": a.kind, "dtype": a.dtype, "samples": smp,
                  "fwd_ms": round(mf, 4), "bwd_ms": round(mb, 4),
                  "fwd_gsamples": round(smp / mf / 1e6, 2), "bwd_gsamples": round(smp / mb / 1e6, 2),
                  "fwd_alg_GBps": round(algorithmic_bytes(cfg, a.kind, el, "fwd") / mf / 1e6, 1),
                  "bwd_alg_GBps": round(algorithmic_bytes(cfg, a.kind, el, "bwd") / mb / 1e6, 1)}))
