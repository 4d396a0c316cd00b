#!/usr/bin/env python
"""Per-kernel times of the fused image-text attention core (DESIGN.md section 3.11) in its three modes, from
torch.profiler in a run of its own.

    python tools/vlfuse_kernels.py [--calls 5] [--out DIR]

Runs ``vl_attention`` forward + backward (training mode, dropout 0.1) on [B, S, 8, 256] inputs at the cfg2 shapes
(B = 2, S = 22323, T = 256 and T = 32), in fp32, TF32 (torch.backends.cuda.matmul.allow_tf32) and bf16 (bf16 inputs),
`calls` times each after a warm-up call, with the profiler recording CUDA activity only.  For each shape and mode it
reports every vlf_* kernel's mean time per call (the sum of its launches in a call; the backward launches vlf_reduce
twice), their total, and that total's share per kernel.  Prints the card's name and power limit, read in the same run;
writes vlfuse_kernels.json and vlfuse_kernels.md under --out when given."""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.det_bench import card  # noqa: E402
from uninext_b200.modules import vl_fusion as vf  # noqa: E402

H, D, S = 8, 256, 22323
SHAPES = (("cfg2_T256", 2, 256), ("cfg2_T32", 2, 32))
MODES = (("fp32", torch.float32, False), ("tf32", torch.float32, True), ("bf16", torch.bfloat16, False))


def short(name):
    return name.split("<")[0].split("(")[0].split("::")[-1].split(" ")[-1]


def profile_mode(B, T, dtype, allow_tf32, calls):
    g = torch.Generator(device="cuda").manual_seed(T)
    q = (torch.randn(B, S, H, D, device="cuda", generator=g) * D ** -0.5).to(dtype)
    k, vv = torch.randn(B, T, H, D, device="cuda", generator=g).to(dtype), torch.randn(B, S, H, D, device="cuda", generator=g).to(dtype)
    vl = torch.randn(B, T, H, D, device="cuda", generator=g).to(dtype)
    mask = torch.ones(B, T, dtype=torch.int64, device="cuda")
    mask[-1, T // 2:] = 0
    bias = vf.text_bias(mask, T)
    go = (torch.randn_like(q), torch.randn_like(k))
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]

    def call():
        o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True)
        torch.autograd.backward((o_v, o_l), go)

    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = allow_tf32
    try:
        call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device="cuda").add_(1)      # the profiler can lose the first records of its window
            for _ in range(calls):
                call()
            torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    us, n = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if "vlf_" in e.name and e.device_time > 0:
            us[short(e.name)] += e.device_time
            n[short(e.name)] += 1
    per_call = {k: round(v / calls / 1e3, 3) for k, v in sorted(us.items(), key=lambda kv: -kv[1])}
    return per_call, {k: v / calls for k, v in n.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vlfuse_kernels needs a CUDA device"
    results = {"device": card(), "S": S, "calls": a.calls}
    lines = [f"Per-kernel time of one vl_attention forward + backward, ms ({results['device']}); S = {S}, H = {H}, "
             f"d = {D}, training mode, dropout 0.1", ""]
    for shape, B, T in SHAPES:
        for mode, dtype, allow_tf32 in MODES:
            ms, launches = profile_mode(B, T, dtype, allow_tf32, a.calls)
            total = sum(ms.values())
            results[f"{shape}_{mode}"] = {"kernels_ms": ms, "launches_per_call": launches, "total_ms": round(total, 3)}
            lines.append(f"{shape} (B = {B}, T = {T}), {mode}: total {total:.3f} ms")
            lines += [f"  {k:24s} {v:8.3f} ms  {100 * v / total:5.1f} %  x{launches[k]:g}" for k, v in ms.items()]
            lines.append("")
            torch.cuda.empty_cache()
    text = "\n".join(lines)
    print(text)
    print(json.dumps(results, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vlfuse_kernels.json"), "w") as fh:
            json.dump(results, fh, indent=1)
        with open(os.path.join(a.out, "vlfuse_kernels.md"), "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
