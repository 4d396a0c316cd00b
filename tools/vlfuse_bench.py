#!/usr/bin/env python
"""The early-fusion block (BiAttentionBlock, DESIGN.md section 3.11): fused kernels against the torch composition of the
same maths (the reference's order of operations), in one process.

    python tools/vlfuse_bench.py [--rounds 3] [--iters 5] [--out DIR]

UNINEXT dims (v 256, l 768, embed 2048, 8 heads), B = 2, S = 22323 (cfg2), T = 256 and T = 32, training mode
(dropout 0.1).  Four arms: fused fp32, fused TF32, torch fp32 and torch TF32 (TF32 = torch.backends.cuda.matmul.allow_tf32,
which the fused path and the torch einsums both follow).  For each T and arm: the block's forward, and forward +
backward, timed with CUDA events over `iters` calls, the arms alternating `rounds` times (medians and the spread of the
round medians); peak memory of one block forward + backward; the attention core alone (``vl_attention`` on
[B, S, 8, 256] inputs, forward + backward) with its achieved TFLOP/s from the FLOP count 2 S T d B H per S x T x d
product (4 in the forward, 10 in the backward); and, at T = 256, the largest relative difference of each of the core's
six outputs (O_v, O_l, dQ, dK, dVv, dVl) against an fp64 restatement.  Prints the card's name and power limit, read in
the same run; writes a JSON copy under --out when given."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.det_bench import card  # noqa: E402
from uninext_b200.modules import vl_fusion as vf  # noqa: E402


ARMS = (("fused", True, False), ("fused_tf32", True, True), ("torch", False, False), ("torch_tf32", False, True))
H, D = 8, 256


def core_flops(B, S, T, backward):
    """FLOPs of the S x T x d products of the attention core: 4 in the forward, 10 in the backward."""
    return 2 * S * T * D * B * H * (14 if backward else 4)


def set_tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on


def core(q, k, vv, vl, bias, fused, go):
    """Forward + backward of the attention core alone."""
    leaves = [t.detach().requires_grad_(True) for t in (q, k, vv, vl)]
    if fused:
        o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True)
    else:
        o_v, o_l = vf.vl_attention_torch(*leaves, bias, True, True, 0.1, True)
    if go is None:
        return o_v, o_l, leaves
    torch.autograd.backward((o_v, o_l), go)
    return o_v, o_l, leaves


def core_errors(q, k, vv, vl, bias, tf32):
    """Largest |fused - fp64| / max |fp64| of the six core outputs, without dropout."""
    go = (torch.randn_like(q), torch.randn_like(k))
    set_tf32(tf32)
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, k, vv, vl)]
    got = list(vf.vl_attention(*leaves, bias, True, True, 0.0, False))
    got += list(torch.autograd.grad(got, leaves, go))
    set_tf32(False)
    leaves = [t.detach().double().requires_grad_(True) for t in (q, k, vv, vl)]
    x = torch.einsum("bshd,bthd->bhst", *leaves[:2]).clamp(-50000, 50000)
    p_l = (x.transpose(2, 3) - x.transpose(2, 3).max(dim=-1, keepdim=True)[0]).softmax(dim=-1)
    b = bias[:, None, None, :].double()
    masked = float(torch.tensor(-9e15, dtype=torch.float32))
    p_v = (x + torch.where(b < -1e15, masked - x, b).detach()).softmax(dim=-1)
    want = [torch.einsum("bhst,bthd->bshd", p_v, leaves[3]), torch.einsum("bhts,bshd->bthd", p_l, leaves[2])]
    want += list(torch.autograd.grad(want, leaves, [g.double() for g in go]))
    return {n: float((g.detach().double() - w.detach()).abs().max() / w.detach().abs().max()) for n, g, w in
            zip(("O_v", "O_l", "dQ", "dK", "dVv", "dVl"), got, want)}


def run(blk, v, l, mask, fused, backward):
    """One call of the block; fused=False runs the same module on the torch composition."""
    if fused:
        out_v, out_l = blk(v, l, mask)
    else:
        orig = vf.fused_supported
        vf.fused_supported = lambda *a, **k: False
        try:
            out_v, out_l = blk(v, l, mask)
        finally:
            vf.fused_supported = orig
    if backward:
        (out_v.sum() + out_l.sum()).backward()


def time_it(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--S", type=int, default=22323)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vlfuse_bench needs a CUDA device"
    torch.manual_seed(0)
    results = {"device": card(), "S": a.S, "B": 2}
    blk = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6).cuda().train()
    old = torch.backends.cuda.matmul.allow_tf32
    for T in (256, 32):
        v = torch.randn(2, a.S, 256, device="cuda", requires_grad=True)
        l = torch.randn(2, T, 768, device="cuda", requires_grad=True)
        mask = torch.ones(2, T, dtype=torch.int64, device="cuda")
        mask[1, T // 2:] = 0
        for backward in (False, True):
            times = {name: [] for name, _, _ in ARMS}
            for _ in range(a.rounds):
                for name, fused, tf32 in ARMS:
                    set_tf32(tf32)
                    times[name].append(time_it(lambda: run(blk, v, l, mask, fused, backward), a.iters))
            for name, _, _ in ARMS:
                key = f"T{T}_{'fwd_bwd' if backward else 'fwd'}_{name}_ms"
                results[key] = round(statistics.median(times[name]), 3)
                results[key + "_spread"] = [round(min(times[name]), 3), round(max(times[name]), 3)]
        for name, fused, tf32 in ARMS:
            set_tf32(tf32)
            blk.zero_grad(set_to_none=True)
            v.grad = l.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            run(blk, v, l, mask, fused, True)
            torch.cuda.synchronize()
            results[f"T{T}_peak_MiB_{name}"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        del v, l
        # the attention core alone: [B, S, 8, 256] inputs as the projections make them (q already scaled)
        g = torch.Generator(device="cuda").manual_seed(T)
        q = torch.randn(2, a.S, H, D, device="cuda", generator=g) * D ** -0.5
        k, vv = torch.randn(2, T, H, D, device="cuda", generator=g), torch.randn(2, a.S, H, D, device="cuda", generator=g)
        vl = torch.randn(2, T, H, D, device="cuda", generator=g)
        bias = vf.text_bias(mask, T)
        go = (torch.randn_like(q), torch.randn_like(k))
        times = {name: [] for name, _, _ in ARMS}
        for _ in range(a.rounds):
            for name, fused, tf32 in ARMS:
                set_tf32(tf32)
                times[name].append(time_it(lambda: core(q, k, vv, vl, bias, fused, go), a.iters))
        for name, _, _ in ARMS:
            ms = statistics.median(times[name])
            results[f"T{T}_core_fwd_bwd_{name}_ms"] = round(ms, 3)
            results[f"T{T}_core_fwd_bwd_{name}_spread"] = [round(min(times[name]), 3), round(max(times[name]), 3)]
            results[f"T{T}_core_fwd_bwd_{name}_TFLOPs"] = round(core_flops(2, a.S, T, True) / ms / 1e9, 1)
        if T == 256:
            for tf32 in (False, True):
                results[f"core_err_vs_fp64_{'tf32' if tf32 else 'fp32'}"] = {
                    n: float(f"{e:.3g}") for n, e in core_errors(q, k, vv, vl, bias, tf32).items()}
        del q, k, vv, vl, go
        torch.cuda.empty_cache()
    set_tf32(old)
    print(json.dumps(results, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vlfuse_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
