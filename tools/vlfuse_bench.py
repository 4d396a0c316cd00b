#!/usr/bin/env python
"""The early-fusion block (BiAttentionBlock, DESIGN.md section 3.11): fused kernels against the torch composition of the
same maths (the reference's order of operations), in one process.

    python tools/vlfuse_bench.py [--rounds 3] [--iters 5] [--out DIR]

UNINEXT dims (v 256, l 768, embed 2048, 8 heads), S = 22323, training mode (dropout 0.1), at three shapes: cfg2 with
B = 2 and T = 256 or T = 32, and cfg5 (B = 1, a 20-token prompt, T = 20).  Six arms: fused fp32, fused TF32, torch fp32,
torch TF32, fused bf16 and torch bf16 (TF32 = torch.backends.cuda.matmul.allow_tf32, which the fused path and the torch
einsums both follow; bf16 = the block built with ``op_dtype=torch.bfloat16`` and run under
``torch.autocast("cuda", torch.bfloat16)``, the core on bf16 tensors).  For each shape and arm: the block's forward, and
forward + backward, timed with CUDA events over `iters` calls, the arms alternating `rounds` times (medians and the
spread of the round medians); peak memory of one block forward + backward; the attention core alone (``vl_attention``,
or ``vl_attention_torch`` for the torch arms, on [B, S, 8, 256] inputs), forward and forward + backward, with its
achieved TFLOP/s from the FLOP count 2 S T d B H per S x T x d product (4 in the forward, 10 in the backward) and that
rate's share of the data-sheet dense rate of the arm's product type (H100 SXM: 67 TFLOP/s fp32, 495 TF32, 989 bf16);
and the largest relative difference of each of the core's six outputs (O_v, O_l, dQ, dK, dVv, dVl) against an fp64
restatement on the same bf16-valued inputs, without dropout.  Prints the card's name and power limit, read in the same
run; writes a JSON copy under --out when given."""
import argparse
import contextlib
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.det_bench import card  # noqa: E402
from uninext_b200.modules import vl_fusion as vf  # noqa: E402


# name, fused, allow_tf32, bf16
ARMS = (("fused", True, False, False), ("fused_tf32", True, True, False), ("torch", False, False, False),
        ("torch_tf32", False, True, False), ("fused_bf16", True, False, True), ("torch_bf16", False, False, True))
SHAPES = (("cfg2_T256", 2, 256), ("cfg2_T32", 2, 32), ("cfg5_T20", 1, 20))
H, D = 8, 256
DATASHEET_TFLOPS = {"fp32": 67.0, "tf32": 495.0, "bf16": 989.0}      # H100 SXM, dense, 700 W


def core_flops(B, S, T, backward):
    """FLOPs of the S x T x d products of the attention core: 4 in the forward, 10 more in the backward."""
    return 2 * S * T * D * B * H * (14 if backward else 4)


def product_type(tf32, bf16):
    return "bf16" if bf16 else ("tf32" if tf32 else "fp32")


def set_tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on


def core(q, k, vv, vl, bias, fused, go):
    """Forward (go None) or forward + backward of the attention core alone."""
    leaves = [t.detach().requires_grad_(go is not None) for t in (q, k, vv, vl)]
    fn = vf.vl_attention if fused else vf.vl_attention_torch
    o_v, o_l = fn(*leaves, bias, True, True, 0.1, True)
    if go is not None:
        torch.autograd.backward((o_v, o_l), go)
    return o_v, o_l


def restate_fp64(q, k, vv, vl, bias, go):
    leaves = [t.detach().double().requires_grad_(True) for t in (q, k, vv, vl)]
    x = torch.einsum("bshd,bthd->bhst", *leaves[:2]).clamp(-50000, 50000)
    p_l = (x.transpose(2, 3) - x.transpose(2, 3).max(dim=-1, keepdim=True)[0]).softmax(dim=-1)
    b = bias[:, None, None, :].double()
    masked = float(torch.tensor(-9e15, dtype=torch.float32))
    p_v = (x + torch.where(b < -1e15, masked - x, b).detach()).softmax(dim=-1)
    want = [torch.einsum("bhst,bthd->bshd", p_v, leaves[3]), torch.einsum("bhts,bshd->bthd", p_l, leaves[2])]
    want += list(torch.autograd.grad(want, leaves, [g.double() for g in go]))
    return [w.detach() for w in want]


def core_errors(q, k, vv, vl, bias, fused, tf32, bf16, go, want):
    """Largest |arm - fp64| / max |fp64| of the six core outputs, without dropout."""
    set_tf32(tf32)
    dt = torch.bfloat16 if bf16 else torch.float32
    leaves = [t.detach().to(dt).requires_grad_(True) for t in (q, k, vv, vl)]
    fn = vf.vl_attention if fused else vf.vl_attention_torch
    got = list(fn(*leaves, bias, True, True, 0.0, False))
    got += list(torch.autograd.grad(got, leaves, [g.to(dt) for g in go]))
    set_tf32(False)
    return {n: float(f"{float((g.detach().double() - w).abs().max() / w.abs().max()):.3g}") for n, g, w in
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
        (out_v.float().sum() + out_l.float().sum()).backward()


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


def arm_context(tf32, bf16):
    set_tf32(tf32)
    return torch.autocast("cuda", torch.bfloat16) if bf16 else contextlib.nullcontext()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--S", type=int, default=22323)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vlfuse_bench needs a CUDA device"
    torch.manual_seed(0)
    results = {"device": card(), "S": a.S, "datasheet_TFLOPs": DATASHEET_TFLOPS}
    blk = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6).cuda().train()
    blk_bf16 = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6,
                                   op_dtype=torch.bfloat16).cuda().train()
    blk_bf16.load_state_dict(blk.state_dict())
    old = torch.backends.cuda.matmul.allow_tf32
    for shape, B, T in SHAPES:
        results[f"{shape}_B"], results[f"{shape}_T"] = B, T
        v = torch.randn(B, a.S, 256, device="cuda", requires_grad=True)
        l = torch.randn(B, T, 768, device="cuda", requires_grad=True)
        mask = torch.ones(B, T, dtype=torch.int64, device="cuda")
        mask[-1, T // 2:] = 0
        for backward in (False, True):
            times = {arm[0]: [] for arm in ARMS}
            for _ in range(a.rounds):
                for name, fused, tf32, bf16 in ARMS:
                    with arm_context(tf32, bf16):
                        times[name].append(time_it(lambda: run(blk_bf16 if bf16 else blk, v, l, mask, fused, backward),
                                                   a.iters))
            for name, *_ in ARMS:
                key = f"{shape}_block_{'fwd_bwd' if backward else 'fwd'}_{name}_ms"
                results[key] = round(statistics.median(times[name]), 3)
                results[key + "_spread"] = [round(min(times[name]), 3), round(max(times[name]), 3)]
        for name, fused, tf32, bf16 in ARMS:
            m = blk_bf16 if bf16 else blk
            m.zero_grad(set_to_none=True)
            v.grad = l.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            with arm_context(tf32, bf16):
                run(m, v, l, mask, fused, True)
            torch.cuda.synchronize()
            results[f"{shape}_block_peak_MiB_{name}"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        blk.zero_grad(set_to_none=True)
        blk_bf16.zero_grad(set_to_none=True)
        del v, l
        # the attention core alone: [B, S, 8, 256] inputs as the projections make them (q already scaled), bf16-valued so
        # that every arm sees the same inputs
        g = torch.Generator(device="cuda").manual_seed(T)
        bfv = lambda t: t.to(torch.bfloat16).float()
        q = bfv(torch.randn(B, a.S, H, D, device="cuda", generator=g) * D ** -0.5)
        k, vv = bfv(torch.randn(B, T, H, D, device="cuda", generator=g)), bfv(torch.randn(B, a.S, H, D, device="cuda", generator=g))
        vl = bfv(torch.randn(B, T, H, D, device="cuda", generator=g))
        bias = vf.text_bias(mask, T)
        go = (bfv(torch.randn_like(q)), bfv(torch.randn_like(k)))
        inputs = {False: (q, k, vv, vl, go), True: tuple(t.to(torch.bfloat16) for t in (q, k, vv, vl)) +
                  (tuple(t.to(torch.bfloat16) for t in go),)}
        for backward in (False, True):
            times = {arm[0]: [] for arm in ARMS}
            for _ in range(a.rounds):
                for name, fused, tf32, bf16 in ARMS:
                    set_tf32(tf32)
                    *qkv, gob = inputs[bf16]
                    times[name].append(time_it(lambda: core(*qkv, bias, fused, gob if backward else None), a.iters))
            for name, fused, tf32, bf16 in ARMS:
                ms = statistics.median(times[name])
                key = f"{shape}_core_{'fwd_bwd' if backward else 'fwd'}_{name}"
                results[key + "_ms"] = round(ms, 3)
                results[key + "_spread"] = [round(min(times[name]), 3), round(max(times[name]), 3)]
                tflops = core_flops(B, a.S, T, backward) / ms / 1e9
                results[key + "_TFLOPs"] = round(tflops, 1)
                results[key + "_of_datasheet"] = round(tflops / DATASHEET_TFLOPS[product_type(tf32, bf16)], 4)
        want = restate_fp64(q, k, vv, vl, bias, go)
        for name, fused, tf32, bf16 in ARMS:
            results[f"{shape}_core_err_vs_fp64_{name}"] = core_errors(q, k, vv, vl, bias, fused, tf32, bf16, go, want)
        del q, k, vv, vl, go, inputs, want
        torch.cuda.empty_cache()
    set_tf32(old)
    print(json.dumps(results, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vlfuse_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
