#!/usr/bin/env python
"""Two-stage query selection (``two_stage_select``, msda_twostage.cuh, DESIGN.md section 3.15) against the reference's
chain (deformable_transformer_dino.py:153-161,216-224: masked_fill x2, enc_output, enc_output_norm, the class head,
bbox_embed + proposals, torch.topk, gather, sigmoid) on the same inputs and modules, in one process on one GPU.

    python tools/two_stage_bench.py [--rounds 5] [--iters 20]

Cases: cfg2 (N = 2, S = 22323, image 1 padded to 75 % x 66 %), k = 900, Still_Classifier and VL_Align, bbox_embed the
reference's three-layer MLP; forward alone
and forward + backward.  Both arms share gen_encoder_output_proposals.  The arms alternate `rounds` times; a round
times `iters` calls, each between CUDA events, and takes their median.  Prints the medians, their spread (min..max of
the round medians), the peak memory of one call above what its inputs hold, the card's name and power limit read in the
same run, and one JSON line per case."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.detpost_bench import card  # noqa: E402
from uninext_b200.modules.deformable_transformer import gen_encoder_output_proposals  # noqa: E402
from uninext_b200.modules.two_stage import two_stage_select  # noqa: E402


def reference_chain(memory, mask, shapes, enc_output, enc_output_norm, class_embed, bbox_embed, k, lang_feat_pool):
    """deformable_transformer_dino.py:153-161,216-224 as the reference writes it."""
    output_proposals, valid = gen_encoder_output_proposals(mask, shapes)
    output_memory = memory.masked_fill(mask.unsqueeze(-1), float(0))
    output_memory = output_memory.masked_fill(~valid, float(0))
    output_memory = enc_output_norm(enc_output(output_memory))
    enc_outputs_class = class_embed(output_memory, lang_feat_pool.unsqueeze(1))
    enc_outputs_coord_unact = bbox_embed(output_memory) + output_proposals
    topk_proposals = torch.topk(enc_outputs_class[..., 0], k, dim=1)[1]
    topk_coords_unact = torch.gather(enc_outputs_coord_unact, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4))
    return enc_outputs_class, enc_outputs_coord_unact, topk_coords_unact.sigmoid(), topk_proposals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--k", type=int, default=900)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("two_stage_bench.py needs a CUDA device")
    from tests.test_gpu_two_stage import user_problem
    dev = "cuda"
    print(card())
    for head in ("still", "vl"):
        shapes, mods, x = user_problem("cfg2", head, box_layers=3)
        n, s = x["memory"].shape[:2]
        memory = x["memory"].clone().requires_grad_(True)
        cot = [torch.randn(n, s, 1, device=dev), torch.randn(n, s, 4, device=dev), torch.randn(n, a.k, 4, device=dev)]
        args = (memory, x["mask"], shapes, mods["enc_output"], mods["enc_output_norm"], mods["class_embed"],
                mods["bbox_embed"], a.k, x["lang_feat_pool"])
        arms = {"fused": two_stage_select, "reference": reference_chain}
        outs = {name: fn(*args) for name, fn in arms.items()}
        agree = {"class": (outs["fused"][0] - outs["reference"][0]).abs().max().item(),
                 "topk_equal_fraction": (outs["fused"][3] == outs["reference"][3]).float().mean().item()}

        def call(fn, backward):
            out = fn(*args)
            if backward:
                torch.autograd.backward(out[:3], cot)
                memory.grad = None
                for m in mods.values():
                    m.zero_grad(set_to_none=True)

        for backward in (False, True):
            times = {name: [] for name in arms}
            peak = {}
            for name, fn in arms.items():                     # warm-up, and the peak of one call
                for _ in range(3):
                    call(fn, backward)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                call(fn, backward)
                torch.cuda.synchronize()
                peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            for _ in range(a.rounds):
                for name, fn in arms.items():
                    ms = []
                    for _ in range(a.iters):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        call(fn, backward)
                        e1.record()
                        torch.cuda.synchronize()
                        ms.append(e0.elapsed_time(e1))
                    times[name].append(statistics.median(ms))
            med = {name: statistics.median(v) for name, v in times.items()}
            case = f"cfg2 N={n} S={s} k={a.k} {head} {'fwd+bwd' if backward else 'fwd'}"
            print(f"{case}: fused {med['fused']:.3f} ms [{min(times['fused']):.3f}..{max(times['fused']):.3f}], "
                  f"reference {med['reference']:.3f} ms [{min(times['reference']):.3f}..{max(times['reference']):.3f}], "
                  f"speed-up {med['reference'] / med['fused']:.2f}x; peak MiB fused {peak['fused']:.1f}, "
                  f"reference {peak['reference']:.1f}")
            print(json.dumps({"case": case, "card": card(), "fused_ms": med["fused"], "reference_ms": med["reference"],
                              "fused_rounds_ms": times["fused"], "reference_rounds_ms": times["reference"],
                              "peak_mib": peak, "agreement": agree}))


if __name__ == "__main__":
    main()
