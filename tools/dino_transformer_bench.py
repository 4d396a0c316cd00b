#!/usr/bin/env python
"""DINO's whole deformable transformer (``DeformableTransformerVLDINO``, DESIGN.md section 3.16): one training forward +
backward at cfg2, in one process on one GPU.

    python tools/dino_transformer_bench.py [--rounds 5] [--iters 5] [--profile-dir DIR]

Workload: N = 2 at 1333 x 800 (image 1 padded to 75 % x 66 %), 256 text tokens, 900 proposals, with and without 200 DN
queries (2 groups, their attention mask), 6 + 6 layers, d_ffn 2048, early fusion on every encoder layer, dropout on.
Arms, alternated `rounds` times (a round times `iters` steps, each between CUDA events, and takes their median):
    eager_fp32   this class, TF32 off
    eager_tf32   this class, TF32 matmuls allowed
    graphed      this class captured with uninext_b200.graphs.GraphedStep, TF32 off
    reference    the reference's class on its own CUDA kernels (oracle/_ref), when its staged files
                 (tests/golden/make_dino_transformer_golden.py) and oracle/_ref/libmsda_refcuda.so are present, TF32 off
Prints one line per arm with the median, the spread (min..max of the round medians) and the peak memory of one step, the
card's name and power limit read in the same run, and one JSON line per case.  With --profile-dir, a separate
torch.profiler run gives the CUDA kernel time of the input preparation (flatten_levels) against the reference's chain.
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.detpost_bench import card  # noqa: E402
from uninext_b200.modules.deformable_transformer import MLP  # noqa: E402
from uninext_b200.modules.dino_transformer import DeformableTransformerVLDINO, flatten_levels  # noqa: E402
from uninext_b200.modules.two_stage import Still_Classifier  # noqa: E402
from uninext_b200.workloads import CONFIGS  # noqa: E402

DEV = "cuda"
K, DN, T, LAYERS, D_FFN = 900, 200, 256, 6, 2048
KW = dict(d_model=256, nhead=8, num_encoder_layers=LAYERS, num_decoder_layers=LAYERS, dim_feedforward=D_FFN,
          dropout=0.1, activation="relu", return_intermediate_dec=True, num_feature_levels=4, dec_n_points=4,
          enc_n_points=4, two_stage=True, two_stage_num_proposals=K, look_forward_twice=True, mixed_selection=False,
          use_checkpoint=False)


def attach_heads(model):
    model.decoder.class_embed = torch.nn.ModuleList(Still_Classifier(256) for _ in range(LAYERS + 1))
    model.decoder.bbox_embed = torch.nn.ModuleList(MLP(256, 256, 4, 3) for _ in range(LAYERS + 1))
    return model


def inputs(dn):
    g = torch.Generator().manual_seed(0)
    shapes = CONFIGS["cfg2"].shapes
    x = {"srcs": [torch.randn(2, 256, h, w, generator=g).to(DEV) for h, w in shapes],
         "pos": [torch.randn(2, 256, h, w, generator=g).to(DEV) for h, w in shapes], "masks": []}
    for h, w in shapes:
        m = torch.zeros(2, h, w, dtype=torch.bool)
        m[1, math.ceil(0.66 * h):, :] = True
        m[1, :, math.ceil(0.75 * w):] = True
        x["masks"].append(m.to(DEV))
    x["lang"] = {"hidden": torch.randn(2, T, 768, generator=g).to(DEV),
                 "masks": torch.tensor([[1] * T, [1] * 40 + [0] * (T - 40)], dtype=torch.int64).to(DEV)}
    x["query_embed"], x["attn_masks"] = (None, None), None
    if dn:
        x["query_embed"] = (torch.randn(2, DN, 256, generator=g).to(DEV), torch.randn(2, DN, 4, generator=g).to(DEV))
        q = DN + K
        m = torch.zeros(q, q, dtype=torch.bool)
        m[DN:, :DN] = True
        half = DN // 2
        m[:half, half:DN] = True
        m[half:DN, :half] = True
        x["attn_masks"] = m.to(DEV)
    return x


def step_fn(model, x):
    def fn():
        lang = {"hidden": x["lang"]["hidden"], "masks": x["lang"]["masks"]}
        out = model(x["srcs"], x["masks"], x["pos"], x["query_embed"], mask_on=True, language_dict_features=lang,
                    task="detection", attn_masks=x["attn_masks"])
        hs, memory, init_ref, inter_ref, enc_class, enc_coord = out[:6]
        loss = hs.square().mean() + inter_ref.mean() + enc_class.mean() + enc_coord.nan_to_num(0, 0, 0).mean()
        loss.backward()
        return loss.detach()
    return fn


def reference_model():
    """The reference's DeformableTransformerVLDINO on its own CUDA kernels, or the reason it is unavailable."""
    from oracle import refcuda
    staged = os.path.join(ROOT, "oracle", "_ref", "dino_transformer", "dino_ref")
    if not os.path.isdir(staged):
        return None, "staged reference files absent (tests/golden/make_dino_transformer_golden.py stages them)"
    if not refcuda.available():
        return None, "oracle/_ref/libmsda_refcuda.so not built"
    import importlib.util
    import types
    spec = importlib.util.spec_from_file_location("make_dino_transformer_golden", os.path.join(
        ROOT, "tests", "golden", "make_dino_transformer_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    import bench
    dino = gen.import_staged(lambda func: bench.reference_kernels_module(refcuda))
    ns = types.SimpleNamespace
    fuse = ns(STABLE_SOFTMAX_2D=False, CLAMP_MIN_FOR_UNDERFLOW=True, CLAMP_MAX_FOR_OVERFLOW=True)
    cfg = ns(MODEL=ns(USE_EARLY_FUSION=True, USE_ADDITIONAL_BERT=False, VL_FUSION_USE_CHECKPOINT=False, DECOUPLE_TGT=True,
                      STILL_TGT_FOR_BOTH=True, DYHEAD=ns(FUSE_CONFIG=fuse),
                      LANGUAGE_BACKBONE=ns(MODEL_TYPE="bert-base-uncased", MAX_QUERY_LEN=T, N_LAYERS=1, LANG_DIM=768),
                      DDETRS=ns(HIDDEN_DIM=256, VL_HIDDEN_DIM=2048, ENC_LAYERS=LAYERS, NUM_VL_LAYERS=LAYERS)))
    return attach_heads(dino.DeformableTransformerVLDINO(**KW, cfg=cfg)).to(DEV), None


def time_arm(fn, tf32, iters):
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms)


def peak_mib(fn, tf32):
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def profile_prep(out_dir):
    """CUDA kernel time of flatten_levels' forward + backward against the reference's chain, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    from tests.test_gpu_dino_transformer import pyramid, reference_chain
    srcs, masks, pos, le = pyramid("cfg2", 256)
    res = {}
    for name, fn in (("flatten_levels", flatten_levels), ("reference_chain", reference_chain)):
        leaves = ([s.clone().requires_grad_(True) for s in srcs], [p.clone().requires_grad_(True) for p in pos],
                  le.clone().requires_grad_(True))

        def call():
            out = fn(leaves[0], masks, leaves[1], leaves[2])
            torch.autograd.backward((out[0], out[2]), (torch.ones_like(out[0]), torch.ones_like(out[2])))
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                call()
            torch.cuda.synchronize()
        kernels = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]
        res[name] = sum(e.device_time_total for e in kernels) / 10 / 1000.0
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"prep_{name}.pt.trace.json"))
    print(f"input preparation fwd+bwd CUDA kernel time per call (torch.profiler): flatten_levels "
          f"{res['flatten_levels']:.3f} ms, reference chain {res['reference_chain']:.3f} ms")
    print(json.dumps({"case": "input preparation cfg2 N=2 fwd+bwd", "card": card(), "kernel_ms": res}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--profile-dir", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dino_transformer_bench.py needs a CUDA device")
    from uninext_b200.graphs import GraphedStep
    print(card())
    torch.manual_seed(0)
    ours = attach_heads(DeformableTransformerVLDINO(**KW)).to(DEV).train()
    ref, why = reference_model()
    for dn in (False, True):
        x = inputs(dn)
        arms = {"eager_fp32": (step_fn(ours, x), False), "eager_tf32": (step_fn(ours, x), True)}
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        arms["graphed"] = (GraphedStep(step_fn(ours, x)).replay, False)
        if ref is not None:
            ref.load_state_dict(ours.state_dict())
            arms["reference"] = (step_fn(ref.train(), x), False)
        for fn, tf32 in arms.values():                                 # warm-up
            for _ in range(2):
                time_arm(fn, tf32, 1)
        peak = {k: peak_mib(fn, tf32) for k, (fn, tf32) in arms.items() if k != "graphed"}
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, (fn, tf32) in arms.items():
                times[k].append(time_arm(fn, tf32, a.iters))
        case = f"cfg2 N=2 S={CONFIGS['cfg2'].S} T={T} k={K} dn={DN if dn else 0} {LAYERS}+{LAYERS} layers fwd+bwd"
        for k, v in times.items():
            print(f"{case} {k}: {statistics.median(v):.2f} ms [{min(v):.2f}..{max(v):.2f}], peak "
                  f"{peak.get(k, float('nan')):.0f} MiB, {card()}")
        if ref is None:
            print(f"{case} reference: unavailable ({why})")
        print(json.dumps({"case": case, "card": card(), "median_ms": {k: statistics.median(v) for k, v in times.items()},
                          "rounds_ms": times, "peak_mib": peak, "reference": None if ref is not None else why}))
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    if a.profile_dir:
        profile_prep(a.profile_dir)


if __name__ == "__main__":
    main()
