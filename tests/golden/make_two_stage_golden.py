#!/usr/bin/env python
"""Regenerate tests/golden/reference/two_stage_*.npz: the reference's two-stage query selection on the CPU, on the cases of
tests/two_stage_case.py.  Needs a reference checkout; the tests themselves do not.

    python tests/golden/make_two_stage_golden.py

What runs is the reference's own code: ``DeformableTransformerVLDINO.gen_encoder_output_proposals``
(deformable_transformer_dino.py:132-162, called unbound on a namespace holding ``enc_output`` / ``enc_output_norm``),
its ``MLP``, and ``Still_Classifier`` / ``VL_Align`` of deformable_detr.py, followed by the statements of :219-224.
deformable_transformer_dino.py is staged by tests/stage_reference.py.  deformable_detr.py is copied verbatim into the
git-ignored oracle/_ref/two_stage/; written here, not copied: stubs of the modules it imports at module level that the two
heads never use (util.box_ops, util.misc, backbone, matcher, segmentation, fvcore.nn).

Stored per case (tests/refgolden.py conventions: large tensors as a sample of their elements with the max-abs scale):
every input and parameter as such a sample (the tests redraw them from the case's seeds), the gradient of memory and of
every parameter, and, whole, the outputs: class logits, coord_unact, reference points and the top-k indices.
"""
import os
import shutil
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
os.environ["MSDA_RECORD_REFERENCE"] = "1"
from oracle.refpy import REFERENCE  # noqa: E402
from tests import refgolden, stage_reference  # noqa: E402
from tests import two_stage_case as tc  # noqa: E402

SRC = os.path.join(REFERENCE, "projects/UNINEXT/uninext/models/deformable_detr/deformable_detr.py")
DEST = os.path.join(ROOT, "oracle", "_ref", "two_stage")

STUBS = {
    "__init__.py": "",
    "util/__init__.py": "",
    "util/box_ops.py": "",
    "util/misc.py": ("NestedTensor = nested_tensor_from_tensor_list = accuracy = get_world_size = interpolate = None\n"
                     "is_dist_avail_and_initialized = inverse_sigmoid = None\n"),
    "models/__init__.py": "",
    "models/deformable_detr/__init__.py": "",
    "models/deformable_detr/backbone.py": "build_backbone = None\n",
    "models/deformable_detr/matcher.py": "build_matcher = None\n",
    "models/deformable_detr/segmentation.py": "dice_loss = sigmoid_focal_loss = token_sigmoid_binary_focal_loss = None\n",
}


def _deformable_detr():
    pkg = os.path.join(DEST, "two_stage_ref")
    for rel, text in STUBS.items():
        path = os.path.join(pkg, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as fh:
            fh.write(text)
    shutil.copyfile(SRC, os.path.join(pkg, "models/deformable_detr/deformable_detr.py"))
    fvcore = types.ModuleType("fvcore")
    fvcore.nn = types.ModuleType("fvcore.nn")
    fvcore.nn.giou_loss = fvcore.nn.smooth_l1_loss = None
    sys.modules.update({"fvcore": fvcore, "fvcore.nn": fvcore.nn})
    sys.path.insert(0, DEST)
    import importlib
    return importlib.import_module("two_stage_ref.models.deformable_detr.deformable_detr")


def _cfg(clamp, log_scale):
    ns = types.SimpleNamespace
    return ns(MODEL=ns(DYHEAD=ns(PRIOR_PROB=0.01, LOG_SCALE=log_scale, FUSE_CONFIG=ns(CLAMP_DOT_PRODUCT=clamp)),
                       LANGUAGE_BACKBONE=ns(LANG_DIM=tc.LANG), DDETRS=ns(HIDDEN_DIM=tc.C)))


def record(name, dino, detr):
    head, clamp, log_scale = tc.CASES[name]
    modules = {"enc_output": torch.nn.Linear(tc.C, tc.C), "enc_output_norm": torch.nn.LayerNorm(tc.C),
               "class_embed": detr.Still_Classifier(tc.C) if head == "still" else detr.VL_Align(_cfg(clamp, log_scale)),
               "bbox_embed": dino.MLP(tc.C, tc.C, 4, 3)}
    params = tc.load_modules(name, modules)
    x = tc.inputs(name)
    memory = x["memory"].clone().requires_grad_(True)
    owner = types.SimpleNamespace(enc_output=modules["enc_output"], enc_output_norm=modules["enc_output_norm"])
    # deformable_transformer_dino.py:216-224
    output_memory, output_proposals = dino.DeformableTransformerVLDINO.gen_encoder_output_proposals(
        owner, memory, x["mask"], tc.SHAPES)
    enc_outputs_class = modules["class_embed"](output_memory, x["lang_feat_pool"].unsqueeze(1))
    enc_outputs_coord_unact = modules["bbox_embed"](output_memory) + output_proposals
    topk_proposals = torch.topk(enc_outputs_class[..., 0], tc.K, dim=1)[1]
    topk_coords_unact = torch.gather(enc_outputs_coord_unact, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4))
    reference_points = topk_coords_unact.sigmoid()
    tc.backward((enc_outputs_class, enc_outputs_coord_unact, reference_points), x)

    group = f"two_stage_{name}"
    for k, v in x.items():
        refgolden.put(group, "in." + k, v)
    for k, v in tc.state(name).items():
        refgolden.put(group, "state." + k, v)
    refgolden.put_raw(group, "out.reference_points", reference_points.detach().numpy())
    refgolden.put_raw(group, "out.enc_outputs_class", enc_outputs_class.detach().numpy())
    refgolden.put_raw(group, "out.enc_outputs_coord_unact", enc_outputs_coord_unact.detach().numpy())
    refgolden.put_raw(group, "out.topk_proposals", topk_proposals.numpy())
    refgolden.put(group, "grad.memory", memory.grad)
    for k, p in params.items():
        refgolden.put(group, "grad." + k, p.grad)
    refgolden.put_raw(group, "param_names", np.array(sorted(params)))
    refgolden.flush(group)
    lg = enc_outputs_class.detach()[..., 0]
    kth = lg.gather(1, topk_proposals[:, -1:])
    print(f"written {group}: logits [{lg.min().item():.4g}, {lg.max().item():.4g}], k-th {kth.flatten().tolist()}, "
          f"clamped {(lg.abs() >= 5e4).sum().item()} of {lg.numel()}")


def main():
    assert stage_reference.stage(), "no reference checkout to stage from"
    dino = stage_reference.import_reference()[3]
    detr = _deformable_detr()
    torch.set_num_threads(os.cpu_count() or 1)
    for name in tc.CASES:
        record(name, dino, detr)


if __name__ == "__main__":
    main()
