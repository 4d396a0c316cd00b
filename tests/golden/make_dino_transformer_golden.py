#!/usr/bin/env python
"""Regenerate tests/golden/reference/dino_transformer_*.npz: the reference's own DeformableTransformerVLDINO
(deformable_transformer_dino.py:49-327) on the CPU, in eval mode, with gradients, on the cases of tests/dino_case.py.
Needs a reference checkout; the tests themselves do not.

    python tests/golden/make_dino_transformer_golden.py

Copied verbatim into the git-ignored oracle/_ref/dino_transformer/: deformable_transformer_dino.py, vlfusion.py,
fuse_helper.py, modeling_bert.py and the ops package.  Written here, not copied: ``util/misc.py`` (``inverse_sigmoid``),
a ``timm`` stub (``DropPath``, unused at drop_path = 0), the two helpers that transformers 5 moved out of
``transformers.modeling_utils`` (pruning is never called), the cfg namespace, and the op's two entry points computed
with the reference's own ``ms_deform_attn_core_pytorch``.  The class heads are the reference's ``Still_Classifier``
(staged by make_two_stage_golden.py) and its ``MLP``.

Per case the seed is the first from ``dino_case.BASE_SEED`` up for which each image's k + 1 largest encoder logits are
more than 1e-3 of their scale apart and the constant logit of dropped rows is not among them.  Stored
(tests/refgolden.py conventions): the seed; a sample of every input; the outputs whole in fp32, except the encoder memory
(a sample); every input gradient and parameter gradient as a sample with its scale; the state_dict keys.
"""
import importlib
import importlib.util
import os
import shutil
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
os.environ["MSDA_RECORD_REFERENCE"] = "1"
from oracle.refpy import REFERENCE  # noqa: E402
from tests import dino_case as dc  # noqa: E402
from tests import refgolden  # noqa: E402

SRC = os.path.join(REFERENCE, "projects/UNINEXT/uninext/models/deformable_detr")
DEST = os.path.join(ROOT, "oracle", "_ref", "dino_transformer")
PKG = os.path.join(DEST, "dino_ref")
COPIES = ["deformable_transformer_dino.py", "vlfusion.py", "fuse_helper.py", "modeling_bert.py",
          "ops/functions/__init__.py", "ops/functions/ms_deform_attn_func.py", "ops/modules/__init__.py",
          "ops/modules/ms_deform_attn.py"]
STUBS = {
    "__init__.py": "",
    "util/__init__.py": "",
    "util/misc.py": ("import torch\n\n\ndef inverse_sigmoid(x, eps=1e-5):\n    x = x.clamp(min=0, max=1)\n"
                     "    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))\n"),
    "models/__init__.py": "",
    "models/deformable_detr/__init__.py": "",
    "models/deformable_detr/ops/__init__.py": "",
}


class _CpuKernels:
    """The reference pybind module's two entry points, computed with the reference's own CPU function."""
    core = None

    @classmethod
    def ms_deform_attn_forward(cls, value, shapes, lsi, loc, attn, im2col_step):
        with torch.no_grad():
            return cls.core(value, shapes, loc, attn)

    @classmethod
    def ms_deform_attn_backward(cls, value, shapes, lsi, loc, attn, grad_output, im2col_step):
        with torch.enable_grad():
            v, lo, at = (t.detach().clone().requires_grad_(True) for t in (value, loc, attn))
            return list(torch.autograd.grad(cls.core(v, shapes, lo, at), (v, lo, at), grad_output))


def _stage():
    for rel, text in STUBS.items():
        path = os.path.join(PKG, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as fh:
            fh.write(text)
    for rel in COPIES:
        dst = os.path.join(PKG, "models/deformable_detr", rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, rel), dst)


def import_staged(kernels):
    """The staged deformable_transformer_dino, with ``kernels`` standing in for the
    op's compiled extension."""
    import transformers.modeling_utils as mu          # before the timm stub: transformers probes for timm on import
    import transformers.models.bert.modeling_bert  # noqa: F401
    import transformers.pytorch_utils as pu
    timm = types.ModuleType("timm")
    timm.models = types.ModuleType("timm.models")
    timm.models.layers = types.ModuleType("timm.models.layers")
    timm.models.layers.DropPath = None
    sys.modules.update({"timm": timm, "timm.models": timm.models, "timm.models.layers": timm.models.layers})
    for name in ("apply_chunking_to_forward", "prune_linear_layer", "find_pruneable_heads_and_indices"):
        if not hasattr(mu, name):
            setattr(mu, name, getattr(pu, name, None))
    import uninext_b200
    uninext_b200.install_dropin()
    sys.path.insert(0, DEST)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        func = importlib.import_module("dino_ref.models.deformable_detr.ops.functions.ms_deform_attn_func")
        dino = importlib.import_module("dino_ref.models.deformable_detr.deformable_transformer_dino")
    func.MSDA = kernels(func)
    return dino


def _cfg(name):
    fusion, decouple, still, _, _ = dc.CASES[name]
    ns = types.SimpleNamespace
    fuse = ns(STABLE_SOFTMAX_2D=False, CLAMP_MIN_FOR_UNDERFLOW=True, CLAMP_MAX_FOR_OVERFLOW=True,
              CLAMP_BERTATTN_MIN_FOR_UNDERFLOW=True, CLAMP_BERTATTN_MAX_FOR_OVERFLOW=True)
    return ns(MODEL=ns(USE_EARLY_FUSION=fusion, USE_ADDITIONAL_BERT=False, VL_FUSION_USE_CHECKPOINT=False,
                       DECOUPLE_TGT=decouple, STILL_TGT_FOR_BOTH=still, DYHEAD=ns(FUSE_CONFIG=fuse),
                       LANGUAGE_BACKBONE=ns(MODEL_TYPE="bert-base-uncased", MAX_QUERY_LEN=256, N_LAYERS=1,
                                            LANG_DIM=dc.LANG),
                       DDETRS=ns(HIDDEN_DIM=dc.C, VL_HIDDEN_DIM=dc.VL_HIDDEN, ENC_LAYERS=dc.ENC_LAYERS,
                                 NUM_VL_LAYERS=dc.VL_LAYERS)))


def build_reference(name, dino, detr):
    kw, _ = dc.config(name)
    model = dino.DeformableTransformerVLDINO(**kw, cfg=_cfg(name))
    return dc.attach_heads(model, detr.Still_Classifier, dino.MLP).eval()


def margins_hold(out):
    """Each image's k + 1 largest logits more than 1e-3 of their scale apart, none of them the dropped rows' logit."""
    lg = out["enc_outputs_class"].detach()[..., 0]
    dropped = lg[1, dc.masks()[0][1].flatten().nonzero()[0, 0]]     # image 1's first padded position
    for b in range(dc.N):
        top = lg[b].topk(dc.K + 1).values
        scale = top.abs().max()
        if (top[:-1] - top[1:]).min() <= 1e-3 * scale or (top - dropped).abs().min() <= 1e-3 * scale:
            return False
    return True


def record(name, dino, detr):
    seed = dc.BASE_SEED[name]
    while True:
        model = build_reference(name, dino, detr)
        params = dc.parameters(model, seed)
        x = dc.inputs(name, seed)
        out, leaves = dc.run(model, name, x, "cpu")
        if margins_hold(out):
            break
        seed += 1
    dc.backward(out, dc.cotangents(out, seed))
    group = f"dino_transformer_{name}"
    refgolden.put_raw(group, "seed", np.array([seed]))
    for k in ("srcs", "pos_embeds"):
        for lvl, t in enumerate(x[k]):
            refgolden.put(group, f"in.{k}.{lvl}", t)
            refgolden.put(group, f"grad.{k}.{lvl}", leaves[k][lvl].grad)
    for k in ("hidden", "dn_label", "dn_bbox"):
        if k in x:
            refgolden.put(group, f"in.{k}", x[k])
            refgolden.put(group, f"grad.{k}", leaves[k].grad)
    for k, v in out.items():
        if k == "memory":
            refgolden.put(group, "out.memory", v)
        else:
            refgolden.put_raw(group, f"out.{k}", v.detach().float().numpy())
    with_grad = sorted(k for k, p in params.items() if p.grad is not None)
    for k in with_grad:
        refgolden.put(group, "grad." + k, params[k].grad)
    refgolden.put_raw(group, "param_names", np.array(with_grad))
    refgolden.put_raw(group, "state_dict_keys", np.array(list(model.state_dict().keys())))
    refgolden.flush(group)
    size = os.path.getsize(os.path.join(refgolden.GOLDEN, f"{group}.npz"))
    print(f"written {group}: seed {seed}, {len(with_grad)} parameter gradients, {size / 1e6:.2f} MB")


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    _stage()

    def cpu_kernels(func):
        _CpuKernels.core = staticmethod(func.ms_deform_attn_core_pytorch)
        return _CpuKernels
    dino = import_staged(cpu_kernels)
    spec = importlib.util.spec_from_file_location("make_two_stage_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_two_stage_golden.py"))
    ts = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ts)
    detr = ts._deformable_detr()
    for name in dc.CASES:
        record(name, dino, detr)


if __name__ == "__main__":
    main()
