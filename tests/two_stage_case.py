"""The cases of the two-stage query selection tests (tests/golden/make_two_stage_golden.py records the reference on them):
inputs and parameters drawn from fixed seeds, so that the stored reference results (tests/golden/reference/two_stage_*.npz)
need not hold them, only a sample of each to show they were drawn alike.

Pyramid [(20, 28), (10, 14), (5, 7), (3, 4)], N = 2 (image 1 padded to 70 % x 60 % of each level), k = 300.  Cases:
    still      Still_Classifier
    vl         VL_Align without the clamp
    vl_clamp   VL_Align with the clamp: scale and bias0 such that the lowest quarter or so of the logits are clamped to
               -5e4, below the selected ones, so that the clamp makes no ties among the selected rows
"""
import math

import torch

SHAPES = [(20, 28), (10, 14), (5, 7), (3, 4)]
S = sum(h * w for h, w in SHAPES)
N, C, LANG, K = 2, 256, 768, 300
CASES = {"still": ("still", False, 0.0), "vl": ("vl", False, 0.0), "vl_clamp": ("vl", True, -8.5)}


def padding_mask():
    """[N, S] bool: image 0 unpadded; image 1 valid in the top-left ceil(0.6 H) x ceil(0.7 W) of each level."""
    rows = []
    for b in range(N):
        lv = []
        for h, w in SHAPES:
            m = torch.zeros(h, w, dtype=torch.bool)
            if b == 1:
                m[math.ceil(0.6 * h):, :] = True
                m[:, math.ceil(0.7 * w):] = True
            lv.append(m.flatten())
        rows.append(torch.cat(lv))
    return torch.stack(rows)


def _gen(name, salt):
    return torch.Generator().manual_seed(1000 * list(CASES).index(name) + salt)


def state(name):
    """Parameters by the reference's names: enc_output.*, enc_output_norm.*, class_embed.*, bbox_embed.layers.*."""
    head, clamp, log_scale = CASES[name]
    g = _gen(name, 1)
    r = lambda *shape, s=1.0: torch.randn(*shape, generator=g) * s
    sd = {"enc_output.weight": r(C, C, s=C ** -0.5), "enc_output.bias": r(C, s=0.1),
          "enc_output_norm.weight": 1 + r(C, s=0.1), "enc_output_norm.bias": r(C, s=0.1)}
    if head == "still":
        sd.update({"class_embed.body.weight": r(1, C, s=C ** -0.5), "class_embed.body.bias": r(1, s=0.5)})
    else:
        sd.update({"class_embed.dot_product_projection_text.weight": r(C, LANG, s=LANG ** -0.5),
                   "class_embed.dot_product_projection_text.bias": r(C, s=0.1),
                   "class_embed.log_scale": torch.tensor([log_scale]), "class_embed.bias_lang": r(LANG, s=0.05),
                   "class_embed.bias0": torch.tensor([-4e4 if clamp else -math.log(0.99 / 0.01)])})
    for i, (fi, fo) in enumerate(((C, C), (C, C), (C, 4))):
        sd[f"bbox_embed.layers.{i}.weight"] = r(fo, fi, s=fi ** -0.5)
        sd[f"bbox_embed.layers.{i}.bias"] = r(fo, s=0.1)
    return sd


def inputs(name):
    """memory [N, S, C], memory_padding_mask [N, S], lang_feat_pool [N, 768] and the cotangents of the four outputs'
    differentiable three: g_class [N, S, 1], g_coord [N, S, 4], g_ref [N, K, 4]."""
    g = _gen(name, 2)
    r = lambda *shape: torch.randn(*shape, generator=g)
    return {"memory": r(N, S, C), "mask": padding_mask(), "lang_feat_pool": r(N, LANG), "g_class": r(N, S, 1),
            "g_coord": r(N, S, 4), "g_ref": r(N, K, 4)}


def load_modules(name, modules):
    """Load state(name) into the dict of modules {'enc_output': .., 'enc_output_norm': .., 'class_embed': ..,
    'bbox_embed': ..}; -> the modules' named parameters by full name."""
    sd = state(name)
    for prefix, m in modules.items():
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")})
    return {f"{p}.{k}": v for p, m in modules.items() for k, v in m.named_parameters()}


def backward(outputs, cot):
    """Backward of (enc_outputs_class, enc_outputs_coord_unact, reference_points) against the case's cotangents."""
    cls, coord, ref = outputs[:3]
    torch.autograd.backward((cls, coord, ref), (cot["g_class"].to(cls.device), cot["g_coord"].to(cls.device),
                                                cot["g_ref"].to(cls.device)))
