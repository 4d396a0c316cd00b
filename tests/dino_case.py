"""The cases of the whole-transformer tests (tests/golden/make_dino_transformer_golden.py records the reference's
DeformableTransformerVLDINO on them): inputs, parameters and cotangents drawn from a seed, so that the stored results
(tests/golden/reference/dino_transformer_*.npz) hold the seed and a sample of each input, not the inputs.

Pyramid [(11, 17), (6, 9), (3, 5), (2, 3)] (levels 0 and 2 have an odd H * W), C = 256, N = 2 (image 1 padded to
70 % x 60 % of each level), 8 text tokens (image 1: 5 valid), 30 proposals, 2 encoder layers (early fusion on the first
only) and 2 decoder layers with box refinement and look_forward_twice.  Cases:
    production   DECOUPLE_TGT = STILL_TGT_FOR_BOTH = True, task detection, no DN queries
    dn           DN queries (2 groups of 5) with their attention mask, DECOUPLE_TGT = False, task detection
    no_fusion    early fusion off (VLFuse -> Identity), DECOUPLE_TGT = True, STILL_TGT_FOR_BOTH = False, task grounding

The generator picks each case's seed (from BASE_SEED[case] upwards) so that each image's k + 1 largest encoder logits are
more than 1e-3 of the logit scale apart and the constant logit of dropped rows is not among them: the GPU's top-k then
picks the reference's rows.
"""
import math

import torch

SHAPES = [(11, 17), (6, 9), (3, 5), (2, 3)]
S = sum(h * w for h, w in SHAPES)
N, C, LANG, T, K = 2, 256, 768, 8, 30
ENC_LAYERS, DEC_LAYERS, VL_LAYERS, D_FFN, VL_HIDDEN = 2, 2, 1, 64, 1024
DN_GROUPS, DN_PER_GROUP = 2, 5
CASES = {          # use_early_fusion, decouple_tgt, still_tgt_for_both, task, dn
    "production": (True, True, True, "detection", False),
    "dn": (True, False, True, "detection", True),
    "no_fusion": (False, True, False, "grounding", False),
}
BASE_SEED = {"production": 100, "dn": 200, "no_fusion": 300}


def config(name):
    fusion, decouple, still, _, _ = CASES[name]
    kw = dict(d_model=C, nhead=8, num_encoder_layers=ENC_LAYERS, num_decoder_layers=DEC_LAYERS, dim_feedforward=D_FFN,
              dropout=0.1, activation="relu", return_intermediate_dec=True, num_feature_levels=len(SHAPES),
              dec_n_points=4, enc_n_points=4, two_stage=True, two_stage_num_proposals=K, look_forward_twice=True,
              mixed_selection=False, use_checkpoint=False)
    flags = dict(use_early_fusion=fusion, num_vl_layers=VL_LAYERS, decouple_tgt=decouple, still_tgt_for_both=still,
                 lang_dim=LANG, vl_hidden_dim=VL_HIDDEN)
    return kw, flags


def masks():
    """Per level [N, H, W] bool: image 0 unpadded; image 1 valid in the top-left ceil(0.6 H) x ceil(0.7 W)."""
    out = []
    for h, w in SHAPES:
        m = torch.zeros(N, h, w, dtype=torch.bool)
        m[1, math.ceil(0.6 * h):, :] = True
        m[1, :, math.ceil(0.7 * w):] = True
        out.append(m)
    return out


def attn_mask():
    """[Q, Q] bool, True = blocked: the matching queries do not see the DN queries, DN groups do not see each other."""
    ndn, q = DN_GROUPS * DN_PER_GROUP, DN_GROUPS * DN_PER_GROUP + K
    m = torch.zeros(q, q, dtype=torch.bool)
    m[ndn:, :ndn] = True
    for g in range(DN_GROUPS):
        a, b = g * DN_PER_GROUP, (g + 1) * DN_PER_GROUP
        m[a:b, :a] = True
        m[a:b, b:ndn] = True
    return m


def parameters(model, seed):
    """Redraw every parameter of ``model`` (this repo's class or the reference's: the names are the same) from the seed,
    in sorted name order, at a scale that keeps every layer's activations O(1)."""
    from torch import nn
    norms = {f"{mn}.weight" for mn, m in model.named_modules() if isinstance(m, nn.LayerNorm)}
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(model.named_parameters()):
            if name in norms:
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith("gamma_v") or name.endswith("gamma_l"):
                p.copy_(0.5 + 0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() >= 2:
                p.copy_(torch.randn(p.shape, generator=g) * p.shape[-1] ** -0.5)
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return dict(model.named_parameters())


def inputs(name, seed):
    """srcs / pos_embeds per level [N, C, H, W], masks, language features {hidden [N, T, 768], masks [N, T] int64},
    the DN queries (label [N, 10, C], unactivated boxes [N, 10, 4]) and attn_masks in the dn case."""
    g = torch.Generator().manual_seed(seed + 1)
    r = lambda *shape: torch.randn(*shape, generator=g)
    x = {"srcs": [r(N, C, h, w) for h, w in SHAPES], "pos_embeds": [r(N, C, h, w) for h, w in SHAPES], "masks": masks(),
         "hidden": r(N, T, LANG), "lang_masks": torch.tensor([[1] * T, [1] * 5 + [0] * (T - 5)], dtype=torch.int64)}
    if CASES[name][4]:
        ndn = DN_GROUPS * DN_PER_GROUP
        x["dn_label"], x["dn_bbox"] = r(N, ndn, C), r(N, ndn, 4)
        x["attn_masks"] = attn_mask()
    return x


def run(model, name, x, device):
    """The forward of ``model`` on the case (mask_on, so memory is returned too); -> (outputs by name, input leaves)."""
    to = lambda t: t.to(device)
    leaves = {"srcs": [to(s).requires_grad_(True) for s in x["srcs"]],
              "pos_embeds": [to(p).requires_grad_(True) for p in x["pos_embeds"]],
              "hidden": to(x["hidden"]).requires_grad_(True)}
    query_embed = (None, None)
    if "dn_label" in x:
        leaves["dn_label"], leaves["dn_bbox"] = to(x["dn_label"]).requires_grad_(True), to(x["dn_bbox"]).requires_grad_(True)
        query_embed = (leaves["dn_label"], leaves["dn_bbox"])
    lang = {"hidden": leaves["hidden"], "masks": to(x["lang_masks"])}
    out = model(leaves["srcs"], [to(m) for m in x["masks"]], leaves["pos_embeds"], query_embed, mask_on=True,
                language_dict_features=lang, task=CASES[name][3],
                attn_masks=to(x["attn_masks"]) if "attn_masks" in x else None)
    hs, memory, init_ref, inter_ref, enc_class, enc_coord, lang_out = out
    return {"hs": hs, "memory": memory, "init_reference": init_ref, "inter_references": inter_ref,
            "enc_outputs_class": enc_class, "enc_outputs_coord_unact": enc_coord, "lang_hidden": lang_out["hidden"]}, leaves


def cotangents(outputs, seed):
    """One random cotangent per differentiable output, drawn in the outputs' order."""
    g = torch.Generator().manual_seed(seed + 2)
    return {k: torch.randn(v.shape, generator=g) for k, v in outputs.items()}


def backward(outputs, cot):
    keys = [k for k, v in outputs.items() if v.requires_grad]
    torch.autograd.backward([outputs[k] for k in keys], [cot[k].to(outputs[k].device) for k in keys])


def attach_heads(model, still_classifier, mlp):
    """The detector's heads (ddetrs_dn.py with box refinement and two stages): DEC_LAYERS + 1 class heads and box MLPs,
    the last of each scoring the encoder memory."""
    from torch import nn
    model.decoder.class_embed = nn.ModuleList(still_classifier(C) for _ in range(DEC_LAYERS + 1))
    model.decoder.bbox_embed = nn.ModuleList(mlp(C, C, 4, 3) for _ in range(DEC_LAYERS + 1))
    return model
