"""Two-stage query selection of the DINO-style transformer (deformable_transformer_dino.py:132-162,216-224): the step
between the encoder and the decoder that scores every memory row, picks the ``num_proposals`` best per image and turns
their boxes into the decoder's initial reference points.

Class-head mirrors with the reference's parameter names, so that a checkpoint's ``class_embed.*`` loads unchanged:
    Still_Classifier:  body                                                               (deformable_detr.py:70-76)
    VL_Align:          dot_product_projection_text, log_scale, bias_lang, bias0           (deformable_detr.py:35-68)
``bbox_embed`` is the reference's ``MLP(256, 256, 4, 3)`` (modules/deformable_transformer.py).

CUDA fp32 tensors of width 256 run the kernels of csrc/msda_twostage.cuh around the two GEMMs (enc_output, bbox_embed);
CPU tensors run the reference's torch chain.  Any other width or dtype on the GPU raises.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from uninext_b200 import _cabi

from .deformable_transformer import gen_encoder_output_proposals

D_MODEL = 256


class Still_Classifier(nn.Module):
    """The encoder's binary class head under STILL_CLS_FOR_ENCODER: ``Linear(hidden_dim, 1)``."""

    def __init__(self, hidden_dim: int = D_MODEL):
        super().__init__()
        self.body = nn.Linear(hidden_dim, 1)

    def forward(self, x, lang_feat=None):
        return self.body(x)

    def logit_affine(self, n: int, lang_feat_pool=None):
        """-> (u [n, C], c [n], clamp): the head as ``logit = x . u[image] + c[image]``."""
        return self.body.weight[0].expand(n, -1), self.body.bias.expand(n), False


class VL_Align(nn.Module):
    """Vision-language alignment score against the language tokens: ``x . proj_text(normalize(e) / 2) / exp(log_scale)
    + normalize(e) . bias_lang + bias0``, clamped to +-5e4 when ``clamp_dot_product``."""

    def __init__(self, hidden_dim: int = D_MODEL, lang_dim: int = 768, log_scale: float = 0.0, prior_prob: float = 0.01,
                 clamp_dot_product: bool = True):
        super().__init__()
        self.clamp_dot_product = clamp_dot_product
        self.dot_product_projection_image = nn.Identity()
        self.dot_product_projection_text = nn.Linear(lang_dim, hidden_dim, bias=True)
        self.log_scale = nn.Parameter(torch.Tensor([log_scale]), requires_grad=True)
        self.bias_lang = nn.Parameter(torch.zeros(lang_dim), requires_grad=True)
        self.bias0 = nn.Parameter(torch.Tensor([-math.log((1 - prior_prob) / prior_prob)]), requires_grad=True)

    def forward(self, x, embedding):
        embedding = F.normalize(embedding, p=2, dim=-1)
        tokens = self.dot_product_projection_text(embedding / 2.0)
        bias = (torch.matmul(embedding, self.bias_lang) + self.bias0).unsqueeze(1).repeat(1, x.shape[1], 1)
        logit = torch.matmul(self.dot_product_projection_image(x), tokens.transpose(-1, -2)) / self.log_scale.exp() + bias
        if self.clamp_dot_product:
            logit = torch.clamp(logit, max=50000)
            logit = torch.clamp(logit, min=-50000)
        return logit

    def logit_affine(self, n: int, lang_feat_pool):
        """-> (u [n, C], c [n], clamp) for one pooled language feature per image ([n, lang_dim])."""
        if lang_feat_pool is None:
            raise ValueError("VL_Align needs lang_feat_pool")
        e = F.normalize(lang_feat_pool, p=2, dim=-1)
        u = self.dot_product_projection_text(e / 2.0) / self.log_scale.exp()
        return u, torch.matmul(e, self.bias_lang) + self.bias0, self.clamp_dot_product


class _Head(torch.autograd.Function):
    """y = enc_output(memory) -> (om = LayerNorm(keep ? y : b_e), logit = clamp(om . u[n] + c[n]))."""

    @staticmethod
    def forward(ctx, y, keep, b_e, gamma, beta, u, c, clamp, eps):
        n, s, w = y.shape
        om = torch.empty_like(y)
        logit = y.new_empty((n, s, 1))
        mean, rstd = y.new_empty((n, s)), y.new_empty((n, s))
        _cabi.call("msda_twostage_head_forward_f32", y, keep, b_e, gamma, beta, u, c, n, s, w, eps, int(clamp), om,
                   logit, mean, rstd, device=y.device)
        ctx.save_for_backward(y, keep, b_e, gamma, beta, u, c, mean, rstd)
        ctx.clamp = int(clamp)
        return om, logit

    @staticmethod
    def backward(ctx, g_om, g_logit):
        y, keep, b_e, gamma, beta, u, c, mean, rstd = ctx.saved_tensors
        n, s, w = y.shape
        g_om, g_logit = g_om.contiguous(), g_logit.contiguous()
        g_y = torch.empty_like(y)
        g_be, g_gamma, g_beta = torch.empty_like(b_e), torch.empty_like(gamma), torch.empty_like(beta)
        g_u, g_c = torch.empty_like(u), torch.empty_like(c)
        nbytes = _cabi.workspace("msda_twostage_head_workspace", n, s, w)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
        _cabi.call("msda_twostage_head_backward_f32", g_om, g_logit, y, keep, b_e, gamma, beta, u, c, mean, rstd, n, s,
                   w, ctx.clamp, g_y, g_be, g_gamma, g_beta, g_u, g_c, ws, nbytes, device=y.device)
        return g_y, None, g_be, g_gamma, g_beta, g_u, g_c, None, None


class _Select(torch.autograd.Function):
    """(box, proposals, logit) -> (coord_unact = box + proposals, reference_points = sigmoid(coord_unact[top-k]), top-k
    rows).  Gradient flows to ``box`` only, as in the reference (proposals are constants, indices carry none)."""

    @staticmethod
    def forward(ctx, box, proposals, logit, k):
        n, s, _ = box.shape
        coord = torch.empty_like(box)
        ref = box.new_empty((n, k, 4))
        idx = torch.empty((n, k), dtype=torch.int64, device=box.device)
        nbytes = _cabi.workspace("msda_twostage_select_workspace", n, s, k)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=box.device)
        _cabi.call("msda_twostage_select_forward_f32", logit, box, proposals, n, s, k, coord, ref, idx, ws, nbytes,
                   device=box.device)
        ctx.save_for_backward(ref, idx)
        ctx.mark_non_differentiable(idx)
        ctx.sizes = (n, s, k)
        return coord, ref, idx

    @staticmethod
    def backward(ctx, g_coord, g_ref, _g_idx):
        ref, idx = ctx.saved_tensors
        n, s, k = ctx.sizes
        g_box = g_coord.contiguous().clone()              # the kernel adds the selected rows' gradient in place
        _cabi.call("msda_twostage_select_backward_f32", g_ref.contiguous(), ref, idx, n, s, k, g_box,
                   device=g_box.device)
        return g_box, None, None, None


def _check_cuda(memory, enc_output, enc_output_norm, class_embed):
    if memory.dtype != torch.float32 or memory.shape[-1] != D_MODEL:
        raise ValueError(f"two_stage_select on CUDA takes fp32 memory of width {D_MODEL}, got {memory.dtype} "
                         f"width {memory.shape[-1]}")
    if not (isinstance(enc_output, nn.Linear) and enc_output.in_features == D_MODEL and enc_output.out_features == D_MODEL
            and enc_output.bias is not None):
        raise ValueError(f"enc_output must be nn.Linear({D_MODEL}, {D_MODEL}) with a bias")
    if not (isinstance(enc_output_norm, nn.LayerNorm) and tuple(enc_output_norm.normalized_shape) == (D_MODEL,)
            and enc_output_norm.elementwise_affine and enc_output_norm.bias is not None):
        raise ValueError(f"enc_output_norm must be nn.LayerNorm({D_MODEL}) with weight and bias")
    if not isinstance(class_embed, (Still_Classifier, VL_Align)):
        raise TypeError("class_embed must be Still_Classifier or VL_Align")
    for p in (enc_output.weight, enc_output.bias, enc_output_norm.weight, enc_output_norm.bias):
        if p.dtype != torch.float32 or p.device != memory.device:
            raise ValueError("enc_output / enc_output_norm parameters must be fp32 on the memory's device")


def two_stage_select(memory, memory_padding_mask, spatial_shapes, enc_output, enc_output_norm, class_embed, bbox_embed,
                     num_proposals: int, lang_feat_pool=None):
    """Encoder memory [N, S, C] -> (enc_outputs_class [N, S, 1], enc_outputs_coord_unact [N, S, 4],
    reference_points [N, k, 4], topk_proposals [N, k] int64), k = ``num_proposals``
    (deformable_transformer_dino.py:216-224 preceded by :132-162).

    ``reference_points`` is not detached: its gradient reaches ``bbox_embed``, ``enc_output``, ``enc_output_norm`` and
    ``memory``.  ``topk_proposals`` orders each image's rows by descending class logit, ties by ascending row
    (``torch.sort(descending=True, stable=True)``), NaN first.  Rows that are padded or whose proposal is invalid enter
    the heads as zeros and have proposals of +inf, so when selected their reference points are 1 with zero gradient.
    The caller keeps the language pooling (``agg_lang_feat``) and the DN concatenation."""
    n, s, _ = memory.shape
    k = int(num_proposals)
    if k < 1 or k > s:
        raise RuntimeError(f"two_stage_select: num_proposals = {k} is out of range for {s} rows")
    output_proposals, keep = gen_encoder_output_proposals(memory_padding_mask, spatial_shapes)
    if not memory.is_cuda:
        output_memory = memory.masked_fill(~keep, float(0))
        output_memory = enc_output_norm(enc_output(output_memory))
        enc_outputs_class = class_embed(output_memory, None if lang_feat_pool is None else lang_feat_pool.unsqueeze(1))
        enc_outputs_coord_unact = bbox_embed(output_memory) + output_proposals
        topk_proposals = torch.sort(enc_outputs_class[..., 0], dim=1, descending=True, stable=True)[1][:, :k]
        topk_coords_unact = torch.gather(enc_outputs_coord_unact, 1, topk_proposals.unsqueeze(-1).repeat(1, 1, 4))
        return enc_outputs_class, enc_outputs_coord_unact, topk_coords_unact.sigmoid(), topk_proposals
    _check_cuda(memory, enc_output, enc_output_norm, class_embed)
    with torch.autocast("cuda", enabled=False):
        y = F.linear(memory, enc_output.weight, enc_output.bias)
        u, c, clamp = class_embed.logit_affine(n, lang_feat_pool)
        u, c = u.float().contiguous(), c.float().reshape(n).contiguous()
        om, enc_outputs_class = _Head.apply(y.contiguous(), keep.to(torch.uint8).contiguous(), enc_output.bias,
                                            enc_output_norm.weight, enc_output_norm.bias, u, c, bool(clamp),
                                            float(enc_output_norm.eps))
        box = bbox_embed(om).contiguous()
        coord, ref, idx = _Select.apply(box, output_proposals, enc_outputs_class, k)
    return enc_outputs_class, coord, ref, idx
