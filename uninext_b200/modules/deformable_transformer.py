"""The pieces of the DINO-style deformable transformer that sit directly on the op's callers
(deformable_transformer_dino.py): the ReID head (two more decoder layers on detached queries, video configs), the
reference-point / proposal generators that feed the op, and the small position-embedding helpers they use.

Sub-module and parameter names are the reference's, so its checkpoints load unchanged:
    DeformableReidHead:   layers.{i}.<decoder layer>, ref_point_head.layers.{0,1}        (_dino.py:504-527)
    MLP:                  layers.{i}                                                       (_dino.py:589-609)
"""
from __future__ import annotations

import copy
import math

import torch
import torch.nn.functional as F
from torch import nn

from uninext_b200 import _cabi

from .deformable_layers import DeformableTransformerDecoderLayer, fp32_under_autocast
from .ms_deform_attn import batched_value_proj, use_batched_value_proj


def inverse_sigmoid(x, eps: float = 1e-5):
    """logit with both arguments of the log clamped at eps (uninext/util/misc.py:493-497)."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


def _projected_values(layers, src, src_padding_mask):
    """One batched value projection for all layers over the loop-invariant encoder memory (SURVEY.md section 8 f-2), when
    every layer is this repo's decoder layer; None otherwise (each layer then projects for itself)."""
    if use_batched_value_proj() and all(isinstance(l, DeformableTransformerDecoderLayer) for l in layers) and src.is_cuda \
            and len(layers) > 1:
        return batched_value_proj([l.cross_attn for l in layers], src, src_padding_mask)
    return None


class MLP(nn.Module):
    """Linear -> ReLU -> ... -> Linear (deformable_transformer_dino.py:575-609)."""

    def __init__(self, input_dim: int, hidden_dim: int, output_dim: int, num_layers: int):
        super().__init__()
        self.num_layers = num_layers
        dims = [input_dim] + [hidden_dim] * (num_layers - 1) + [output_dim]
        self.layers = nn.ModuleList(nn.Linear(i, o) for i, o in zip(dims[:-1], dims[1:]))

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = layer(x)
            if i < self.num_layers - 1:
                x = F.relu(x)
        return x


class _SinePosEmbed(torch.autograd.Function):
    """get_sine_pos_embed as one kernel per direction (msda_sine_pos_embed_forward/backward_f32)."""

    @staticmethod
    def forward(ctx, pos, num_pos_feats, temperature, exchange_xy):
        p2 = pos.contiguous().float()
        n = p2.shape[-1]
        r = p2.numel() // n
        out = torch.empty((*p2.shape[:-1], n * num_pos_feats), dtype=torch.float32, device=pos.device)
        _cabi.call("msda_sine_pos_embed_forward_f32", p2, r, n, num_pos_feats, float(temperature), int(exchange_xy),
                   out, device=pos.device)
        ctx.save_for_backward(p2)
        ctx.cfg = (r, n, num_pos_feats, float(temperature), int(exchange_xy), pos.dtype)
        return out

    @staticmethod
    def backward(ctx, g):
        (p2,) = ctx.saved_tensors
        r, n, f, t, xy, dt = ctx.cfg
        g = g.contiguous().float()
        gp = torch.empty_like(p2)
        _cabi.call("msda_sine_pos_embed_backward_f32", p2, g, r, n, f, t, xy, gp, device=p2.device)
        return gp.to(dt), None, None, None


def get_sine_pos_embed(pos_tensor: torch.Tensor, num_pos_feats: int = 128, temperature: int = 10000,
                       exchange_xy: bool = True) -> torch.Tensor:
    """[.., Q, n] positions in [0, 1] -> [.., Q, n * num_pos_feats] sine embedding (deformable_transformer_dino.py:612-646):
    component k, feature j = sin / cos (j even / odd) of ``pos_k * 2*pi / temperature ** (2 * (j // 2) / num_pos_feats)``;
    with ``exchange_xy`` the y block comes first.  CUDA tensors: one hand-written kernel per direction.  An odd
    ``num_pos_feats`` raises ValueError: the reference interleaves equal halves of sines and cosines, so it has no
    value to give."""
    if num_pos_feats % 2:
        raise ValueError(f"get_sine_pos_embed takes an even num_pos_feats, got {num_pos_feats}")
    if pos_tensor.is_cuda and pos_tensor.dtype == torch.float32:
        return _SinePosEmbed.apply(pos_tensor, int(num_pos_feats), temperature, bool(exchange_xy))
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=pos_tensor.device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    arg = pos_tensor.unsqueeze(-1) * (2 * math.pi) / dim_t                         # [.., n, F]
    emb = torch.stack((arg[..., 0::2].sin(), arg[..., 1::2].cos()), dim=-1).flatten(-2)
    order = list(range(pos_tensor.shape[-1]))
    if exchange_xy and len(order) >= 2:
        order[0], order[1] = 1, 0
    return emb[..., order, :].flatten(-2)


def valid_ratios_from_masks(masks):
    """Per level ``(valid_W / W, valid_H / H)`` from the padding masks [N, H_l, W_l] -> [N, L, 2]
    (get_valid_ratio, deformable_transformer_dino.py:164-171).  (With a flattened mask, msda_valid_counts gives the same
    counts in one launch: see gen_encoder_output_proposals.)"""
    out = []
    for m in masks:
        _, h, w = m.shape
        vh = (~m[:, :, 0]).sum(1).float() / h
        vw = (~m[:, 0, :]).sum(1).float() / w
        out.append(torch.stack((vw, vh), -1))
    return torch.stack(out, 1)


_PIXEL_CENTRES = {}


def _pixel_centres(shapes_key, device):
    """Un-normalised pixel centres (x + 0.5, y + 0.5) and (W_l, H_l) per flattened pyramid position: constants of the
    pyramid, built once per (shapes, device)."""
    key = (shapes_key, str(device))
    hit = _PIXEL_CENTRES.get(key)
    if hit is None:
        xy, wh = [], []
        for h, w in shapes_key:
            ys = torch.arange(h, dtype=torch.float32, device=device) + 0.5
            xs = torch.arange(w, dtype=torch.float32, device=device) + 0.5
            yy, xx = torch.meshgrid(ys, xs, indexing="ij")
            xy.append(torch.stack((xx.reshape(-1), yy.reshape(-1)), -1))
            wh.append(torch.tensor([float(w), float(h)], device=device).expand(h * w, 2))
        lvl = torch.cat([torch.full((h * w,), i, dtype=torch.long, device=device) for i, (h, w) in enumerate(shapes_key)])
        hit = _PIXEL_CENTRES[key] = (torch.cat(xy), torch.cat(wh), lvl)
    return hit


def _shapes_key(spatial_shapes):
    if torch.is_tensor(spatial_shapes):
        spatial_shapes = spatial_shapes.tolist()
    return tuple((int(h), int(w)) for h, w in spatial_shapes)


def _level_args(spatial_shapes, level_start_index, device):
    """(device [L,2] int64, device [L] int64, S) for the geometry kernels; host values come from the cached shapes key."""
    key = _shapes_key(spatial_shapes)
    hit = _LEVEL_TENSORS.get((key, str(device)))
    if hit is None:
        ss = torch.as_tensor(key, dtype=torch.long, device=device)
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
        hit = _LEVEL_TENSORS[(key, str(device))] = (ss, lsi, sum(h * w for h, w in key))
    return hit


_LEVEL_TENSORS = {}


def get_reference_points(spatial_shapes, valid_ratios, device=None):
    """Encoder reference points [N, S, L, 2] (deformable_transformer_dino.py:289-301): pixel centre of every pyramid
    position, normalised by the valid extent of ITS level, then scaled by every level's valid ratio.  CUDA: one kernel
    (msda_encoder_ref_points_f32, level table read on the device).  CPU: the pixel grid is a constant of ``spatial_shapes``
    and is cached; per call only one divide and one multiply remain."""
    device = device or valid_ratios.device
    if valid_ratios.is_cuda and valid_ratios.dtype == torch.float32 and not valid_ratios.requires_grad:
        ss, lsi, s_total = _level_args(spatial_shapes, None, valid_ratios.device)
        n, l = valid_ratios.shape[0], ss.shape[0]
        vr = valid_ratios.contiguous()
        ref = torch.empty((n, s_total, l, 2), dtype=torch.float32, device=vr.device)
        _cabi.call("msda_encoder_ref_points_f32", vr, ss, lsi, n, s_total, l, ref, device=vr.device)
        return ref
    xy, wh, lvl = _pixel_centres(_shapes_key(spatial_shapes), device)
    ref = xy[None] / (valid_ratios[:, lvl] * wh[None])                  # [N, S, 2]
    return ref[:, :, None] * valid_ratios[:, None]


def gen_encoder_output_proposals(memory_padding_mask, spatial_shapes, base_scale: float = 0.05):
    """Two-stage proposals from the pyramid geometry (the part of deformable_transformer_dino.py:132-162 that does not
    touch learned weights): -> (output_proposals [N, S, 4] in logit space, +inf where padded or outside (0.01, 0.99);
    keep [N, S, 1] bool = positions whose memory survives).  The caller applies ``enc_output`` / ``enc_output_norm`` to
    ``memory.masked_fill(~keep, 0)``."""
    shapes = _shapes_key(spatial_shapes)
    n = memory_padding_mask.shape[0]
    device = memory_padding_mask.device
    if memory_padding_mask.is_cuda:                 # two launches: valid extents per (image, level), then the proposals
        ss, lsi, s_total = _level_args(spatial_shapes, None, device)
        l = ss.shape[0]
        m8 = memory_padding_mask.to(torch.uint8).contiguous()
        counts = torch.empty((n, l, 2), dtype=torch.int32, device=device)
        prop = torch.empty((n, s_total, 4), dtype=torch.float32, device=device)
        keep = torch.empty((n, s_total, 1), dtype=torch.uint8, device=device)
        _cabi.call("msda_valid_counts", m8, ss, lsi, n, s_total, l, counts, device=device)
        _cabi.call("msda_encoder_proposals_f32", m8, counts, ss, lsi, n, s_total, l, float(base_scale), prop, keep,
                   device=device)
        return prop, keep.bool()
    xy, wh, lvl = _pixel_centres(shapes, device)
    counts, cur = [], 0
    for h, w in shapes:
        m = memory_padding_mask[:, cur:cur + h * w].view(n, h, w)
        counts.append(torch.stack(((~m[:, 0, :]).sum(1), (~m[:, :, 0]).sum(1)), -1))          # (valid_W, valid_H)
        cur += h * w
    valid = torch.stack(counts, 1).float()                                                       # [N, L, 2]
    grid = xy[None] / valid[:, lvl]                                    # (x + 0.5) / valid_W, (y + 0.5) / valid_H
    size = (base_scale * (2.0 ** lvl.float()))[None, :, None].expand(n, -1, 2)
    prop = torch.cat((grid, size), -1)
    ok = ((prop > 0.01) & (prop < 0.99)).all(-1, keepdim=True)
    prop = torch.log(prop / (1 - prop))
    keep = ok & ~memory_padding_mask.unsqueeze(-1)
    return prop.masked_fill(~keep, float("inf")), keep


class DeformableReidHead(nn.Module):
    """Two (``num_layers``) more decoder layers over the encoder memory, fed with detached decoder queries and their
    boxes (deformable_transformer_dino.py:504-527; ddetrs_vid.py calls it once per key / reference frame)."""

    def __init__(self, embed_dim, decoder_layer, num_layers):
        super().__init__()
        self.layers = nn.ModuleList(copy.deepcopy(decoder_layer) for _ in range(num_layers))
        self.num_layers = num_layers
        self.ref_point_head = MLP(2 * embed_dim, embed_dim, embed_dim, 2)
        self.op_dtype = getattr(decoder_layer, "op_dtype", None)

    @fp32_under_autocast
    def forward(self, tgt, reference_points, src, src_spatial_shapes, src_level_start_index, src_valid_ratios,
                query_pos=None, src_padding_mask=None, attn_masks=None):
        if reference_points.shape[-1] != 4:
            raise ValueError("reference_points.shape[-1] should be 4")
        ref_in = reference_points[:, :, None] * torch.cat((src_valid_ratios, src_valid_ratios), -1)[:, None]
        query_pos = self.ref_point_head(get_sine_pos_embed(ref_in[:, :, 0, :]))      # the same for every layer
        output = tgt
        values = _projected_values(self.layers, src, src_padding_mask)
        for i, layer in enumerate(self.layers):
            kw = {} if values is None else {"projected_value": values[i]}
            output = layer(output, query_pos, ref_in, src, src_spatial_shapes, src_level_start_index,
                           src_padding_mask, attn_masks, **kw)
        return output


class DeformableTransformerDecoder(nn.Module):
    """The DINO-style decoder loop around the decoder layers (deformable_transformer_dino.py:429-501): per layer the
    reference boxes are scaled by the valid ratios, turned into a sine embedding -> ``ref_point_head`` -> query_pos, the
    layer runs, and (when ``bbox_embed`` is attached by the detector, as the reference does) the boxes are refined and
    detached for the next layer.  ``src`` never changes inside the loop, so all layers' ``value_proj(src)`` run as one
    batched GEMM up front."""

    def __init__(self, embed_dim, decoder_layer, num_layers, return_intermediate=False, look_forward_twice=False,
                 use_checkpoint=False):
        super().__init__()
        self.layers = nn.ModuleList(copy.deepcopy(decoder_layer) for _ in range(num_layers))
        self.num_layers = num_layers
        self.return_intermediate = return_intermediate
        self.look_forward_twice = look_forward_twice
        self.use_checkpoint = use_checkpoint
        if use_checkpoint:
            raise ValueError("activation checkpointing is not supported by this decoder")
        self.ref_point_head = MLP(2 * embed_dim, embed_dim, embed_dim, 2)
        self.bbox_embed = None              # attached by the detector (iterative box refinement), like the reference
        self.class_embed = None
        self.op_dtype = getattr(decoder_layer, "op_dtype", None)

    @fp32_under_autocast
    def forward(self, tgt, reference_points, src, src_spatial_shapes, src_level_start_index, src_valid_ratios,
                query_pos=None, src_padding_mask=None, attn_masks=None):
        output = tgt
        bs = output.shape[0]
        if reference_points.dim() == 2:
            reference_points = reference_points.unsqueeze(0).repeat(bs, 1, 1)
        values = _projected_values(self.layers, src, src_padding_mask)
        intermediate, intermediate_refs = [], []
        for lid, layer in enumerate(self.layers):
            if reference_points.shape[-1] == 4:
                ref_in = reference_points[:, :, None] * torch.cat((src_valid_ratios, src_valid_ratios), -1)[:, None]
            else:
                assert reference_points.shape[-1] == 2
                ref_in = reference_points[:, :, None] * src_valid_ratios[:, None]
            query_pos = self.ref_point_head(get_sine_pos_embed(ref_in[:, :, 0, :]))
            kw = {} if values is None else {"projected_value": values[lid]}
            output = layer(output, query_pos, ref_in, src, src_spatial_shapes, src_level_start_index, src_padding_mask,
                           attn_masks, **kw)
            if self.bbox_embed is not None:                                   # iterative box refinement
                tmp = self.bbox_embed[lid](output)
                if reference_points.shape[-1] == 4:
                    new_ref = (tmp + inverse_sigmoid(reference_points)).sigmoid()
                else:
                    new_ref = torch.cat((tmp[..., :2] + inverse_sigmoid(reference_points), tmp[..., 2:]), -1).sigmoid()
                reference_points = new_ref.detach()
            if self.return_intermediate:
                intermediate.append(output)
                intermediate_refs.append(new_ref if (self.look_forward_twice and self.bbox_embed is not None)
                                         else reference_points)
        if self.return_intermediate:
            return torch.stack(intermediate), torch.stack(intermediate_refs)
        return output, reference_points
