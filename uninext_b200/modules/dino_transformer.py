"""DINO's whole deformable transformer on the library (deformable_transformer_dino.py:28-327,554-573): the encoder's input
preparation, the vision-language encoder loop, two-stage query selection, the denoising-query concatenation and the
decoder, with the reference's class names, forward signatures, return tuples and parameter names, so that a UNINEXT
checkpoint loads with ``strict=True`` and ``ddetrs_dn.py`` can use the class in place of the reference's.

    flatten_levels                    the pyramid -> the encoder's [N, S, C] inputs: one kernel (csrc/msda_flatten.cuh)
                                      and ``msda_valid_counts``; the level tables are cached, nothing reads the device
    DeformableTransformerEncoderVL    vl_layers.{i} (VLFuse or Identity), layers.{i}, lang_layers.{i} (Identity)
    DeformableTransformerVLDINO       encoder.*, decoder.*, level_embed, tgt_embed, enc_output, enc_output_norm, resizer

The reference's ``cfg`` fields become keyword arguments, as ``VLFuse`` does here.  Two-stage only, as the reference
asserts; the additional BERT layers and activation checkpointing raise.  On CUDA, after one warm-up call (the level
table check of ``MSDeformAttn``), forward and backward do not synchronise with the host, so a training step can be
captured with ``uninext_b200.graphs.GraphedStep``.
"""
from __future__ import annotations

import copy
import ctypes
import functools

import torch
import torch.nn.functional as F
from torch import nn

from uninext_b200 import _cabi

from .deformable_layers import DeformableTransformerDecoderLayer, DeformableTransformerEncoderLayer
from .deformable_transformer import (_LEVEL_TENSORS, DeformableTransformerDecoder, _level_args, _shapes_key,
                                     get_reference_points)
from .ms_deform_attn import MSDeformAttn
from .two_stage import two_stage_select
from .vl_fusion import BiMultiHeadAttention, VLFuse

MAX_LEVELS = 8            # msda_flatten.h
MAX_CHANNELS = 1024


def _cast_fp32(x):
    """torch.cuda.amp.custom_fwd(cast_inputs=torch.float32)'s cast: CUDA floating tensors to fp32, through lists, tuples
    and dicts."""
    if torch.is_tensor(x):
        return x.float() if x.is_cuda and x.is_floating_point() else x
    if isinstance(x, dict):
        return {k: _cast_fp32(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_cast_fp32(v) for v in x)
    return x


def _fp32_nested_under_autocast(forward):
    """The reference's ``@custom_fwd(cast_inputs=torch.float32)`` on forwards that take nested arguments (the ``srcs``
    list, ``language_dict_features``): under autocast the inputs are cast and the forward runs with autocast off."""
    @functools.wraps(forward)
    def wrapper(self, *args, **kwargs):
        if torch.is_autocast_enabled("cuda"):
            with torch.autocast("cuda", enabled=False):
                return forward(self, *_cast_fp32(args), **_cast_fp32(kwargs))
        return forward(self, *args, **kwargs)
    return wrapper


def _host_shapes(spatial_shapes):
    """The level shapes as Python ints.  For a level table that ``flatten_levels`` returned (a cached tensor) they are
    looked up, not read from the device."""
    if torch.is_tensor(spatial_shapes):
        for (key, _), (ss, _, _) in list(_LEVEL_TENSORS.items()):
            if ss is spatial_shapes:
                return key
    return _shapes_key(spatial_shapes)


_LEVEL_SIZES = {}


def _level_inv_sizes(shapes, device):
    """[L, 2] fp32 (1 / W_l, 1 / H_l), each an fp32 division, built once per (shapes, device).  torch divides a CUDA
    tensor by a Python scalar as a multiply by the scalar's fp32 reciprocal, so ``valid.float() / H`` on CUDA is
    ``valid.float() * (1 / H)`` bit for bit."""
    key = (shapes, str(device))
    hit = _LEVEL_SIZES.get(key)
    if hit is None:
        one = torch.ones((), dtype=torch.float32)
        inv = [[(one / torch.tensor(float(w))).item(), (one / torch.tensor(float(h))).item()] for h, w in shapes]
        hit = _LEVEL_SIZES[key] = torch.tensor(inv, dtype=torch.float32, device=device)
    return hit


def _ptrs(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _ints(values):
    return (ctypes.c_int * len(values))(*values)


class _FlattenLevels(torch.autograd.Function):
    """(level_embed, shapes, *srcs, *pos_embeds, *masks) -> (src_flatten, lvl_pos_embed_flatten, mask_flatten uint8)."""

    @staticmethod
    def forward(ctx, level_embed, shapes, *tensors):
        nl = len(shapes)
        srcs, pos, masks = tensors[:nl], tensors[nl:2 * nl], tensors[2 * nl:]
        n, c = srcs[0].shape[:2]
        s = sum(h * w for h, w in shapes)
        src_flat = level_embed.new_empty((n, s, c))
        pos_flat = level_embed.new_empty((n, s, c))
        mask_flat = torch.empty((n, s), dtype=torch.uint8, device=level_embed.device)
        _cabi.call("msda_flatten_levels_forward_f32", _ptrs(srcs), _ptrs(pos), _ptrs(masks),
                   _ints([h for h, _ in shapes]), _ints([w for _, w in shapes]), nl, n, c, level_embed, src_flat,
                   pos_flat, mask_flat, device=level_embed.device)
        ctx.mark_non_differentiable(mask_flat)
        ctx.cfg = (shapes, n, c, level_embed.shape[0])
        return src_flat, pos_flat, mask_flat

    @staticmethod
    def backward(ctx, g_src, g_pos, _g_mask):
        shapes, n, c, le_rows = ctx.cfg
        nl = len(shapes)
        need = ctx.needs_input_grad
        want_le, want_src, want_pos = need[0], any(need[2:2 + nl]), any(need[2 + nl:2 + 2 * nl])
        dev = g_src.device if g_src is not None else g_pos.device
        new = lambda h, w: torch.empty((n, c, h, w), dtype=torch.float32, device=dev)
        grad_src = [new(h, w) for h, w in shapes] if want_src else None
        grad_pos = [new(h, w) for h, w in shapes] if want_pos else None
        zeros = lambda: torch.zeros((n, sum(h * w for h, w in shapes), c), dtype=torch.float32, device=dev)
        g_src = (zeros() if g_src is None else g_src.contiguous()) if want_src else None
        g_pos = (zeros() if g_pos is None else g_pos.contiguous()) if (want_pos or want_le) else None
        hs, ws = _ints([h for h, _ in shapes]), _ints([w for _, w in shapes])
        g_le, work, nbytes = None, None, 0
        if want_le:
            g_le = torch.empty((le_rows, c), dtype=torch.float32, device=dev)     # rows past L embed no level
            g_le[nl:].zero_()
            nbytes = _cabi.workspace("msda_flatten_levels_workspace", hs, ws, nl, n, c)
            work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _cabi.call("msda_flatten_levels_backward_f32", g_src, g_pos, hs, ws, nl, n, c,
                   None if grad_src is None else _ptrs(grad_src), None if grad_pos is None else _ptrs(grad_pos), g_le,
                   work, nbytes, device=dev)
        per_level = lambda grads, i: None if grads is None or not need[i] else grads[(i - 2) % nl]
        return (g_le, None, *[per_level(grad_src, 2 + i) for i in range(nl)],
                *[per_level(grad_pos, 2 + nl + i) for i in range(nl)], *[None] * nl)


def _check_cuda(srcs, masks, pos_embeds, level_embed):
    nl = len(srcs)
    if not 1 <= nl <= MAX_LEVELS or len(masks) != nl or len(pos_embeds) != nl or level_embed.shape[0] < nl:
        raise ValueError(f"flatten_levels takes 1 .. {MAX_LEVELS} levels with one mask, one pos_embed and one level_embed "
                         f"row each, got {nl} srcs, {len(masks)} masks, {len(pos_embeds)} pos_embeds, "
                         f"{level_embed.shape[0]} level_embed rows")
    n, c = srcs[0].shape[:2]
    if c % 4 or c > MAX_CHANNELS:
        raise ValueError(f"flatten_levels on CUDA takes C % 4 == 0 and C <= {MAX_CHANNELS}, got C = {c}")
    dev = level_embed.device
    if level_embed.dtype != torch.float32 or level_embed.shape[1] != c:
        raise ValueError(f"level_embed must be fp32 [L, {c}], got {level_embed.dtype} {tuple(level_embed.shape)}")
    for s, p, m in zip(srcs, pos_embeds, masks):
        if s.dim() != 4 or s.shape[:2] != (n, c) or p.shape != s.shape or m.shape != (n, *s.shape[2:]):
            raise ValueError(f"flatten_levels: src {tuple(s.shape)}, pos {tuple(p.shape)}, mask {tuple(m.shape)} do not "
                             f"form one [{n}, {c}, H, W] level")
        if s.dtype != torch.float32 or p.dtype != torch.float32 or m.dtype != torch.bool:
            raise ValueError("flatten_levels on CUDA takes fp32 srcs and pos_embeds and bool masks")
        if s.device != dev or p.device != dev or m.device != dev:
            raise ValueError("flatten_levels: every tensor must be on level_embed's device")


def flatten_levels(srcs, masks, pos_embeds, level_embed):
    """The encoder's inputs from the pyramid (deformable_transformer_dino.py:181-201): srcs[l], pos_embeds[l]
    [N, C, H_l, W_l], masks[l] [N, H_l, W_l] bool, level_embed [>= L, C] -> (src_flatten [N, S, C], mask_flatten [N, S]
    bool, lvl_pos_embed_flatten [N, S, C] = pos + level_embed[l], spatial_shapes [L, 2] int64, level_start_index [L]
    int64, valid_ratios [N, L, 2] = (valid W / W, valid H / H)).

    CUDA: one kernel writes the three flattened tensors (bit for bit the reference's copies and one fp32 add), one more
    counts the valid extents; gradients reach srcs, pos_embeds and level_embed.  The level tables come from the tensors'
    shapes and are cached per pyramid, so nothing reads the device.  CPU tensors run the reference's torch chain."""
    shapes = tuple((int(s.shape[-2]), int(s.shape[-1])) for s in srcs)
    if not level_embed.is_cuda:
        src_flatten, mask_flatten, lvl_pos_embed_flatten = [], [], []
        for lvl, (src, mask, pos_embed) in enumerate(zip(srcs, masks, pos_embeds)):
            src_flatten.append(src.flatten(2).transpose(1, 2))
            mask_flatten.append(mask.flatten(1))
            lvl_pos_embed_flatten.append(pos_embed.flatten(2).transpose(1, 2) + level_embed[lvl].view(1, 1, -1))
        spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=level_embed.device)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
        ratios = []
        for m in masks:
            _, h, w = m.shape
            ratios.append(torch.stack(((~m[:, 0, :]).sum(1).float() / w, (~m[:, :, 0]).sum(1).float() / h), -1))
        return (torch.cat(src_flatten, 1), torch.cat(mask_flatten, 1), torch.cat(lvl_pos_embed_flatten, 1), spatial_shapes,
                level_start_index, torch.stack(ratios, 1))
    _check_cuda(srcs, masks, pos_embeds, level_embed)
    dev = level_embed.device
    n, nl = srcs[0].shape[0], len(srcs)
    src_flat, pos_flat, mask_flat = _FlattenLevels.apply(
        level_embed, shapes, *[s.contiguous() for s in srcs], *[p.contiguous() for p in pos_embeds],
        *[m.contiguous().view(torch.uint8) for m in masks])
    ss, lsi, s_total = _level_args(shapes, None, dev)
    counts = torch.empty((n, nl, 2), dtype=torch.int32, device=dev)              # (valid W, valid H)
    _cabi.call("msda_valid_counts", mask_flat, ss, lsi, n, s_total, nl, counts, device=dev)
    valid_ratios = counts.float() * _level_inv_sizes(shapes, dev)               # valid.float() / H, as get_valid_ratio
    return src_flat, mask_flat.view(torch.bool), pos_flat, ss, lsi, valid_ratios


def agg_lang_feat(features, mask, pool_type="average"):
    """Pooled language feature per image (deformable_transformer_dino.py:28-43): features [N, T, C], mask [N, T] ->
    [N, C], the mean over the valid tokens ("average") or their maximum ("max")."""
    if pool_type == "average":
        embedded = features * mask.unsqueeze(-1).float()
        return embedded.sum(1) / (mask.sum(-1).unsqueeze(-1).float())
    if pool_type == "max":
        return torch.stack([torch.max(features[i][mask[i]], 0)[0] for i in range(len(features))], dim=0)
    raise ValueError("pool_type should be average or max")


class FeatureResizer(nn.Module):
    """Linear, LayerNorm (eps 1e-12) and dropout (deformable_transformer_dino.py:554-573)."""

    def __init__(self, input_feat_size, output_feat_size, dropout, do_ln=True):
        super().__init__()
        self.do_ln = do_ln
        self.fc = nn.Linear(input_feat_size, output_feat_size, bias=True)
        self.layer_norm = nn.LayerNorm(output_feat_size, eps=1e-12)
        self.dropout = nn.Dropout(dropout)

    def forward(self, encoder_features):
        x = self.fc(encoder_features)
        if self.do_ln:
            x = self.layer_norm(x)
        return self.dropout(x)


class DeformableTransformerEncoderVL(nn.Module):
    """The vision-language encoder loop (deformable_transformer_dino.py:278-327): per layer the early-fusion block
    (``vl_layers.{i}``: a copy of ``vl_fusion_layer`` on the first ``num_vl_layers`` layers, Identity after), the encoder
    layer on the visual stream and ``lang_layers.{i}``.  The reference points come from one kernel."""

    def __init__(self, vl_fusion_layer, encoder_layer, lang_encoder_layer, num_layers, use_checkpoint=False,
                 num_vl_layers=None):
        super().__init__()
        if use_checkpoint:
            raise ValueError("activation checkpointing is not supported by this encoder")
        if not isinstance(lang_encoder_layer, nn.Identity):
            raise ValueError("the additional BERT language layers are not supported: lang_encoder_layer must be Identity")
        num_vl_layers = num_layers if num_vl_layers is None else num_vl_layers
        if not 0 <= num_vl_layers <= num_layers:
            raise ValueError(f"num_vl_layers = {num_vl_layers} is out of range for {num_layers} layers")
        self.vl_layers = nn.ModuleList(copy.deepcopy(vl_fusion_layer) if i < num_vl_layers else nn.Identity()
                                       for i in range(num_layers))
        self.layers = nn.ModuleList(copy.deepcopy(encoder_layer) for _ in range(num_layers))
        self.lang_layers = nn.ModuleList(copy.deepcopy(lang_encoder_layer) for _ in range(num_layers))
        self.num_layers = num_layers
        self.use_checkpoint = use_checkpoint

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        return get_reference_points(_host_shapes(spatial_shapes), valid_ratios, device)

    @_fp32_nested_under_autocast
    def forward(self, src, spatial_shapes, level_start_index, valid_ratios, pos=None, padding_mask=None,
                language_dict_features=None, task=None):
        output = {"visual": src, "lang": language_dict_features}
        reference_points = self.get_reference_points(spatial_shapes, valid_ratios, device=src.device)
        for vl_layer, layer, lang_layer in zip(self.vl_layers, self.layers, self.lang_layers):
            output = vl_layer(output) if isinstance(vl_layer, nn.Identity) else vl_layer(output, task=task)
            output["visual"] = layer(output["visual"], pos, reference_points, spatial_shapes, level_start_index,
                                     padding_mask)
            output = lang_layer(output)
        return output


class DeformableTransformerVLDINO(nn.Module):
    """deformable_transformer_dino.py:49-275.  Constructor arguments in the reference's order; the reference's ``cfg``
    fields are keyword arguments: ``use_early_fusion`` (MODEL.USE_EARLY_FUSION), ``num_vl_layers``
    (MODEL.DDETRS.NUM_VL_LAYERS), ``decouple_tgt`` / ``still_tgt_for_both`` (MODEL.DECOUPLE_TGT / STILL_TGT_FOR_BOTH),
    ``lang_dim`` (MODEL.LANGUAGE_BACKBONE.LANG_DIM), ``vl_hidden_dim`` (MODEL.DDETRS.VL_HIDDEN_DIM),
    ``use_additional_bert`` (MODEL.USE_ADDITIONAL_BERT, must be False).  ``two_stage`` must be True.

    The detector attaches ``decoder.class_embed`` and ``decoder.bbox_embed`` (num_decoder_layers + 1 heads each, as
    ddetrs_dn.py does); the last of each scores the encoder memory in ``two_stage_select``."""

    def __init__(self, d_model=256, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=1024,
                 dropout=0.1, activation="relu", return_intermediate_dec=False, num_feature_levels=4, dec_n_points=4,
                 enc_n_points=4, two_stage=False, two_stage_num_proposals=300, look_forward_twice=False,
                 mixed_selection=False, use_checkpoint=False, *, use_early_fusion=True, num_vl_layers=None,
                 decouple_tgt=True, still_tgt_for_both=True, lang_dim=768, vl_hidden_dim=2048,
                 use_additional_bert=False):
        super().__init__()
        if not two_stage:
            raise ValueError("DeformableTransformerVLDINO is two-stage only (the reference asserts two_stage in forward)")
        if use_additional_bert:
            raise ValueError("the additional BERT language layers (USE_ADDITIONAL_BERT) are not supported")
        if use_checkpoint:
            raise ValueError("activation checkpointing is not supported")
        self.d_model = d_model
        self.nhead = nhead
        self.two_stage = two_stage
        self.two_stage_num_proposals = two_stage_num_proposals
        encoder_layer = DeformableTransformerEncoderLayer(d_model, dim_feedforward, dropout, activation,
                                                          num_feature_levels, nhead, enc_n_points)
        vl_fusion_layer = (VLFuse(img_dim=d_model, lang_dim=lang_dim, embed_dim=vl_hidden_dim, n_head=8,
                                  enc_layers=num_encoder_layers, dropout=0.1) if use_early_fusion else nn.Identity())
        self.encoder = DeformableTransformerEncoderVL(vl_fusion_layer, encoder_layer, nn.Identity(), num_encoder_layers,
                                                      use_checkpoint, num_vl_layers=num_vl_layers)
        decoder_layer = DeformableTransformerDecoderLayer(d_model, dim_feedforward, dropout, activation,
                                                          num_feature_levels, nhead, dec_n_points)
        self.decoder = DeformableTransformerDecoder(d_model, decoder_layer, num_decoder_layers, return_intermediate_dec,
                                                    look_forward_twice, use_checkpoint)
        self.level_embed = nn.Parameter(torch.Tensor(num_feature_levels, d_model))
        self.tgt_embed = nn.Embedding(self.two_stage_num_proposals, d_model)
        self.enc_output = nn.Linear(d_model, d_model)
        self.enc_output_norm = nn.LayerNorm(d_model)
        self.mixed_selection = mixed_selection
        self._reset_parameters()
        self.resizer = FeatureResizer(input_feat_size=768, output_feat_size=d_model, dropout=0.1)
        self.decouple_tgt = decouple_tgt
        self.still_tgt_for_both = still_tgt_for_both

    def _reset_parameters(self):
        """deformable_transformer_dino.py:103-115 (the resizer is built after it, as there)."""
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, MSDeformAttn):
                m._reset_parameters()
            if isinstance(m, BiMultiHeadAttention):                     # fuse_helper.py:42-56
                for lin in (m.v_proj, m.l_proj, m.values_v_proj, m.values_l_proj, m.out_v_proj, m.out_l_proj):
                    nn.init.xavier_uniform_(lin.weight)
                    lin.bias.data.fill_(0)
        nn.init.normal_(self.level_embed)

    @_fp32_nested_under_autocast
    def forward(self, srcs, masks, pos_embeds, query_embed=None, mask_on=False, language_dict_features=None, task=None,
                attn_masks=None, return_src_info=False):
        assert language_dict_features is not None
        src_flatten, mask_flatten, lvl_pos_embed_flatten, spatial_shapes, level_start_index, valid_ratios = \
            flatten_levels(srcs, masks, pos_embeds, self.level_embed)
        shapes = [(int(s.shape[-2]), int(s.shape[-1])) for s in srcs]

        vl_feats_dict = self.encoder(src_flatten, spatial_shapes, level_start_index, valid_ratios, lvl_pos_embed_flatten,
                                     mask_flatten, language_dict_features, task=task)
        memory, language_dict_features = vl_feats_dict["visual"], vl_feats_dict["lang"]

        lang_feat_pool = agg_lang_feat(language_dict_features["hidden"], language_dict_features["masks"])
        ref_feat = self.resizer(lang_feat_pool).unsqueeze(1)
        bs = memory.shape[0]
        nl = self.decoder.num_layers
        enc_outputs_class, enc_outputs_coord_unact, reference_points, _ = two_stage_select(
            memory, mask_flatten, shapes, self.enc_output, self.enc_output_norm, self.decoder.class_embed[nl],
            self.decoder.bbox_embed[nl], self.two_stage_num_proposals, lang_feat_pool)
        if query_embed[1] is not None:                                  # denoising queries first
            reference_points = torch.cat([query_embed[1].sigmoid(), reference_points], 1)
        init_reference_out = reference_points
        tgt = self.tgt_embed.weight[None].repeat(bs, 1, 1)
        if query_embed[0] is not None:
            tgt = torch.cat([query_embed[0], tgt], 1)
        # "+ 0.0 *" keeps the unused branch's parameters in the graph, with zero gradients (deformable_transformer_dino.py:234-252)
        if self.decouple_tgt:
            if self.still_tgt_for_both or task == "detection":
                tgt_new = tgt + 0.0 * ref_feat
            elif task == "grounding":
                tgt_new = ref_feat + 0.0 * tgt
            else:
                raise ValueError("task should be detection or grounding")
        else:
            tgt_new = ref_feat.repeat(1, self.two_stage_num_proposals, 1)
            if query_embed[0] is not None:
                tgt_new = torch.cat([query_embed[0], tgt_new], 1)
            tgt_new += 0.0 * torch.sum(self.tgt_embed.weight)

        hs, inter_references = self.decoder(tgt_new, reference_points, memory, spatial_shapes, level_start_index,
                                            valid_ratios, query_pos=None, src_padding_mask=mask_flatten,
                                            attn_masks=attn_masks)
        inter_references_out = inter_references
        if mask_on:
            if return_src_info:
                src_info_dict = {"src": memory.detach(), "src_spatial_shapes": spatial_shapes,
                                 "src_level_start_index": level_start_index, "src_valid_ratios": valid_ratios,
                                 "src_padding_mask": mask_flatten}
                return (hs, memory, init_reference_out, inter_references_out, enc_outputs_class, enc_outputs_coord_unact,
                        language_dict_features, src_info_dict)
            return (hs, memory, init_reference_out, inter_references_out, enc_outputs_class, enc_outputs_coord_unact,
                    language_dict_features)
        return hs, init_reference_out, inter_references_out, enc_outputs_class, enc_outputs_coord_unact, language_dict_features
