"""UNINEXT's early-fusion block: ``BiMultiHeadAttention``, ``BiAttentionBlock`` and ``VLFuse`` with the reference's
constructor arguments and parameter names (fuse_helper.py:7-179, vlfusion.py:64-120), so a UNINEXT checkpoint's fusion
weights load unchanged.

The attention core -- logits, both clamps, the masked vision softmax, the text softmax, both dropouts and the two
products -- runs in the fused CUDA kernels of msda_vlfuse.cuh (DESIGN.md section 3.11), which never store the
[B*H, S, T] logits.  When torch allows TF32 matmuls (``allow_tf32``, ``set_float32_matmul_precision("high")`` or
``fp32_precision = "tf32"``) the kernels of msda_vlfuse_tc.cuh run its products on TF32 tensor cores instead.  On bf16
inputs the kernels of msda_vlfuse_bf16.cuh run them on bf16 tensor cores; ``op_dtype=torch.bfloat16`` on the modules
casts the core's inputs to bf16.  The six projections are cuBLAS GEMMs (``F.linear``).  ``vl_attention_torch`` restates
the core with torch ops; it serves CPU tensors, ``stable_softmax_2d=True``, other dtypes and shapes outside the kernels'
limits (head_dim 128 / 256, T <= 256).
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn.functional as F
from torch import nn

from .. import _cabi
from .._precision import tf32_allowed
from .deformable_layers import fp32_under_autocast

MAX_TEXT_TOKENS = 256
HEAD_DIMS = (128, 256)
MASK_FILL = -9e15          # fuse_helper.py:100


def text_bias(attention_mask_l, T: int):
    """The additive mask the reference builds (fuse_helper.py:96-107): the mask value itself where it is non-zero,
    -9e15 where it is zero, added to the fp32 logits.  A fully padded row therefore gets one and the same logit in every
    column, and its softmax is uniform."""
    if attention_mask_l is None:
        return None
    assert attention_mask_l.dim() == 2 and attention_mask_l.shape[1] == T, attention_mask_l.shape
    return attention_mask_l.masked_fill(attention_mask_l == 0, MASK_FILL).to(torch.float32).contiguous()


def vl_attention_torch(q, k, vv, vl, bias=None, clamp_min=True, clamp_max=True, dropout_p=0.0, training=False,
                       stable_softmax_2d=False):
    """The attention core with torch ops, in the reference's order of operations.  q, vv: [B, S, H, d] (q already
    scaled); k, vl: [B, T, H, d]; bias: [B, T] from ``text_bias`` or None.  Returns O_v [B, S, H, d], O_l [B, T, H, d]."""
    x = torch.einsum("bshd,bthd->bhst", q, k)
    if stable_softmax_2d:
        x = x - x.max()
    if clamp_min:
        x = x.clamp(min=-50000)
    if clamp_max:
        x = x.clamp(max=50000)
    y = x.transpose(2, 3)
    y = y - y.max(dim=-1, keepdim=True)[0]
    if clamp_min:
        y = y.clamp(min=-50000)
    if clamp_max:
        y = y.clamp(max=50000)
    p_l = y.softmax(dim=-1)
    if bias is not None:
        x = x + bias[:, None, None, :].to(x.dtype)
    p_v = x.softmax(dim=-1)
    p_v = F.dropout(p_v, p=dropout_p, training=training)
    p_l = F.dropout(p_l, p=dropout_p, training=training)
    o_v = torch.einsum("bhst,bthd->bshd", p_v, vl)
    o_l = torch.einsum("bhts,bshd->bthd", p_l, vv)
    return o_v, o_l


def fused_supported(q, k, stable_softmax_2d=False, vv=None, vl=None) -> bool:
    """Whether the CUDA kernels serve this call (anything else runs ``vl_attention_torch``): fp32 q and k, or q, k, vv
    and vl all bf16."""
    if q.dtype == torch.float32:
        dtype_ok = k.dtype == torch.float32
    else:
        dtype_ok = q.dtype == torch.bfloat16 and all(t is not None and t.dtype == torch.bfloat16 for t in (k, vv, vl))
    return (q.is_cuda and k.is_cuda and not stable_softmax_2d and dtype_ok
            and q.shape[-1] in HEAD_DIMS and 1 <= k.shape[1] <= MAX_TEXT_TOKENS and q.shape[1] >= 1)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _workspace(B, H, S, T, D, device):
    lib = _cabi.load()
    n = ctypes.c_int64(0)
    _cabi.check(lib.msda_vlfuse_workspace(B, H, S, T, D, ctypes.byref(n)), "msda_vlfuse_workspace")
    return torch.empty(max(n.value, 16), dtype=torch.uint8, device=device)


def draw_seed(device):
    """A dropout seed drawn from torch's CUDA generator: it follows torch.manual_seed and is drawn anew on every replay of
    a captured CUDA graph."""
    return torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=device)


def dropout_masks(seed, B, H, S, T, p):
    """The keep-masks (1.0 / 0.0) the kernels apply for this seed: vision [B, H, S, T], text [B, H, T, S]."""
    mv = torch.empty(B, H, S, T, dtype=torch.float32, device=seed.device)
    ml = torch.empty(B, H, T, S, dtype=torch.float32, device=seed.device)
    _cabi.check(_cabi.load().msda_vlfuse_dropout_mask_f32(_ptr(seed), B, H, S, T, ctypes.c_float(p), _ptr(mv), _ptr(ml),
                                                          _stream()), "msda_vlfuse_dropout_mask_f32")
    return mv, ml


MODES = ("f32", "tf32", "bf16")     # the C ABI's msda_vlfuse_{forward,backward}_<mode>


class VLAttentionFunction(torch.autograd.Function):
    """Fused attention core: (q, k, vv, vl) in [B, L, H, d] -> (O_v, O_l).  Saves O(S + T) statistics per head.  ``mode``
    selects the kernels (``MODES``; "bf16" takes and returns bf16 tensors, the others fp32); the backward runs in the
    forward's mode, since it recomputes the logits against the statistics the forward saved."""

    @staticmethod
    def forward(ctx, q, k, vv, vl, bias, clamp_min, clamp_max, dropout_p, seed, mode="f32"):
        q, k, vv, vl = (t.contiguous() for t in (q, k, vv, vl))
        B, S, H, D = q.shape
        T = k.shape[1]
        o_v = torch.empty_like(q)
        o_l = torch.empty_like(k)
        stats = torch.empty(B * H * (S + T) * 2, dtype=torch.float32, device=q.device)
        ws = _workspace(B, H, S, T, D, q.device)
        name = f"msda_vlfuse_forward_{mode}"
        _cabi.check(getattr(_cabi.load(), name)(
            _ptr(q), _ptr(k), _ptr(vv), _ptr(vl), _ptr(bias), B, H, S, T, D, int(clamp_min), int(clamp_max),
            ctypes.c_float(dropout_p), _ptr(seed), _ptr(o_v), _ptr(o_l), _ptr(stats), _ptr(ws), ws.numel(), _stream()),
            name)
        ctx.save_for_backward(q, k, vv, vl, bias, seed, o_v, o_l, stats)
        ctx.cfg = (clamp_min, clamp_max, dropout_p, mode)
        return o_v, o_l

    @staticmethod
    def backward(ctx, go_v, go_l):
        q, k, vv, vl, bias, seed, o_v, o_l, stats = ctx.saved_tensors
        clamp_min, clamp_max, dropout_p, mode = ctx.cfg
        B, S, H, D = q.shape
        T = k.shape[1]
        go_v = torch.zeros_like(o_v) if go_v is None else go_v.contiguous()
        go_l = torch.zeros_like(o_l) if go_l is None else go_l.contiguous()
        dq, dk, dvv, dvl = (torch.empty_like(t) for t in (q, k, vv, vl))
        ws = _workspace(B, H, S, T, D, q.device)
        name = f"msda_vlfuse_backward_{mode}"
        _cabi.check(getattr(_cabi.load(), name)(
            _ptr(go_v), _ptr(go_l), _ptr(q), _ptr(k), _ptr(vv), _ptr(vl), _ptr(bias), _ptr(o_v), _ptr(o_l), _ptr(stats),
            B, H, S, T, D, int(clamp_min), int(clamp_max), ctypes.c_float(dropout_p), _ptr(seed), _ptr(dq), _ptr(dk),
            _ptr(dvv), _ptr(dvl), _ptr(ws), ws.numel(), _stream()), name)
        return dq, dk, dvv, dvl, None, None, None, None, None, None


def vl_attention(q, k, vv, vl, bias=None, clamp_min=True, clamp_max=True, dropout_p=0.0, training=False,
                 stable_softmax_2d=False, seed=None):
    """The attention core, fused where ``fused_supported`` holds, else ``vl_attention_torch``.  ``seed`` (a CUDA int64
    tensor of one element) keys the fused dropout; by default one is drawn with ``draw_seed``.  The fused products run
    on bf16 tensor cores for bf16 inputs (outputs and gradients bf16), whatever the TF32 setting; for fp32 inputs on
    TF32 tensor cores when torch allows TF32 matmuls at the time of the forward (``tf32_allowed``), in fp32 otherwise.
    The backward keeps the forward's mode."""
    if not fused_supported(q, k, stable_softmax_2d, vv, vl):
        return vl_attention_torch(q, k, vv, vl, bias, clamp_min, clamp_max, dropout_p, training, stable_softmax_2d)
    p = float(dropout_p) if training else 0.0
    if p > 0.0 and seed is None:
        seed = draw_seed(q.device)
    mode = "bf16" if q.dtype == torch.bfloat16 else ("tf32" if tf32_allowed() else "f32")
    return VLAttentionFunction.apply(q, k, vv, vl, bias, bool(clamp_min), bool(clamp_max), p, seed if p > 0.0 else None,
                                     mode)


def _fuse_flag(cfg, name, default):
    if cfg is None:
        return default
    return bool(getattr(cfg.MODEL.DYHEAD.FUSE_CONFIG, name))


def _check_op_dtype(op_dtype):
    if op_dtype not in (None, torch.bfloat16):
        raise ValueError(f"op_dtype must be None or torch.bfloat16, not {op_dtype!r}")
    return op_dtype


class BiMultiHeadAttention(nn.Module):
    """fuse_helper.py:7-139.  The three softmax / clamp flags come from ``cfg.MODEL.DYHEAD.FUSE_CONFIG`` when a cfg is
    given, else from the keyword arguments (defaults: the reference config's).

    ``op_dtype`` (new, no reference counterpart): None keeps the reference's fp32 block (run in fp32 under autocast);
    ``torch.bfloat16`` leaves autocast on and runs the attention core in bf16 -- q, k and both values are cast to bf16
    before it and its outputs back to the projections' dtype after it.  Parameters stay fp32."""

    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, cfg=None, stable_softmax_2d=False,
                 clamp_min_for_underflow=True, clamp_max_for_overflow=True, op_dtype=None):
        super().__init__()
        self.op_dtype = _check_op_dtype(op_dtype)
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.head_dim = embed_dim // num_heads
        self.v_dim = v_dim
        self.l_dim = l_dim
        assert self.head_dim * num_heads == embed_dim, (embed_dim, num_heads)
        self.scale = self.head_dim ** (-0.5)
        self.dropout = dropout
        self.v_proj = nn.Linear(v_dim, embed_dim)
        self.l_proj = nn.Linear(l_dim, embed_dim)
        self.values_v_proj = nn.Linear(v_dim, embed_dim)
        self.values_l_proj = nn.Linear(l_dim, embed_dim)
        self.out_v_proj = nn.Linear(embed_dim, v_dim)
        self.out_l_proj = nn.Linear(embed_dim, l_dim)
        self.stable_softmax_2d = _fuse_flag(cfg, "STABLE_SOFTMAX_2D", stable_softmax_2d)
        self.clamp_min_for_underflow = _fuse_flag(cfg, "CLAMP_MIN_FOR_UNDERFLOW", clamp_min_for_underflow)
        self.clamp_max_for_overflow = _fuse_flag(cfg, "CLAMP_MAX_FOR_OVERFLOW", clamp_max_for_overflow)
        for lin in (self.v_proj, self.l_proj, self.values_v_proj, self.values_l_proj, self.out_v_proj, self.out_l_proj):
            nn.init.xavier_uniform_(lin.weight)
            lin.bias.data.fill_(0)

    @fp32_under_autocast
    def forward(self, v, l, attention_mask_l=None):
        B, S, _ = v.shape
        T = l.shape[1]
        H, D = self.num_heads, self.head_dim
        q = (self.v_proj(v) * self.scale).view(B, S, H, D)
        k = self.l_proj(l).view(B, T, H, D)
        vv = self.values_v_proj(v).view(B, S, H, D)
        vl = self.values_l_proj(l).view(B, T, H, D)
        proj_dtype = q.dtype
        if self.op_dtype is not None:
            q, k, vv, vl = (t.to(self.op_dtype) for t in (q, k, vv, vl))
        o_v, o_l = vl_attention(q, k, vv, vl, text_bias(attention_mask_l, T), self.clamp_min_for_underflow,
                                self.clamp_max_for_overflow, self.dropout, self.training, self.stable_softmax_2d)
        o_v, o_l = o_v.to(proj_dtype), o_l.to(proj_dtype)
        return self.out_v_proj(o_v.reshape(B, S, self.embed_dim)), self.out_l_proj(o_l.reshape(B, T, self.embed_dim))


class BiAttentionBlock(nn.Module):
    """fuse_helper.py:142-179 (BiAttentionBlockForCheckpoint): pre-LayerNorm on both streams, the attention, then
    v + gamma_v * delta_v and l + gamma_l * delta_l.  UNINEXT builds it with drop_path = 0; other values are refused.
    ``op_dtype``: see ``BiMultiHeadAttention``."""

    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, drop_path=0.0, init_values=1e-4, cfg=None,
                 op_dtype=None, **attn_flags):
        super().__init__()
        if drop_path != 0.0:
            raise ValueError("BiAttentionBlock: only drop_path = 0 (what UNINEXT builds) is implemented")
        self.op_dtype = _check_op_dtype(op_dtype)
        self.layer_norm_v = nn.LayerNorm(v_dim)
        self.layer_norm_l = nn.LayerNorm(l_dim)
        self.attn = BiMultiHeadAttention(v_dim, l_dim, embed_dim, num_heads, dropout=dropout, cfg=cfg, op_dtype=op_dtype,
                                         **attn_flags)
        self.gamma_v = nn.Parameter(init_values * torch.ones(v_dim))
        self.gamma_l = nn.Parameter(init_values * torch.ones(l_dim))

    @fp32_under_autocast
    def forward(self, v, l, attention_mask_l=None, task=None):
        v = self.layer_norm_v(v)
        l = self.layer_norm_l(l)
        delta_v, delta_l = self.attn(v, l, attention_mask_l=attention_mask_l)
        return v + self.gamma_v * delta_v, l + self.gamma_l * delta_l


class VLFuse(nn.Module):
    """vlfusion.py:64-120: the early-fusion block over the reference's feature dict
    ``{"visual": [B, S, img_dim], "lang": {"hidden": [B, T, lang_dim], "masks": [B, T]}}``.  The reference recomputes the
    block under gradient checkpointing to bound its memory; the fused block stores no S x T tensor, so it runs once.
    ``op_dtype``: see ``BiMultiHeadAttention``."""

    def __init__(self, img_dim=256, lang_dim=768, embed_dim=2048, n_head=8, enc_layers=6, dropout=0.1, op_dtype=None,
                 **attn_flags):
        super().__init__()
        self.op_dtype = _check_op_dtype(op_dtype)
        self.b_attn = BiAttentionBlock(img_dim, lang_dim, embed_dim, n_head, dropout=dropout, drop_path=0.0,
                                       init_values=1.0 / enc_layers, op_dtype=op_dtype, **attn_flags)

    def forward(self, x, task=None):
        lang = x["lang"]
        visual, hidden = self.b_attn(x["visual"], lang["hidden"], lang["masks"], task)
        lang["hidden"] = hidden
        return {"visual": visual, "lang": lang}
