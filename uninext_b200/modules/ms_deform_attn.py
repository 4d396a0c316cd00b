"""``MSDeformAttn`` -- the nn.Module around the op, API- and checkpoint-compatible with the reference
(ops/modules/ms_deform_attn.py:30-116): same constructor, same four Linear sub-modules and parameter names
(``sampling_offsets``, ``attention_weights``, ``value_proj``, ``output_proj`` -- the optimiser selects
``sampling_offsets`` by name, train_net.py:163-164), same initialisation, same forward signature and maths.

``op_dtype=torch.bfloat16`` (new) stores value / output in bf16 for the op (fp32 sampling locations and attention
weights, fp32 accumulation); the default reproduces the reference's fp32 behaviour, including the fp32 cast under
autocast (ms_deform_attn.py:78).
"""
from __future__ import annotations

import math
import warnings

import torch
import torch.nn.functional as F
from torch import nn

from uninext_b200.functions import MSDeformAttnFunction, MSDeformAttnFunctionBF16
from uninext_b200.functions.fused import linear_colsum, sampling_prologue


_LEVELS_OK = {}


def check_levels(spatial_shapes: torch.Tensor, level_start_index, len_in: int) -> None:
    """The reference asserts ``(H_l * W_l).sum() == Len_in`` on every forward (ms_deform_attn.py:91), which costs a
    device->host sync per call.  The kernels trust the device-resident level table (an inconsistent one means
    out-of-bounds gathers and, in backward, out-of-bounds reds), so it IS validated -- once per distinct table: the result
    is cached on (storage, version, Len_in), later calls with the same tensor are free."""
    key = (spatial_shapes.data_ptr(), spatial_shapes._version, spatial_shapes.device, int(len_in),
           None if level_start_index is None else (level_start_index.data_ptr(), level_start_index._version))
    if _LEVELS_OK.get(key):
        return
    hw = spatial_shapes.detach().cpu().tolist()
    if any(h <= 0 or w <= 0 for h, w in hw):
        raise AssertionError(f"spatial_shapes must be positive, got {hw}")
    sizes = [h * w for h, w in hw]
    assert sum(sizes) == len_in, f"sum(H_l * W_l) = {sum(sizes)} != Len_in = {len_in}"            # ms_deform_attn.py:91
    if level_start_index is not None:
        starts = level_start_index.detach().cpu().tolist()
        want = [sum(sizes[:i]) for i in range(len(sizes))]
        assert starts == want, f"level_start_index {starts} does not match spatial_shapes (expected {want})"
    if len(_LEVELS_OK) > 256:
        _LEVELS_OK.clear()
    _LEVELS_OK[key] = True


def _power_of_two(n: int) -> bool:
    if not isinstance(n, int) or n < 0:
        raise ValueError(f"invalid input for _is_power_of_2: {n} (type: {type(n)})")
    return n != 0 and (n & (n - 1)) == 0


class MSDeformAttn(nn.Module):
    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4, op_dtype=None, fused=True, gemm="auto"):
        super().__init__()
        if d_model % n_heads:
            raise ValueError(f"d_model must be divisible by n_heads, but got {d_model} and {n_heads}")
        if not _power_of_two(d_model // n_heads):
            warnings.warn("MSDeformAttn: a power-of-two head dimension is what the tiled sm_90a kernels cover; "
                          "other sizes run on the generic kernel.")
        self.im2col_step = 64                     # accepted for drop-in compatibility (ms_deform_attn.py:48)
        self.d_model, self.n_levels, self.n_heads, self.n_points = d_model, n_levels, n_heads, n_points
        self.op_dtype = op_dtype
        self.fused = fused           # one-pass prologue / bias-gradient kernels around the GEMMs (same maths)
        # forward products of value_proj / output_proj / the sampling projection:
        #   "auto"    (default) hand-written TF32 GEMM kernels ("tcgen05" is the historical name; wgmma on sm_90a) when torch.backends.cuda.matmul.allow_tf32 is set (TF32
        #             rounding is then what the caller asked for), cuBLAS fp32 otherwise (1e-4 parity with the reference);
        #   "tcgen05" / "cublas" force one or the other.
        # value_proj's bias and padding-mask zeroing ride in the hand-written GEMM's epilogue (no masked_fill pass).
        self.gemm = gemm
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, d_model)
        self.output_proj = nn.Linear(d_model, d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        """Reference scheme (ms_deform_attn.py:62-76): zero offset/weight matrices; offset bias = a ring of directions,
        head k pointing at angle 2*pi*k/M (max-norm normalised), point p at distance p+1; Xavier projections."""
        with torch.no_grad():
            self.sampling_offsets.weight.zero_()
            ang = torch.arange(self.n_heads, dtype=torch.float32) * (2.0 * math.pi / self.n_heads)
            ring = torch.stack((ang.cos(), ang.sin()), dim=-1)
            ring = ring / ring.abs().amax(dim=-1, keepdim=True)
            dist = torch.arange(1, self.n_points + 1, dtype=torch.float32)
            bias = ring[:, None, None, :] * dist[None, None, :, None]                    # [M, 1, P, 2]
            self.sampling_offsets.bias.copy_(bias.expand(-1, self.n_levels, -1, -1).reshape(-1))
            self.attention_weights.weight.zero_()
            self.attention_weights.bias.zero_()
            nn.init.xavier_uniform_(self.value_proj.weight)
            self.value_proj.bias.zero_()
            nn.init.xavier_uniform_(self.output_proj.weight)
            self.output_proj.bias.zero_()

    def sampling_locations(self, offsets, reference_points, input_spatial_shapes):
        """offsets [N,Lq,M,L,P,2] (pixels) -> normalised locations (ms_deform_attn.py:103-112)."""
        ref = reference_points[:, :, None, :, None, :]
        if reference_points.shape[-1] == 2:
            wh = input_spatial_shapes.flip(-1).to(offsets.dtype)                          # (W_l, H_l)
            return ref + offsets / wh[None, None, None, :, None, :]
        if reference_points.shape[-1] == 4:
            return ref[..., :2] + offsets / self.n_points * ref[..., 2:] * 0.5
        raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} instead.")

    def _forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                 input_padding_mask, projected_value=None):
        n, lq, _ = query.shape
        s = input_flatten.shape[1]
        m, l, p = self.n_heads, self.n_levels, self.n_points
        check_levels(input_spatial_shapes, input_level_start_index, s)
        fused = (self.fused and query.is_cuda and query.dtype == torch.float32 and l * p <= 32
                 and not reference_points.requires_grad)
        if projected_value is not None:        # value_proj (+ padding mask) already applied, e.g. batched over decoder layers
            value = projected_value
        else:
            if fused:      # bias + padding-mask zeroing in the GEMM epilogue (ms_deform_attn.py:95-97 as one kernel)
                value = linear_colsum(input_flatten, self.value_proj, gemm=self.gemm, row_mask=input_padding_mask)
            else:
                value = self.value_proj(input_flatten)
                if input_padding_mask is not None:
                    value = value.masked_fill(input_padding_mask[..., None], 0.0)
        value = value.view(n, s, m, self.d_model // m)
        if fused:
            loc, weights = sampling_prologue(query, self.sampling_offsets, self.attention_weights, reference_points,
                                             input_spatial_shapes, m, l, p, gemm=self.gemm)
        else:
            offsets = self.sampling_offsets(query).view(n, lq, m, l, p, 2)
            weights = F.softmax(self.attention_weights(query).view(n, lq, m, l * p), dim=-1).view(n, lq, m, l, p)
            loc = self.sampling_locations(offsets, reference_points, input_spatial_shapes)
        if self.op_dtype == torch.bfloat16:
            out = MSDeformAttnFunctionBF16.apply(value, input_spatial_shapes, input_level_start_index, loc, weights,
                                                 self.im2col_step).to(query.dtype)
        else:
            out = MSDeformAttnFunction.apply(value, input_spatial_shapes, input_level_start_index, loc.contiguous(),
                                             weights.contiguous(), self.im2col_step)
        return linear_colsum(out, self.output_proj, gemm=self.gemm) if fused else self.output_proj(out)

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None, *, projected_value=None):
        """query [N,Lq,C]; reference_points [N,Lq,L,2|4]; input_flatten [N,S,C]; returns [N,Lq,C].
        ``projected_value`` (keyword-only, beyond the reference): ``value_proj(input_flatten)`` with the padding mask
        already applied, [N,S,C] -- see ``batched_value_proj``."""
        if self.op_dtype is None and torch.is_autocast_enabled():
            # reference: @custom_fwd(cast_inputs=float32) on forward (ms_deform_attn.py:78)
            with torch.autocast("cuda", enabled=False):
                f = lambda t: t.float() if t is not None and t.is_floating_point() else t
                return self._forward(f(query), f(reference_points), f(input_flatten), input_spatial_shapes,
                                     input_level_start_index, input_padding_mask, f(projected_value))
        return self._forward(query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                             input_padding_mask, projected_value)


# The strided-batched GEMM (shared A, batch = 6) plus its accumulate-in-place backward is an experiment: the decoder loops
# use it only on request (MSDA_BATCHED_VPROJ=1 or use_batched_value_proj(True)).
_BATCHED_VPROJ = __import__("os").environ.get("MSDA_BATCHED_VPROJ") == "1"


def use_batched_value_proj(flag=None) -> bool:
    """Query / set whether the decoder loops project the memory for all layers in one batched GEMM."""
    global _BATCHED_VPROJ
    if flag is not None:
        _BATCHED_VPROJ = bool(flag)
    return _BATCHED_VPROJ


def batched_value_proj(attn_modules, input_flatten, input_padding_mask=None):
    """``[m.value_proj(input_flatten) for m in attn_modules]`` with the padding mask applied, as ONE batched GEMM.
    The decoder's layers (and the ReID head's) all project the SAME encoder memory (deformable_transformer_dino.py:451-475:
    ``src`` is loop-invariant), so the six [256 -> 256] projections of 44 646 tokens become one [256 -> 6 x 256] launch,
    one bias epilogue and one mask pass instead of six of each.  Returns a list of [N, S, C] tensors (views of one
    [L, N*S, C] buffer), to be passed as ``projected_value=``."""
    from uninext_b200.functions.fused import batched_linear
    mods = list(attn_modules)
    n, s, c = input_flatten.shape
    w = torch.stack([m.value_proj.weight for m in mods])
    b = torch.stack([m.value_proj.bias for m in mods])
    y = batched_linear(input_flatten.reshape(n * s, c), w, b)                     # [L, N*S, C]
    if input_padding_mask is not None:
        y = y.masked_fill(input_padding_mask.reshape(1, n * s, 1), 0.0)
    return [y[i].view(n, s, -1) for i in range(len(mods))]
