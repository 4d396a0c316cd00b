"""Mask pasting for UNINEXT inference (DESIGN.md section 3.12, row f-5): stride-4 mask logits -> masks at the original
image size in one kernel (uninext_b200/csrc/msda_maskpaste.cuh, ``msda_mask_paste_f32``).

Every inference path of the reference runs the same torch chain on the logits of the CondInst head
(``dynamic_mask_with_coords``):

    F.interpolate(logits, size=(4*H4, 4*W4), mode="bilinear", align_corners=False).sigmoid() [> mask_thres]
      [:, :, :h, :w]                                        # crop the padding (h, w = resized image size)
    F.interpolate(..., size=(H_out, W_out), mode="nearest")  # original image size

and materialises each step at the padded input resolution.  ``paste_masks`` computes the same masks with one launch that
writes nothing but its result.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from uninext_b200 import _cabi


def paste_masks(mask_logits: torch.Tensor, image_size: Sequence[int], output_size: Sequence[int], mask_stride: int = 4,
                threshold: Optional[float] = 0.5) -> torch.Tensor:
    """mask_logits [I, Hs, Ws] or [I, 1, Hs, Ws] at ``mask_stride``; image_size = (h, w), the resized image inside the
    padded input, 1 <= h <= mask_stride * Hs (w likewise); output_size = (H_out, W_out).

    Returns ``torch.bool`` [I, H_out, W_out] with ``sigmoid(logit) > threshold``, or, with ``threshold=None``, the fp32
    probabilities.  The bool tensor is a view of the kernel's uint8 output, not a copy.  Non-fp32 logits are cast with
    ``.float()`` first, as the reference chain computes in fp32.

    Reference call sites (``projects/UNINEXT/uninext/``) and the one call each becomes:
      * ``uninext_img.py:474-479`` then ``models/ddetrs.py:1060-1064`` (``segmentation_postprocess``, nearest resize of the
        thresholded masks, ``.byte()``): ``paste_masks(mask_pred_i, image_size, (height, width), self.mask_stride,
        self.mask_thres)``; ``.byte()`` of the result if uint8 is wanted.
      * ``uninext_vid.py:620-622`` (probabilities of one track, resized to the original frame):
        ``paste_masks(track_masks, image_size, (height, width), 4, threshold=None)``.
      * ``uninext_vid.py:1187-1192`` (cropped but not resized; a bilinear resize follows in the callers): the crop is the
        output, ``paste_masks(mask_pred_per_image, image_size, image_size, self.mask_stride,
        self.mask_thres if binary_mask else None)``.
      * ``uninext_vid.py:1264-1266`` and ``:1335-1337`` (``> 0.5`` after the nearest resize):
        ``paste_masks(track_masks, image_size, ori_size, 4, 0.5)``.
      * ``uninext_vid.py:1428-1431`` (one track per call, ``> 0.5``): ``paste_masks(mask_i, image_sizes, ori_size, 4,
        0.5)[0]``.
    """
    if not mask_logits.is_cuda:
        raise RuntimeError("paste_masks: Not implemented on the CPU")
    if mask_logits.dim() == 4 and mask_logits.shape[1] == 1:
        mask_logits = mask_logits[:, 0]
    if mask_logits.dim() != 3:
        raise ValueError(f"paste_masks: mask_logits must be [I, Hs, Ws] or [I, 1, Hs, Ws], got {tuple(mask_logits.shape)}")
    i, hs, ws = mask_logits.shape
    h, w = (int(v) for v in image_size)
    out_h, out_w = (int(v) for v in output_size)
    stride = int(mask_stride)
    if stride < 1 or not (1 <= h <= stride * hs and 1 <= w <= stride * ws) or out_h < 1 or out_w < 1:
        raise ValueError(f"paste_masks: need 1 <= image_size <= mask_stride * logits size and a positive output size; "
                         f"got logits {hs}x{ws}, stride {stride}, image_size {(h, w)}, output_size {(out_h, out_w)}")
    binary = threshold is not None
    out = torch.empty((i, out_h, out_w), dtype=torch.uint8 if binary else torch.float32, device=mask_logits.device)
    if i > 0:
        x = mask_logits.float().contiguous()
        lib = _cabi.load()
        with torch.cuda.device(x.device):
            _cabi.check(lib.msda_mask_paste_f32(x.data_ptr(), i, hs, ws, stride, h, w, out_h, out_w,
                                                float(threshold) if binary else 0.0, int(binary), out.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), "msda_mask_paste_f32")
    return out.view(torch.bool) if binary else out
