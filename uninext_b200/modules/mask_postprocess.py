"""Mask pasting for UNINEXT inference (DESIGN.md section 3.12, row f-5): stride-4 mask logits -> masks at the original
image size in one kernel (uninext_b200/csrc/msda_maskpaste.cuh, ``msda_mask_paste_f32``).

Every inference path of the reference runs the same torch chain on the logits of the CondInst head
(``dynamic_mask_with_coords``):

    F.interpolate(logits, size=(4*H4, 4*W4), mode="bilinear", align_corners=False).sigmoid() [> mask_thres]
      [:, :, :h, :w]                                        # crop the padding (h, w = resized image size)
    F.interpolate(..., size=(H_out, W_out), mode="nearest")  # original image size

and materialises each step at the padded input resolution.  ``paste_masks`` computes the same masks with one launch that
writes nothing but its result.

``paste_masks_rle`` and ``encode_masks_rle`` go one step further for the evaluators and trackers, which copy every mask
to the host and run-length encode it there with ``pycocotools.mask.encode``: they return the same ``{"size", "counts"}``
dicts, computed on the device (csrc/msda_maskrle.cuh, DESIGN.md section 3.14) with two host synchronisations per call.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
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
        _cabi.call("msda_mask_paste_f32", x, i, hs, ws, stride, h, w, out_h, out_w, float(threshold) if binary else 0.0,
                   int(binary), out, device=x.device)
    return out.view(torch.bool) if binary else out


def _check_paste_args(mask_logits, image_size, output_size, mask_stride, fn):
    """paste_masks' argument checks."""
    if not mask_logits.is_cuda:
        raise RuntimeError(f"{fn}: Not implemented on the CPU")
    if mask_logits.dim() == 4 and mask_logits.shape[1] == 1:
        mask_logits = mask_logits[:, 0]
    if mask_logits.dim() != 3:
        raise ValueError(f"{fn}: mask_logits must be [I, Hs, Ws] or [I, 1, Hs, Ws], got {tuple(mask_logits.shape)}")
    i, hs, ws = mask_logits.shape
    h, w = (int(v) for v in image_size)
    out_h, out_w = (int(v) for v in output_size)
    stride = int(mask_stride)
    if stride < 1 or not (1 <= h <= stride * hs and 1 <= w <= stride * ws) or out_h < 1 or out_w < 1:
        raise ValueError(f"{fn}: need 1 <= image_size <= mask_stride * logits size and a positive output size; "
                         f"got logits {hs}x{ws}, stride {stride}, image_size {(h, w)}, output_size {(out_h, out_w)}")
    return mask_logits, i, hs, ws, h, w, out_h, out_w, stride


def paste_masks_rle(mask_logits: torch.Tensor, image_size: Sequence[int], output_size: Sequence[int], mask_stride: int = 4,
                    threshold: float = 0.5) -> List[dict]:
    """The COCO RLE of ``paste_masks(mask_logits, image_size, output_size, mask_stride, threshold)``, bit for bit, without
    storing the full-resolution masks: one ``{"size": [H_out, W_out], "counts": bytes}`` per instance, what
    ``pycocotools.mask.encode(np.asfortranarray(mask[:, :, None].astype(np.uint8)))[0]`` returns for that mask.  The
    arguments and their checks are paste_masks', except that ``threshold`` must be a number: RLE is binary.

    Reference call sites (``projects/UNINEXT/uninext/``), each one call for all instances:
      * ``uninext_vid.py:1425-1432`` (``inference_vis``, per track: paste, ``> 0.5``, ``.cpu()``, ``mask_util.encode``):
        ``paste_masks_rle(output_mask[indices], image_sizes, ori_size, 4, 0.5)``.
      * ``uninext_vid.py:1263-1271`` + ``:1686-1700`` (``inference_mot`` with ``mots=True``, then
        ``encode_track_results``): ``paste_masks_rle(track_masks, image_size, ori_size, 4, 0.5)``.
    """
    if threshold is None:
        raise ValueError("paste_masks_rle: threshold must be a number: run-length encoding is binary")
    mask_logits, i, hs, ws, h, w, out_h, out_w, stride = _check_paste_args(mask_logits, image_size, output_size,
                                                                           mask_stride, "paste_masks_rle")
    if i == 0:
        return []
    x = mask_logits.float().contiguous()
    return _encode(x.device, i, out_h, out_w, "msda_mask_rle_count_f32", x, i, hs, ws, stride, h, w, out_h, out_w,
                   float(threshold))


def encode_masks_rle(masks: torch.Tensor) -> List[dict]:
    """COCO RLE of binary masks [I, H, W] (``torch.bool`` or ``torch.uint8``, nonzero = set) on the GPU: one
    ``{"size": [H, W], "counts": bytes}`` per instance, what ``pycocotools.mask.encode`` returns for ``masks[i] != 0``.

    Reference call site: ``detectron2/evaluation/coco_evaluation.py:478-490`` (``instances_to_coco_json``, every COCO /
    LVIS / RefCOCO mask evaluation) encodes each ``pred_masks`` row on the host; ``encode_masks_rle(pred_masks)`` before
    the instances move to the CPU gives the same list (the evaluator still decodes ``counts`` to str).
    """
    if not masks.is_cuda:
        raise RuntimeError("encode_masks_rle: Not implemented on the CPU")
    if masks.dim() != 3 or masks.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"encode_masks_rle: masks must be bool or uint8 [I, H, W], got {masks.dtype} "
                         f"{tuple(masks.shape)}")
    i, out_h, out_w = masks.shape
    if i == 0:
        return []
    if out_h < 1 or out_w < 1:
        raise ValueError(f"encode_masks_rle: masks must have at least one pixel, got {tuple(masks.shape)}")
    m = masks.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    return _encode(m.device, i, out_h, out_w, "msda_mask_rle_count_u8", m, i, out_h, out_w)


def _encode(device, i, out_h, out_w, count, *count_args) -> List[dict]:
    """Both steps of a call: the entry point ``count`` on ``count_args`` and the workspace, then msda_mask_rle_encode.
    Two host synchronisations: one reads the number of boundaries B, which sizes the positions (4 B each) and the
    characters (at most 7 per count, B + I counts); one brings the offsets and characters back."""
    n = _cabi.workspace("msda_mask_rle_workspace", i, out_h, out_w)
    ws = torch.empty(n, dtype=torch.uint8, device=device)
    _cabi.call(count, *count_args, ws, n, device=device)
    boundaries = int(ws[: 8 * (i * out_w + 1)].view(torch.int64)[-1])                    # synchronisation 1
    pos = torch.empty(4 * boundaries, dtype=torch.uint8, device=device)
    head = 8 * (i + 1)
    out = torch.empty(head + 7 * (boundaries + i), dtype=torch.uint8, device=device)     # byte offsets, characters
    _cabi.call("msda_mask_rle_encode", i, out_h, out_w, boundaries, ws, n, pos if boundaries else None, out,
               out.data_ptr() + head, device=device)
    host = torch.empty(out.numel(), dtype=torch.uint8, pin_memory=True)
    host.copy_(out, non_blocking=True)                                                   # on device's current stream
    torch.cuda.current_stream(device).synchronize()                                      # synchronisation 2
    buf = host.numpy()
    offs = buf[:head].view(np.int64)
    data = buf[head:head + int(offs[i])].tobytes()
    size = [out_h, out_w]
    return [{"size": list(size), "counts": data[offs[k]:offs[k + 1]]} for k in range(i)]
