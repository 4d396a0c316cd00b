"""Detection post-processing for UNINEXT inference (DESIGN.md section 3.13, row f-6): grounding logits -> class scores ->
class-aware NMS -> top-k boxes, scores and labels for the whole batch in two kernel launches
(uninext_b200/csrc/msda_detpost.cuh, ``msda_detpost_f32``).

Every image-style inference call of the reference runs, per image in a Python loop (``uninext_img.py:393-472``, and its
copy ``uninext_vid.py:1092-1197``):

    logits = convert_grounding_to_od_logits(box_cls[i], C, positive_map)   # a Python loop over the classes
    prob = logits.sigmoid(); prob = sqrt(prob * iou_pred[i].sigmoid())      # with the IoU branch
    keep = batched_nms(box_cxcywh_to_xyxy(box_pred[i]), *prob.max(1), 0.7)  # OTA on; a keep list of host-known length
    topk(prob[keep].flatten(), min(max_num_inst, K*C)); boxes -> xyxy, Boxes.scale(w, h)

which synchronises with the host once per class and again for the NMS result.  ``postprocess_detections`` computes the
same outputs without a host round trip, so it can be captured into a CUDA graph with the rest of a frame.

``select_track_detections`` does the same for the video trackers' paths (``inference_mot`` and ``inference_vis`` of
``uninext_vid.py``): score threshold, class-aware NMS and the kept queries, ready for ``tracker.match``.
"""
from __future__ import annotations

import functools
from typing import Dict, NamedTuple, Optional, Sequence, Tuple, Union

import torch

from uninext_b200 import _cabi

MAX_QUERIES, MAX_TOKENS, MAX_CLASSES = 1024, 256, 4096      # include/msda_b200.h (and msda_trackpost.h)
LAUNCHES = 2                                                  # per call, whatever B, Q, C and nms_iou (both entry points)


class Detections(NamedTuple):
    """``[B, max_num_inst]`` each (``boxes`` ``[B, max_num_inst, 4]``), ``count`` ``[B]``.  Entries at and past
    ``count[b]`` hold the fill values: score 0, label -1, query_index -1, box 0."""
    scores: torch.Tensor          # fp32, descending per image
    labels: torch.Tensor          # int32 class index c, 0-based (the reference's pred_classes)
    boxes: torch.Tensor           # fp32 xyxy in pixels of the image size (Boxes.scale(w, h))
    query_index: torch.Tensor     # int32 index into the Q queries: gathers the matching mask logits
    count: torch.Tensor           # int32 valid entries per image, min(max_num_inst, K*C)


@functools.lru_cache(maxsize=64)
def _csr(items: Tuple[Tuple[int, Tuple[int, ...]], ...], device: torch.device) -> Tuple[torch.Tensor, torch.Tensor]:
    """positive map content -> (class_start [C + 1], tokens [nnz]) int32 on the device.  Cached per
    distinct content: one small host-to-device copy the first time, none afterwards (nor inside a graph capture)."""
    starts, toks = [0], []
    for _, t in items:
        toks.extend(t)
        starts.append(len(toks))
    return torch.tensor(starts, dtype=torch.int32, device=device), torch.tensor(toks, dtype=torch.int32, device=device)


# Cached device tensors that a captured CUDA graph reads: never freed, whatever the LRU caches above drop.
_CAPTURED: Dict[int, torch.Tensor] = {}


@functools.lru_cache(maxsize=256)
def _sizes(sizes: Tuple[Tuple[int, int], ...], device: torch.device) -> torch.Tensor:
    return torch.tensor(sizes, dtype=torch.int32, device=device)


def positive_map_to_csr(positive_map: Dict[int, Sequence[int]], num_tokens: int,
                        device: Union[str, torch.device] = "cuda") -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's ``positive_map_label_to_token`` ({label: [token, ...]}, labels 1..C) as CSR on ``device``: class c
    (= label - 1) owns ``tokens[class_start[c]:class_start[c + 1]]``, in the listed order.  Raises ValueError for labels
    that are not exactly 1..C (the reference raises IndexError or leaves zero columns), for an empty token list (the
    reference's mean is NaN) and for a token outside [0, num_tokens)."""
    labels = sorted(int(k) for k in positive_map)
    if not labels or labels != list(range(1, len(labels) + 1)):
        raise ValueError(f"positive_map: labels must be exactly 1..C, got {labels[:8]}{'...' if len(labels) > 8 else ''}")
    items = tuple((k, tuple(int(t) for t in positive_map[k])) for k in labels)
    for k, t in items:
        if not t:
            raise ValueError(f"positive_map: label {k} has no tokens")
        if min(t) < 0 or max(t) >= num_tokens:
            raise ValueError(f"positive_map: label {k} has a token outside [0, {num_tokens}): {list(t)}")
    if len(items) > MAX_CLASSES:
        raise ValueError(f"positive_map: at most {MAX_CLASSES} classes, got {len(items)}")
    return _csr(items, torch.device(device))


def postprocess_detections(box_cls: torch.Tensor, box_pred: torch.Tensor, positive_map: Dict[int, Sequence[int]],
                           image_sizes: Union[Sequence[Sequence[int]], torch.Tensor], iou_pred: Optional[torch.Tensor] = None,
                           nms_iou: Optional[float] = 0.7, max_num_inst: int = 100) -> Detections:
    """box_cls [B, Q, T] token logits, box_pred [B, Q, 4] normalised cxcywh, iou_pred [B, Q, 1] / [B, Q] or None,
    positive_map = the reference's ``positive_map_label_to_token``, image_sizes = B pairs (h, w) or an int32 CUDA tensor
    [B, 2].  ``nms_iou=None`` is the reference's OTA-off branch (no NMS); ``max_num_inst`` is 100 for detection, 1 for
    grounding and SOT.  Q <= 1024, T <= 256, C <= 4096, 1 <= max_num_inst <= Q*C.

    The result equals the reference chain's scores, pred_classes, pred_boxes and the query each came from, in its order.
    One deliberate difference: ``uninext_vid.py``'s copy calls ``topk(100)`` without ``min`` and raises when K*C < 100;
    here ``count`` is then below 100, as in ``uninext_img.py``.  Non-fp32 inputs are cast with ``.float()``.

    Reference call sites (``projects/UNINEXT/uninext/``), with ``nms = 0.7 if self.ota else None``:
      * ``uninext_img.py:284`` (detection / grounding): ``postprocess_detections(box_cls, box_pred, positive_map,
        image_sizes, iou_pred, nms, 100 if task == "detection" else 1)``; the masks follow with
        ``n = int(d.count[b]); paste_masks(mask_pred[b][d.query_index[b, :n]], image_size, output_size, 4, self.mask_thres)``.
      * ``uninext_vid.py:511`` (SOT), ``:751`` (``inference_ytbvos``) and ``:889`` (``inference_ytbvos_3f``): all three
        are reached only from ``task == "sot"`` with the map ``{1: [0]}``, so ``max_num_inst=1``:
        ``postprocess_detections(box_cls, box_pred, {1: [0]}, image_sizes, iou_pred, nms, 1)``.  The two VOS sites pass
        ``binary_mask=False``: their masks are the probabilities cropped to the image, ``paste_masks(mask_pred[b][
        d.query_index[b, :1]], image_size, image_size, 4, threshold=None)``.

    The positive map and the image sizes become small device tensors, cached per distinct content.  Those used while a
    CUDA graph is being captured are kept for the life of the process, so the graph's replays never read freed memory
    even after the cache has dropped them.
    """
    b, q, t, dev, iou_pred = _check_inputs("postprocess_detections", box_cls, box_pred, iou_pred)
    class_start, tokens = positive_map_to_csr(positive_map, t, dev)
    c = class_start.numel() - 1
    k = int(max_num_inst)
    if not 1 <= k <= q * c:
        raise ValueError(f"postprocess_detections: need 1 <= max_num_inst <= Q*C = {q * c}, got {k}")
    sizes = _device_sizes("postprocess_detections", "image_sizes", "image sizes", image_sizes, b, dev)
    _hold_while_capturing(class_start, tokens, sizes)
    x = box_cls.float().contiguous()
    bx = box_pred.float().contiguous()
    ws_bytes = _cabi.workspace("msda_detpost_workspace", b, q, t, c, k)
    out = Detections(torch.empty((b, k), dtype=torch.float32, device=dev), torch.empty((b, k), dtype=torch.int32, device=dev),
                     torch.empty((b, k, 4), dtype=torch.float32, device=dev),
                     torch.empty((b, k), dtype=torch.int32, device=dev), torch.empty((b,), dtype=torch.int32, device=dev))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=dev)
    _cabi.call("msda_detpost_f32", x, bx, iou_pred, class_start, tokens, sizes, b, q, t, c, int(nms_iou is not None),
               float(nms_iou) if nms_iou is not None else 0.0, k, out.scores, out.labels, out.query_index, out.boxes,
               out.count, ws, ws.numel(), device=dev)
    return out


def _check_inputs(fn: str, box_cls: torch.Tensor, box_pred: torch.Tensor, iou_pred: Optional[torch.Tensor]):
    """(B, Q, T, device, iou_pred as contiguous fp32 or None) after the checks both entry points share."""
    if not (box_cls.is_cuda and box_pred.is_cuda and (iou_pred is None or iou_pred.is_cuda)):
        raise RuntimeError(f"{fn}: Not implemented on the CPU")
    if box_cls.dim() != 3 or box_pred.shape != (*box_cls.shape[:2], 4):
        raise ValueError(f"{fn}: need box_cls [B, Q, T] and box_pred [B, Q, 4], got "
                         f"{tuple(box_cls.shape)} and {tuple(box_pred.shape)}")
    b, q, t = box_cls.shape
    if iou_pred is not None:
        if iou_pred.shape not in ((b, q, 1), (b, q)):
            raise ValueError(f"{fn}: iou_pred must be [B, Q, 1] or [B, Q], got {tuple(iou_pred.shape)}")
        iou_pred = iou_pred.float().contiguous()
    if not (1 <= q <= MAX_QUERIES and 1 <= t <= MAX_TOKENS):
        raise ValueError(f"{fn}: need 1 <= Q <= {MAX_QUERIES} and 1 <= T <= {MAX_TOKENS}, got Q={q}, T={t}")
    return b, q, t, box_cls.device, iou_pred


def _device_sizes(fn: str, arg: str, what: str, sizes, b: int, dev: torch.device) -> torch.Tensor:
    """B pairs (h, w) -> an int32 [B, 2] device tensor, cached per distinct content; a CUDA tensor [B, 2] as int32."""
    if isinstance(sizes, torch.Tensor):
        if not sizes.is_cuda or sizes.shape != (b, 2):
            raise ValueError(f"{fn}: an {arg} tensor must be a CUDA tensor [B, 2] (h, w)")
        return sizes.to(torch.int32).contiguous()
    out = _sizes(tuple((int(s[0]), int(s[1])) for s in sizes), dev)
    if out.shape != (b, 2):
        raise ValueError(f"{fn}: {b} images but {out.shape[0]} {what}")
    return out


def _hold_while_capturing(*held: torch.Tensor) -> None:
    """Keep cached device tensors that a CUDA graph being captured reads for the life of the process."""
    if torch.cuda.is_current_stream_capturing():
        for t in held:
            _CAPTURED[id(t)] = t


class TrackDetections(NamedTuple):
    """``[B, Q]`` each (``boxes`` ``[B, Q, 4]``), ``count`` ``[B]``, in keep order.  Entries at and past ``count[b]``
    hold the fill values: score 0, label -1, query_index -1, box 0."""
    scores: torch.Tensor          # fp32 max over the classes (the reference's box_score), descending per frame
    labels: torch.Tensor          # int32 argmax over the classes, 0-based (det_labels)
    boxes: torch.Tensor           # fp32: xyxy in pixels of ori_size ("xyxy_pixels"), or normalised cxcywh ("cxcywh")
    query_index: torch.Tensor     # int32 index into the Q queries: gathers pred_inst_embed and pred_masks
    count: torch.Tensor           # int32 kept queries per frame, >= 1


_BOX_FORMATS = {"cxcywh": _cabi.TRACKPOST_CXCYWH, "xyxy_pixels": _cabi.TRACKPOST_XYXY_PIXELS}


def select_track_detections(box_cls: torch.Tensor, box_pred: torch.Tensor, positive_map: Dict[int, Sequence[int]],
                            iou_pred: Optional[torch.Tensor] = None, *, score_thres: float, nms_iou: float,
                            box_format: str, ori_sizes: Union[Sequence[Sequence[int]], torch.Tensor, None] = None
                            ) -> TrackDetections:
    """The per-frame detections the video trackers hand to ``tracker.match`` (``uninext_vid.py:1224-1250``
    ``inference_mot``, ``:1380-1415`` ``inference_vis``), for B frames in two kernel launches
    (``msda_trackpost_f32``, include/msda_trackpost.h) without a host round trip.

    box_cls [B, Q, T] token logits, box_pred [B, Q, 4] normalised cxcywh, iou_pred [B, Q, 1] / [B, Q] or None,
    positive_map = the reference's ``positive_map_label_to_token``.  Per frame: the class scores of
    ``postprocess_detections``; ``max_score`` and ``label`` per query; the candidates ``max_score > score_thres`` in
    query order; torchvision's ``batched_nms`` on them at ``nms_iou`` (0.7 for MOT, 0.9 for VIS); the kept queries in
    keep order (score descending, ties to the lower query).  When no query passes the threshold, the result is the one
    query of the largest ``max_score``, without NMS; on exact ties the lowest query, where the reference leaves the
    choice to CPU ``topk``.  ``box_format="xyxy_pixels"`` gives MOT's ``det_bboxes[:, :4]``: each box scaled by
    (W, H, W, H) of ``ori_sizes[b]`` = (h, w) (B pairs or an int32 CUDA tensor [B, 2]), then converted to xyxy.  The
    reference scales ``pred_boxes`` in place; here the input is left as it is.  ``box_format="cxcywh"`` gives VIS's
    normalised boxes unchanged.  Q <= 1024, T <= 256, C <= 4096.  Non-fp32 inputs are cast with ``.float()``.

    The caller reads ``n = int(count[b])`` (the one host read per frame) and passes ``query_index[b, :n]``'s rows of
    ``pred_inst_embed`` and ``pred_masks`` to the tracker (INTEGRATION.md section 6).
    """
    fn = "select_track_detections"
    b, q, t, dev, iou_pred = _check_inputs(fn, box_cls, box_pred, iou_pred)
    if box_format not in _BOX_FORMATS:
        raise ValueError(f"{fn}: box_format must be one of {sorted(_BOX_FORMATS)}, got {box_format!r}")
    class_start, tokens = positive_map_to_csr(positive_map, t, dev)
    c = class_start.numel() - 1
    sizes = None
    if box_format == "xyxy_pixels":
        if ori_sizes is None:
            raise ValueError(f"{fn}: box_format='xyxy_pixels' needs ori_sizes")
        sizes = _device_sizes(fn, "ori_sizes", "ori_sizes", ori_sizes, b, dev)
    _hold_while_capturing(class_start, tokens, *(() if sizes is None else (sizes,)))
    x = box_cls.float().contiguous()
    bx = box_pred.float().contiguous()
    ws_bytes = _cabi.workspace("msda_trackpost_workspace", b, q, t, c)
    out = TrackDetections(torch.empty((b, q), dtype=torch.float32, device=dev),
                          torch.empty((b, q), dtype=torch.int32, device=dev),
                          torch.empty((b, q, 4), dtype=torch.float32, device=dev),
                          torch.empty((b, q), dtype=torch.int32, device=dev), torch.empty((b,), dtype=torch.int32, device=dev))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=dev)
    _cabi.call("msda_trackpost_f32", x, bx, iou_pred, class_start, tokens, sizes, b, q, t, c, float(score_thres),
               float(nms_iou), _BOX_FORMATS[box_format], out.scores, out.labels, out.query_index, out.boxes, out.count,
               ws, ws.numel(), device=dev)
    return out
