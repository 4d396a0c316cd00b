"""The video trackers' association steps on the GPU, each in eight kernel launches per frame with its state in device
tensors and no host synchronisation until the caller reads the result:

- ``IDOLTracker`` for video instance segmentation (DESIGN.md section 3.18, row f-10): mask NMS, bi-softmax matching,
  new ids, backdrops and the track memory (uninext_b200/csrc/msda_tracker.cuh, ``msda_idol_match_f32``,
  include/msda_tracker.h).  The reference's ``IDOL_Tracker.match`` (``projects/UNINEXT/uninext/models/tracker.py:207-298``)
  walks every pair of detections in Python for its mask NMS, and reads the device back for every pair, every matched
  row and every backdrop test.
- ``QuasiDenseTracker`` for BDD MOT and MOTS (DESIGN.md section 3.19, row f-11): box duplicate removal, bi-softmax
  matching against the tracklets and last frame's backdrops, new ids and the track memory
  (uninext_b200/csrc/msda_qdtrack.cuh, ``msda_qdtrack_match_f32``, include/msda_qdtrack.h).  The reference's
  ``QuasiDenseEmbedTracker.match`` (``models/tracker.py:304-503``) loops over the rows in Python for its duplicate
  removal, its matching and its backdrops, rebuilds its memo from per-tracklet dicts every frame, and reads the device
  back for every matched row.
"""
from __future__ import annotations

import warnings
from typing import List, NamedTuple, Optional, Tuple

import torch

from uninext_b200 import _cabi

MAX_ROWS, MAX_TRACKLETS, MAX_MEMORY = 1024, 1024, 64              # include/msda_tracker.h
LAUNCHES = 8                                                        # per frame, whatever n, the tracklets and the branch
_STATE_HEADER, _FLAGS = 4, 2                                        # MSDA_IDOL_STATE_INTS(T) = 4 + 5 T; the error word


class TrackResult(NamedTuple):
    """One frame's association, on the device.  ``IDOLTracker``: ``ids[r]`` for input row r: >= 0 a tracklet id, -1 a
    backdrop, -2 neither, -3 removed by the mask NMS (or past the frame's row count); ``rows[:count]`` the rows with an
    id >= 0 in row order (-1 after them).  ``QuasiDenseTracker``: ``order[p]`` the input row at score-sorted position p
    (-1 past the row count) and ``ids[p]`` its id: >= 0 a tracklet id, -1 left, -2 suppressed, -3 a duplicate (or past
    the row count); ``rows[:count]`` the input rows with an id >= 0 in sorted order."""
    ids: torch.Tensor             # int32 [n_cap]
    rows: torch.Tensor            # int32 [n_cap]
    count: torch.Tensor           # int32 [1]
    order: Optional[torch.Tensor] = None      # int32 [n_cap], QuasiDenseTracker only


def _check_devices(who: str, dev: torch.device, **tensors) -> None:
    """Every input on the tracker's CUDA device."""
    for name, t in tensors.items():
        if not t.is_cuda:
            raise RuntimeError(f"{who}: Not implemented on the CPU")
        if t.device != dev:
            raise ValueError(f"{who}: {name} is on {t.device}, the tracker on {dev}")


def _workspace(cache: dict, key, query: str, *sizes, device) -> torch.Tensor:
    """The workspace for these sizes, queried and allocated once per key."""
    ws = cache.get(key)
    if ws is None:
        ws = cache[key] = torch.empty(_cabi.workspace(query, *sizes), dtype=torch.uint8, device=device)
    return ws


def _raise_on_flags(who: str, flags: int, max_tracklets: int, what: str) -> None:
    """The sticky error word (the same bits for both trackers) as RuntimeError."""
    if flags & _cabi.IDOL_OVERFLOW:
        raise RuntimeError(f"{who}: more than max_tracklets={max_tracklets} live tracklets; the tracker "
                           "kept its state from before that frame and cannot continue")
    if flags & _cabi.IDOL_BAD_ROW:
        raise RuntimeError(f"{who}: a row index was outside the {what} given")


def temporal_weights(memory_len: int) -> torch.Tensor:
    """[memory_len, memory_len] fp32: row l - 1 holds the reference's ``torch.range(0.0, 1, 1/l)[1:]`` (its
    ``temporal_weight`` for a ring of l embeddings), computed by torch itself so that the bits are the reference's."""
    table = torch.zeros(memory_len, memory_len, dtype=torch.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                     # torch.range is deprecated
        for length in range(1, memory_len + 1):
            row = torch.range(0.0, 1, 1 / length)[1:]
            if row.numel() != length:
                raise ValueError(f"memory_len={memory_len}: torch.range(0, 1, 1/{length}) has {row.numel() + 1} "
                                 f"elements, not {length + 1}")
            table[length - 1, :length] = row
    return table


class IDOLTracker:
    """Drop-in for the reference's ``IDOL_Tracker`` with ``match_metric="bisoftmax"`` (the only metric its call site,
    ``uninext_vid.py:338-350``, uses; others raise ValueError).  Takes the reference's keyword arguments; those its
    ``match`` never reads (``obj_score_thr``, ``memo_backdrop_frames``, ``nms_conf_thr``, ``nms_backdrop_iou_thr``,
    ``nms_class_iou_thr``, ``with_cats``) are accepted and ignored.  Of a tracklet it keeps what ``match`` reads: the
    id, last frame, exist-frame count, EMA embedding and the rings of the last ``memory_len`` embeddings and scores, not
    the box, label, velocity, acc_frame or the backdrop list.

    ``max_tracklets`` (1..1024) bounds the live tracklets; a frame that would exceed it changes no state, and the next
    host read (``read`` or ``match``) raises RuntimeError, as does every later one: the tracker never drops a tracklet
    silently.  ``memory_len`` is 1..64, ``memo_tracklet_frames`` >= 1 and ``match_score_thr`` >= 0 (a tracklet is
    matched by one row at most).  Deliberate difference: exact ties of the matching score go to the lowest tracklet id.
    """

    def __init__(self, nms_thr_pre=0.7, nms_thr_post=0.3, init_score_thr=0.2, addnew_score_thr=0.5, obj_score_thr=0.1,
                 match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1, memo_momentum=0.5,
                 nms_conf_thr=0.5, nms_backdrop_iou_thr=0.5, nms_class_iou_thr=0.7, with_cats=True,
                 match_metric="bisoftmax", long_match=False, frame_weight=False, temporal_weight=False, memory_len=10,
                 *, max_tracklets: int = 1024, device="cuda"):
        if match_metric != "bisoftmax":
            raise ValueError(f"IDOLTracker: only match_metric='bisoftmax' is built, got {match_metric!r}")
        if not 0 <= memo_momentum <= 1:
            raise ValueError(f"IDOLTracker: memo_momentum must be in [0, 1], got {memo_momentum}")
        if not 1 <= int(memory_len) <= MAX_MEMORY:
            raise ValueError(f"IDOLTracker: memory_len must be in 1..{MAX_MEMORY}, got {memory_len}")
        if int(memo_tracklet_frames) < 1:
            raise ValueError(f"IDOLTracker: memo_tracklet_frames must be >= 1, got {memo_tracklet_frames}")
        if match_score_thr < 0:
            raise ValueError(f"IDOLTracker: match_score_thr must be >= 0, got {match_score_thr}")
        if not 1 <= int(max_tracklets) <= MAX_TRACKLETS:
            raise ValueError(f"IDOLTracker: max_tracklets must be in 1..{MAX_TRACKLETS}, got {max_tracklets}")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("IDOLTracker: Not implemented on the CPU")
        self.nms_thr_pre, self.nms_thr_post = float(nms_thr_pre), float(nms_thr_post)
        self.init_score_thr, self.addnew_score_thr = float(init_score_thr), float(addnew_score_thr)
        self.match_score_thr, self.memo_momentum = float(match_score_thr), float(memo_momentum)
        self.memo_tracklet_frames, self.memory_len = int(memo_tracklet_frames), int(memory_len)
        self.long_match, self.frame_weight, self.temporal_weight = bool(long_match), bool(frame_weight), bool(temporal_weight)
        self.max_tracklets = int(max_tracklets)
        self.flags = ((_cabi.IDOL_LONG_MATCH if self.long_match else 0) |
                      (_cabi.IDOL_FRAME_WEIGHT if self.frame_weight else 0) |
                      (_cabi.IDOL_TEMPORAL_WEIGHT if self.temporal_weight else 0))
        self._tw = temporal_weights(self.memory_len).to(self.device)
        T = self.max_tracklets
        self.state = torch.zeros(_STATE_HEADER + 5 * T, dtype=torch.int32, device=self.device)
        self.device = self.state.device                             # with its index
        self.dim = None
        self._ws = {}
        self._arange = {}

    # ---- state, as the tests read it ----------------------------------------------------------------------------------
    def tracklets(self) -> dict:
        """{id: dict(last_frame, exist_frame, embed, long_embed [len, D], long_score [len])} of the live tracklets, in
        ascending id order (a host read, for tests and debugging)."""
        T = self.max_tracklets
        st = self.state.cpu()
        live = int(st[0])
        order = st[_STATE_HEADER:_STATE_HEADER + T]
        out = {}
        for c in range(live):
            s = int(order[c])
            ln = int(st[_STATE_HEADER + 4 * T + s])
            out[int(st[_STATE_HEADER + T + s])] = dict(
                last_frame=int(st[_STATE_HEADER + 2 * T + s]), exist_frame=int(st[_STATE_HEADER + 3 * T + s]),
                embed=self.embed[s].cpu(), long_embed=self.ring_embed[s, :ln].cpu(), long_score=self.ring_score[s, :ln].cpu())
        return out

    @property
    def num_tracklets(self) -> int:
        """The next new id (the reference's ``num_tracklets``); a host read."""
        return int(self.state[1])

    # ---- the association ----------------------------------------------------------------------------------------------
    def _run(self, masks: torch.Tensor, embeds: torch.Tensor, scores: torch.Tensor, rows: torch.Tensor,
             count: torch.Tensor, frame_id: int) -> TrackResult:
        """masks [n_src, h, w] fp32, embeds [n_src, D] fp32, scores [n_cap] fp32, rows int32 [n_cap] into n_src,
        count int32 [1] on the device."""
        dev = self.device
        _check_devices("IDOLTracker", dev, masks=masks, embeds=embeds, scores=scores, rows=rows, count=count)
        n_src, h, w = masks.shape
        n_cap, D = rows.numel(), embeds.shape[1]
        if embeds.shape[0] != n_src or scores.numel() != n_cap:
            raise ValueError(f"IDOLTracker: {n_src} masks, {embeds.shape[0]} embeddings, {scores.numel()} scores and "
                             f"{n_cap} rows do not agree")
        if not 1 <= n_cap <= MAX_ROWS:
            raise ValueError(f"IDOLTracker: need 1..{MAX_ROWS} rows, got {n_cap}")
        if h * w >= 1 << 24:
            raise ValueError(f"IDOLTracker: masks of {h} x {w} pixels: need h * w < 2^24")
        if self.dim is None:
            T, L = self.max_tracklets, self.memory_len
            self.dim = D
            self.embed = torch.zeros(T, D, dtype=torch.float32, device=dev)
            self.ring_embed = torch.zeros(T, L, D, dtype=torch.float32, device=dev)
            self.ring_score = torch.zeros(T, L, dtype=torch.float32, device=dev)
        elif D != self.dim:
            raise ValueError(f"IDOLTracker: embeddings of {D} channels, the tracker holds {self.dim}")
        ws = _workspace(self._ws, (n_cap, h, w), "msda_idol_workspace", n_cap, self.max_tracklets, D, h, w, device=dev)
        out = TrackResult(torch.empty(n_cap, dtype=torch.int32, device=dev), torch.empty(n_cap, dtype=torch.int32, device=dev),
                          torch.empty(1, dtype=torch.int32, device=dev))
        _cabi.call("msda_idol_match_f32", masks.float().contiguous(), embeds.float().contiguous(),
                   scores.float().contiguous(), rows.to(torch.int32).contiguous(), count.to(torch.int32), n_src, n_cap,
                   h, w, D, self.nms_thr_pre, self.nms_thr_post, self.init_score_thr, self.addnew_score_thr,
                   self.match_score_thr, self.memo_momentum, self.memo_tracklet_frames, self.memory_len, self.flags,
                   self._tw, int(frame_id), self.max_tracklets, self.state, self.embed, self.ring_embed,
                   self.ring_score, out.ids, out.rows, out.count, ws, ws.numel(), device=dev)
        return out

    def match_selected(self, dets, b: int, pred_masks: torch.Tensor, pred_inst_embed: torch.Tensor,
                       frame_id: int) -> TrackResult:
        """Frame b of ``select_track_detections``' output (``dets``, with ``box_format="cxcywh"``): rows
        ``dets.query_index[b, :dets.count[b]]`` of ``pred_masks`` ([B, Q, 1, h, w] or [B, Q, h, w] stride-4 logits) and
        ``pred_inst_embed`` ([B, Q, D]), with the scores ``dets.scores[b]``.  The row count is read on the device and
        nothing synchronises with the host; ``read`` gives the tracked queries' rows and ids."""
        masks = pred_masks[b]
        if masks.dim() == 4:
            if masks.shape[1] != 1:
                raise ValueError(f"IDOLTracker: pred_masks must be [B, Q, 1, h, w] or [B, Q, h, w], got "
                                 f"{tuple(pred_masks.shape)}")
            masks = masks[:, 0]
        if masks.dim() != 3 or pred_inst_embed.dim() != 3:
            raise ValueError(f"IDOLTracker: need pred_masks [B, Q, (1,) h, w] and pred_inst_embed [B, Q, D], got "
                             f"{tuple(pred_masks.shape)} and {tuple(pred_inst_embed.shape)}")
        return self._run(masks, pred_inst_embed[b], dets.scores[b], dets.query_index[b], dets.count[b:b + 1], frame_id)

    def read(self, result: TrackResult) -> Tuple[List[int], List[int]]:
        """The one host read per frame: (rows, ids) of the tracked rows, in row order.  Raises RuntimeError when the
        tracker has overflowed ``max_tracklets`` or was given a row index outside its masks."""
        ids, rows, n = self._fetch(result)
        return rows, [int(ids[r]) for r in rows]

    def _fetch(self, result: TrackResult):
        host = torch.cat((result.ids, result.rows, result.count, self.state[_FLAGS:_FLAGS + 1])).cpu()
        _raise_on_flags("IDOLTracker", int(host[-1]), self.max_tracklets, "masks")
        n_cap = result.ids.numel()
        n = int(host[2 * n_cap])
        return host[:n_cap], host[n_cap:n_cap + n].tolist(), n

    def match(self, bboxes: torch.Tensor, labels: torch.Tensor, masks: torch.Tensor, track_feats: torch.Tensor,
              frame_id: int, indices):
        """The reference's ``match``: bboxes [n, 5] (the score last), labels [n], masks [n, 1, h, w] logits, track_feats
        [n, D], all CUDA; returns ``(bboxes[keep], labels[keep], ids, indices[keep])`` with ``ids`` a CPU int64 tensor
        and ``indices`` a list, after one host read."""
        n = bboxes.shape[0]
        if n == 0:
            raise ValueError("IDOLTracker.match: no detections (the caller always passes at least one)")
        if not (bboxes.is_cuda and masks.is_cuda and track_feats.is_cuda):
            raise RuntimeError("IDOLTracker: Not implemented on the CPU")
        if masks.dim() != 4 or masks.shape[:2] != (n, 1) or track_feats.shape[0] != n or len(indices) != n:
            raise ValueError(f"IDOLTracker.match: need masks [n, 1, h, w], track_feats [n, D] and n indices for "
                             f"n = {n}, got {tuple(masks.shape)}, {tuple(track_feats.shape)} and {len(indices)}")
        rows = self._arange.get(n)
        if rows is None:
            rows = self._arange[n] = torch.arange(n, dtype=torch.int32, device=self.device)
        count = torch.full((1,), n, dtype=torch.int32, device=self.device)
        res = self._run(masks[:, 0], track_feats, bboxes[:, -1], rows, count, frame_id)
        ids, _, _ = self._fetch(res)
        keep = [r for r in range(n) if int(ids[r]) != -3]
        keep_t = torch.tensor(keep, dtype=torch.long, device=bboxes.device)
        return (bboxes[keep_t], labels[keep_t.to(labels.device)], ids[keep].long(),
                [indices[r] for r in keep])


_QD_STATE_HEADER = 4                                                # MSDA_QD_STATE_INTS(T) = 4 + 4 T + 1024


class QuasiDenseTracker:
    """Drop-in for the reference's ``QuasiDenseEmbedTracker`` with ``match_metric="bisoftmax"`` and ``with_cats=True``,
    the settings of its one call site (``uninext_vid.py:323-336``, BDD ``box_track`` and ``seg_track_20``); the other
    metrics, ``with_cats=False`` and ``memo_backdrop_frames`` other than 0 or 1 raise ValueError.  Takes the reference's
    keyword arguments.  Of a tracklet it keeps what ``match`` reads: the id, last frame, label and embedding, not the box,
    velocity or acc_frame (``memo_bboxes`` and ``memo_vs`` are never used); of the backdrops, last frame's labels and
    embeddings.

    ``max_tracklets`` (1..1024) bounds the live tracklets; a frame that would exceed it changes no state, and the next
    host read (``read`` or ``match``) raises RuntimeError, as does every later one.  Frames hold at most 1024 rows,
    ``memo_tracklet_frames`` >= 1, ``memo_momentum`` is in [0, 1] and ``match_score_thr`` >= 0.  Deliberate differences:
    the rows are sorted by score with a stable sort (ties keep their row order), and exact ties of the matching score go
    to the lowest memo column.
    """

    def __init__(self, init_score_thr=0.8, obj_score_thr=0.5, match_score_thr=0.5, memo_tracklet_frames=10,
                 memo_backdrop_frames=1, memo_momentum=0.8, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3,
                 nms_class_iou_thr=0.7, with_cats=True, match_metric="bisoftmax", *, max_tracklets: int = 1024,
                 device="cuda"):
        if match_metric != "bisoftmax":
            raise ValueError(f"QuasiDenseTracker: only match_metric='bisoftmax' is built, got {match_metric!r}")
        if not with_cats:
            raise ValueError("QuasiDenseTracker: only with_cats=True is built")
        if memo_backdrop_frames not in (0, 1):
            raise ValueError(f"QuasiDenseTracker: memo_backdrop_frames must be 0 or 1, got {memo_backdrop_frames}")
        if not 0 <= memo_momentum <= 1:
            raise ValueError(f"QuasiDenseTracker: memo_momentum must be in [0, 1], got {memo_momentum}")
        if int(memo_tracklet_frames) < 1:
            raise ValueError(f"QuasiDenseTracker: memo_tracklet_frames must be >= 1, got {memo_tracklet_frames}")
        if match_score_thr < 0:
            raise ValueError(f"QuasiDenseTracker: match_score_thr must be >= 0, got {match_score_thr}")
        if not 1 <= int(max_tracklets) <= MAX_TRACKLETS:
            raise ValueError(f"QuasiDenseTracker: max_tracklets must be in 1..{MAX_TRACKLETS}, got {max_tracklets}")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("QuasiDenseTracker: Not implemented on the CPU")
        self.init_score_thr, self.obj_score_thr = float(init_score_thr), float(obj_score_thr)
        self.match_score_thr, self.memo_momentum = float(match_score_thr), float(memo_momentum)
        self.nms_conf_thr, self.nms_backdrop_iou_thr = float(nms_conf_thr), float(nms_backdrop_iou_thr)
        self.nms_class_iou_thr = float(nms_class_iou_thr)
        self.memo_tracklet_frames, self.memo_backdrop_frames = int(memo_tracklet_frames), int(memo_backdrop_frames)
        self.max_tracklets = int(max_tracklets)
        self.flags = _cabi.QD_BACKDROPS if self.memo_backdrop_frames else 0
        T = self.max_tracklets
        self.state = torch.zeros(_QD_STATE_HEADER + 4 * T + _cabi.QD_MAX_BACKDROPS, dtype=torch.int32,
                                 device=self.device)
        self.device = self.state.device                             # with its index
        self.dim = None
        self._ws = {}
        self._arange = {}

    # ---- state, as the tests read it ----------------------------------------------------------------------------------
    def tracklets(self) -> dict:
        """{id: dict(last_frame, label, embed)} of the live tracklets in ascending id order (a host read)."""
        T, h = self.max_tracklets, _QD_STATE_HEADER
        st = self.state.cpu()
        out = {}
        for c in range(int(st[0])):
            s = int(st[h + c])
            out[int(st[h + T + s])] = dict(last_frame=int(st[h + 2 * T + s]), label=int(st[h + 3 * T + s]),
                                           embed=self.embed[s].cpu())
        return out

    def backdrops(self) -> dict:
        """Last frame's backdrops, dict(labels [m] int64, embeds [m, D]), in their row order (a host read)."""
        st = self.state.cpu()
        m, base = int(st[3]), _QD_STATE_HEADER + 4 * self.max_tracklets
        embeds = self.backdrop_embed[:m].cpu() if self.dim is not None else torch.zeros(0, 0)
        return dict(labels=st[base:base + m].long(), embeds=embeds)

    @property
    def num_tracklets(self) -> int:
        """The next new id (the reference's ``num_tracklets``); a host read."""
        return int(self.state[1])

    # ---- the association ----------------------------------------------------------------------------------------------
    def _run(self, boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, embeds: torch.Tensor,
             rows: torch.Tensor, count: torch.Tensor, frame_id: int) -> TrackResult:
        """boxes [n_cap, 4] xyxy, scores [n_cap], labels [n_cap], rows int32 [n_cap] into embeds [n_src, D], count int32
        [1], all on the device."""
        dev = self.device
        _check_devices("QuasiDenseTracker", dev, boxes=boxes, scores=scores, labels=labels, embeds=embeds, rows=rows,
                       count=count)
        n_cap = rows.numel()
        n_src, D = embeds.shape
        if boxes.shape != (n_cap, 4) or scores.numel() != n_cap or labels.numel() != n_cap:
            raise ValueError(f"QuasiDenseTracker: {tuple(boxes.shape)} boxes, {scores.numel()} scores, "
                             f"{labels.numel()} labels and {n_cap} rows do not agree")
        if not 1 <= n_cap <= MAX_ROWS:
            raise ValueError(f"QuasiDenseTracker: need 1..{MAX_ROWS} rows, got {n_cap}")
        if self.dim is None:
            self.dim = D
            self.embed = torch.zeros(self.max_tracklets, D, dtype=torch.float32, device=dev)
            self.backdrop_embed = torch.zeros(_cabi.QD_MAX_BACKDROPS, D, dtype=torch.float32, device=dev)
        elif D != self.dim:
            raise ValueError(f"QuasiDenseTracker: embeddings of {D} channels, the tracker holds {self.dim}")
        ws = _workspace(self._ws, n_cap, "msda_qdtrack_workspace", n_cap, self.max_tracklets, D, device=dev)
        out = TrackResult(*(torch.empty(n, dtype=torch.int32, device=dev) for n in (n_cap, n_cap, 1, n_cap)))
        _cabi.call("msda_qdtrack_match_f32", boxes.float().contiguous(), scores.float().contiguous(),
                   labels.to(torch.int32).contiguous(), embeds.float().contiguous(), rows.to(torch.int32).contiguous(),
                   count.to(torch.int32), n_src, n_cap, D, self.init_score_thr, self.obj_score_thr,
                   self.match_score_thr, self.nms_conf_thr, self.nms_backdrop_iou_thr, self.nms_class_iou_thr,
                   self.memo_momentum, self.memo_tracklet_frames, self.flags, int(frame_id), self.max_tracklets,
                   self.state, self.embed, self.backdrop_embed, out.order, out.ids, out.rows, out.count, ws,
                   ws.numel(), device=dev)
        return out

    def match_selected(self, dets, b: int, pred_inst_embed: torch.Tensor, frame_id: int) -> TrackResult:
        """Frame b of ``select_track_detections``' output (``dets``, with ``box_format="xyxy_pixels"``): its boxes,
        scores and labels in keep order, and rows ``dets.query_index[b, :dets.count[b]]`` of ``pred_inst_embed``
        ([B, Q, D]).  The row count is read on the device and nothing synchronises with the host; ``read`` gives the
        tracked rows of ``dets`` and their ids."""
        if pred_inst_embed.dim() != 3:
            raise ValueError(f"QuasiDenseTracker: need pred_inst_embed [B, Q, D], got {tuple(pred_inst_embed.shape)}")
        return self._run(dets.boxes[b], dets.scores[b], dets.labels[b], pred_inst_embed[b], dets.query_index[b],
                         dets.count[b:b + 1], frame_id)

    def _fetch(self, result: TrackResult):
        host = torch.cat((result.ids, result.order, result.rows, result.count, self.state[2:3])).cpu()
        _raise_on_flags("QuasiDenseTracker", int(host[-1]), self.max_tracklets, "embeddings")
        n_cap = result.ids.numel()
        return host[:n_cap], host[n_cap:2 * n_cap], host[2 * n_cap:2 * n_cap + int(host[3 * n_cap])].tolist()

    def read(self, result: TrackResult) -> Tuple[List[int], List[int]]:
        """The one host read per frame: (rows, ids) of the tracked rows, in score order.  Raises RuntimeError when the
        tracker has overflowed ``max_tracklets`` or was given a row index outside its embeddings."""
        ids, _, rows = self._fetch(result)
        return rows, [int(i) for i in ids if i >= 0]

    def match(self, bboxes: torch.Tensor, labels: torch.Tensor, track_feats: torch.Tensor, frame_id: int, indices):
        """The reference's ``match``: bboxes [n, 5] (xyxy, then the score), labels [n], track_feats [n, D], all CUDA;
        returns ``(bboxes, labels, ids, indices)`` of the kept rows in score order, with ``ids`` a CPU int64 tensor,
        after one host read.  As in the reference, ``indices`` is the caller's list filtered by the kept positions of
        the sorted rows, not reordered: the two agree when the rows come in score order, as they do from
        ``select_track_detections``."""
        n = bboxes.shape[0]
        if n == 0:
            raise ValueError("QuasiDenseTracker.match: no detections (the caller always passes at least one)")
        if not (bboxes.is_cuda and labels.is_cuda and track_feats.is_cuda):
            raise RuntimeError("QuasiDenseTracker: Not implemented on the CPU")
        if bboxes.dim() != 2 or bboxes.shape[1] != 5 or labels.numel() != n or track_feats.shape[0] != n or \
                len(indices) != n:
            raise ValueError(f"QuasiDenseTracker.match: need bboxes [n, 5], labels [n], track_feats [n, D] and n "
                             f"indices for n = {n}, got {tuple(bboxes.shape)}, {tuple(labels.shape)}, "
                             f"{tuple(track_feats.shape)} and {len(indices)}")
        rows = self._arange.get(n)
        if rows is None:
            rows = self._arange[n] = torch.arange(n, dtype=torch.int32, device=self.device)
        count = torch.full((1,), n, dtype=torch.int32, device=self.device)
        res = self._run(bboxes[:, :4], bboxes[:, 4], labels, track_feats, rows, count, frame_id)
        ids, order, _ = self._fetch(res)
        keep = [p for p in range(n) if int(ids[p]) != -3]
        src = torch.tensor([int(order[p]) for p in keep], dtype=torch.long, device=bboxes.device)
        return bboxes[src], labels[src], ids[keep].long(), [indices[p] for p in keep]
