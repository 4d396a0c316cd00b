"""Shared by tests/test_tracker_host.py, tests/test_gpu_tracker.py, tests/golden/make_tracker_golden.py and
tools/tracker_bench.py: seeded multi-frame VIS sequences for the IDOL tracker, and a restatement of its association step
written from DESIGN.md section 3.18's semantics (not from the reference's code) that runs with torch on any device.

Masks are built from disjoint random pixel sets, one per object, so that every IoU is far from the thresholds: a
detection of an object covers 92 % of its set or more (IoU >= 0.92 with another such detection: a duplicate), a partial
covers 25 % (IoU about 0.25: kept by the NMS, not a backdrop), and detections of different objects do not overlap
(IoU 1e-6 / (union + 1e-6)).  Scores sit on a grid of 1/1000 + 1/2000, away from every score threshold.
"""
import hashlib
import warnings

import numpy as np
import torch

# The reference's settings for VIS (config.py:130-133, uninext_vid.py:338-350).
VIS_SETTINGS = dict(nms_thr_pre=0.5, nms_thr_post=0.05, init_score_thr=0.2, addnew_score_thr=0.2, obj_score_thr=0.1,
                    match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1, memo_momentum=0.8,
                    nms_conf_thr=0.5, nms_backdrop_iou_thr=0.5, nms_class_iou_thr=0.7, with_cats=True,
                    match_metric="bisoftmax", memory_len=3)
# (long_match, frame_weight, temporal_weight): the three the call site can produce, and (T, F, F).
FLAG_SETS = [(True, True, True), (False, True, False), (False, False, False), (True, False, False)]


def settings(flags, **over):
    lm, fw, tw = flags
    return dict(VIS_SETTINGS, long_match=lm, frame_weight=fw, temporal_weight=tw, **over)


# ---- the restatement ------------------------------------------------------------------------------------------------
def binarise(masks):
    """[n, h, w] logits -> bool, as the reference binarises (sigmoid > 0.5 on the tensor's device)."""
    return masks.sigmoid() > 0.5


def iou_matrix(bits):
    """[n, h, w] bool -> (iou [n, n] fp32 from int64 counts, iou64 [n, n] float64)."""
    b = bits.reshape(bits.shape[0], -1).double()
    inter = torch.round(b @ b.t()).long()                 # exact: counts < 2^24
    size = bits.reshape(bits.shape[0], -1).sum(1)
    union = size[:, None] + size[None, :] - inter
    iou = (inter.float() + 1e-6) / (union.float() + 1e-6)
    iou64 = (inter.double() + 1e-6) / (union.double() + 1e-6)
    return iou.cpu().numpy(), iou64.cpu().numpy()


class Restated:
    """The association step of DESIGN.md section 3.18 with the tracklets in a dict.  ``margins`` collects, in float64,
    each decision's distance from flipping."""

    def __init__(self, nms_thr_pre, nms_thr_post, init_score_thr, addnew_score_thr, match_score_thr,
                 memo_tracklet_frames, memo_momentum, long_match, frame_weight, temporal_weight, memory_len, **_ignored):
        f32 = np.float32
        self.pre, self.post = f32(nms_thr_pre), f32(nms_thr_post)
        self.init_thr, self.new_thr, self.match_thr = f32(init_score_thr), f32(addnew_score_thr), f32(match_score_thr)
        self.frames, self.m = memo_tracklet_frames, memo_momentum
        self.long_match, self.frame_weight, self.temporal_weight = long_match, frame_weight, temporal_weight
        self.L = memory_len
        self.tracks = {}
        self.next_id = 0
        self.margins = []
        self.weighted_rows = 0                 # rows that took the frame-weight branch
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            self.tw = {l: torch.range(0.0, 1, 1 / l)[1:] for l in range(1, memory_len + 1)}

    def _memo(self, device):
        rows = []
        for tid in sorted(self.tracks):
            v = self.tracks[tid]
            if self.long_match:
                w = torch.stack(v["long_score"])
                if self.temporal_weight:
                    w = w + self.tw[len(w)]
                e = torch.stack(v["long_embed"])
                rows.append((e * w[:, None]).sum(0) / w.sum())
            else:
                rows.append(v["embed"])
        return torch.stack(rows).to(device)

    def step(self, scores, masks, embeds, frame_id):
        """scores [n] fp32 (any device), masks [n, h, w] logits, embeds [n, D] -> (keep rows, ids of the kept rows)."""
        n = scores.shape[0]
        dev = embeds.device
        iou, iou64 = iou_matrix(binarise(masks))
        for thr in (self.pre, self.post):
            off = np.abs(iou64 - float(thr))[np.triu_indices(n, 1)]
            self.margins.append(off.min() if off.size else 1.0)
        keep = []
        for j in range(n):
            if not any(iou[i, j] > self.pre for i in keep):
                keep.append(j)
        sc = scores.detach().cpu().numpy().astype(np.float32)[keep]
        e = embeds[keep].float()
        ids = [-2] * len(keep)
        empty = not self.tracks
        if not empty:
            cols = sorted(self.tracks)
            memo = self._memo(dev)
            feats = e @ memo.t()
            s_all = ((feats.softmax(1) + feats.softmax(0)) / 2).cpu().numpy()
            f64 = e.double() @ memo.double().t()
            s64_all = ((f64.softmax(1) + f64.softmax(0)) / 2).cpu().numpy()
            ef = np.array([self.tracks[c]["exist_frame"] for c in cols], np.float32)
            taken = np.zeros(len(cols), bool)
            for i in range(len(keep)):
                s = np.where(taken, np.float32(0), s_all[i]).astype(np.float32)
                s64 = np.where(taken, 0.0, s64_all[i])
                p = s > np.float32(0.5)
                if self.frame_weight:
                    self.margins.append(np.abs(s64[~taken] - 0.5).min() if (~taken).any() else 1.0)
                if self.frame_weight and p.sum() > 1:
                    self.weighted_rows += 1
                    mean = np.float32(ef[p].sum()) / np.float32(p.sum())
                    w = np.where(p, s * ef, s * mean).astype(np.float32)
                    w64 = np.where(p, s64 * ef, s64 * float(ef[p].mean()))
                else:
                    w, w64 = s, s64
                j = int(np.argmax(w))
                self.margins.append(abs(w64[j] - float(self.match_thr)))
                if w[j] > self.match_thr:
                    if len(w64) > 1:
                        self.margins.append(w64[j] - np.delete(w64, j).max())
                    ids[i] = cols[j]
                    taken[j] = True
        thr = self.init_thr if empty else self.new_thr
        for i in range(len(keep)):
            self.margins.append(abs(float(sc[i]) - float(thr)))
            if ids[i] == -2 and sc[i] > thr:
                ids[i] = self.next_id
                self.next_id += 1
        for i in range(len(keep)):
            if ids[i] == -2 and all(iou[keep[a], keep[i]] < self.post for a in range(i)):
                ids[i] = -1
        self._update(ids, keep, e, torch.from_numpy(sc), frame_id)
        return keep, ids

    def _update(self, ids, keep, e, sc, frame_id):
        for i, tid in enumerate(ids):
            if tid < 0:
                continue
            x, s = e[i].cpu(), sc[i]
            v = self.tracks.get(tid)
            if v is None:
                self.tracks[tid] = dict(embed=x, long_embed=[x], long_score=[s], last_frame=frame_id, exist_frame=1)
            else:
                v["embed"] = (1 - self.m) * v["embed"] + self.m * x
                v["long_embed"] = (v["long_embed"] + [x])[-self.L:]
                v["long_score"] = (v["long_score"] + [s])[-self.L:]
                v["last_frame"] = frame_id
                v["exist_frame"] += 1
        for tid in [t for t, v in self.tracks.items() if frame_id - v["last_frame"] >= self.frames]:
            del self.tracks[tid]


# ---- sequences ------------------------------------------------------------------------------------------------------
class World:
    """Objects with a disjoint pixel set and a base embedding each; a frame lists (object, kind, score) detections,
    kind "full", "dup" (a near copy, after its object's row), "part" (a 25 % piece with an unrelated embedding),
    "weak" (the object's pixels with a zero embedding: every tracklet scores (1/T + 1/3) / 2 for it when the frame has
    three such rows), "merge" (object a's pixels with an embedding between objects a and b)."""

    def __init__(self, num_objects, h, w, dim, seed, scale=24.0):
        self.g = np.random.default_rng(seed)
        self.h, self.w, self.dim = h, w, dim
        owner = self.g.integers(0, num_objects + 1, size=h * w)          # num_objects: background
        self.pixels = [np.flatnonzero(owner == k) for k in range(num_objects)]
        base = self.g.standard_normal((num_objects, dim))
        self.base = base / np.linalg.norm(base, axis=1, keepdims=True) * np.sqrt(scale)

    def frame(self, dets):
        """dets: [(obj, kind, score, other)] in row order -> (scores [n] fp32, masks [n, 1, h, w] fp32, embeds [n, D])."""
        g, n = self.g, len(dets)
        masks = -(1.0 + 3.0 * g.random((n, self.h * self.w)))
        embeds = np.zeros((n, self.dim))
        for r, (obj, kind, score, other) in enumerate(dets):
            px = self.pixels[obj]
            if kind == "dup":
                px = px[g.random(px.size) < 0.96]
            elif kind == "part":
                px = px[: max(1, px.size // 4)]
            masks[r, px] = 1.0 + 3.0 * g.random(px.size)
            if kind == "weak":
                pass
            elif kind == "part":
                v = g.standard_normal(self.dim)
                embeds[r] = v / np.linalg.norm(v) * np.sqrt(24.0) * 0.3
            elif kind == "merge":
                embeds[r] = 0.62 * self.base[obj] + 0.38 * self.base[other]
            else:
                embeds[r] = self.base[obj] + 0.05 * g.standard_normal(self.dim)
        scores = np.array([d[2] for d in dets], np.float32)
        return (torch.from_numpy(scores), torch.from_numpy(masks.astype(np.float32)).reshape(n, 1, self.h, self.w),
                torch.from_numpy(embeds.astype(np.float32)))


def _score(g, lo, hi):
    """A score in (lo, hi) on the grid k / 1000 + 1 / 2000."""
    return float(np.floor(g.uniform(lo, hi) * 1000) / 1000 + 0.0005)


def golden_sequence(seed, h=40, w=72, dim=32, frames=18):
    """[(scores, masks, embeds)] for `frames` frames, n <= 48 rows each: frames 0-4 track objects that come and stay,
    with duplicates, a partial detection (left at -2) and a low-score row (a backdrop); in frames 3 and 4 two objects
    are absent and one row resembles both; frames 5-14 hold only three weak low-score rows, so every tracklet expires
    after 10 absent frames; frame 15 starts afresh with new objects."""
    world = World(40, h, w, dim, seed)
    g = world.g
    out = []
    for f in range(frames):
        dets = []
        if f < 5:
            dets = [[o, "full", _score(g, 0.55, 0.95), None] for o in range(8 + f)]
            dets.append([36, "full", _score(g, 0.05, 0.15), None])       # low score: a backdrop
            dets.append([1, "dup", _score(g, 0.3, 0.5), None])
            dets.append([2, "part", _score(g, 0.06, 0.18), None])        # overlaps object 2: stays at -2
            if f in (3, 4):                                             # objects 4 and 5 absent; a row like both
                dets = [d for d in dets if d[0] not in (4, 5)]
                dets.append([4, "merge", _score(g, 0.6, 0.9), 5] if f == 3 else [5, "merge", _score(g, 0.6, 0.9), 4])
        elif f < 15:
            dets = [[30 + i, "weak", _score(g, 0.02, 0.15), None] for i in range(3)]
        else:
            dets = [[o, "full", _score(g, 0.55, 0.95), None] for o in range(16, 24)]
            dets.append([37, "full", _score(g, 0.05, 0.15), None])
        order = sorted(range(len(dets)), key=lambda i: -dets[i][2])
        out.append(world.frame([tuple(dets[i]) for i in order]))
    return out


def random_sequence(seed, n, h, w, dim=64, frames=4):
    """Large frames for the GPU tests: about n rows over n * 3 / 4 objects, with duplicates and partials."""
    objects = max(2, (3 * n) // 4)
    world = World(objects + 8, h, w, dim, seed)
    g = world.g
    out = []
    for f in range(frames):
        present = np.flatnonzero(g.random(objects) < 0.85)
        dets = [(int(o), "full", _score(g, 0.05, 0.95), None) for o in present]
        extra = n - len(dets)
        for o in g.choice(present, size=max(0, min(extra, len(present))), replace=False):
            dets.append((int(o), "dup" if g.random() < 0.5 else "part", _score(g, 0.01, 0.2), None))
        dets = dets[:n]
        order = sorted(range(len(dets)), key=lambda i: -dets[i][2])
        out.append(world.frame([dets[i] for i in order]))
    return out


def checksum(seq):
    """sha256 of a sequence's bytes: pins the generator's output."""
    h = hashlib.sha256()
    for frame in seq:
        for t in frame:
            h.update(t.numpy().tobytes())
    return h.hexdigest()[:16]


# ---- the reference's chain, for timing --------------------------------------------------------------------------------
def _pair_iou(a, b):
    """IoU of two [.., h, w] bool masks as int8 products summed (models/tracker.py:17-24's arithmetic)."""
    a, b = a.char(), b.char()
    inter = (a * b).sum(-1).sum(-1)
    union = (a + b - a * b).sum(-1).sum(-1)
    return (inter + 1e-6) / (union + 1e-6)


class ReferenceChain(Restated):
    """The reference's host-driven structure on the tensors' device, for tools/tracker_bench.py: the mask NMS as a pair
    loop with one host read per pair, the matching loop with host reads per row, the backdrop loop with one per
    unassigned row, the memo stacked from per-tracklet lists every frame (with a host-made temporal weight copied to
    the device per tracklet) and the memory updated id by id.  Its ids are Restated's; masks are [n, 1, h, w] here."""

    def step(self, scores, masks, embeds, frame_id):
        dev = masks.device
        n = masks.shape[0]
        seg = masks.sigmoid() > 0.5
        keep = [True] * n
        for i in range(n - 1):
            if not keep[i]:
                continue
            for j in range(i + 1, n):
                if keep[j] and _pair_iou(seg[i], seg[j]) > float(self.pre):
                    keep[j] = False
        rows = [r for r in range(n) if keep[r]]
        sc, e, m = scores[rows], embeds[rows], masks[rows]
        ids = torch.full((len(rows),), -2, dtype=torch.long)
        empty = not self.tracks
        if not empty:
            cols = sorted(self.tracks)
            memo = []
            for k in cols:
                v = self.tracks[k]
                if self.long_match:
                    w = torch.stack(v["long_score"])
                    if self.temporal_weight:
                        w = w + self.tw[len(w)].to(w)
                    memo.append(((torch.stack(v["long_embed"]) * w.unsqueeze(1)).sum(0) / w.sum())[None])
                else:
                    memo.append(v["embed"][None])
            memo = torch.cat(memo)
            ef = torch.tensor([self.tracks[k]["exist_frame"] for k in cols], dtype=torch.long).to(memo)
            cid = torch.tensor(cols, dtype=torch.long).to(memo)
            feats = torch.mm(e, memo.t())
            s = (feats.softmax(dim=1) + feats.softmax(dim=0)) / 2
            for i in range(len(rows)):
                if self.frame_weight:
                    p = (cid > -1) & (s[i, :] > 0.5)
                    if (s[i, p] > 0.5).sum() > 1:
                        ws = s.clone()
                        fw = ef[s[i, :][cid > -1] > 0.5]
                        ws[i, p] = ws[i, p] * fw
                        ws[i, ~p] = ws[i, ~p] * fw.mean()
                        conf, j = torch.max(ws[i, :], dim=0)
                    else:
                        conf, j = torch.max(s[i, :], dim=0)
                else:
                    conf, j = torch.max(s[i, :], dim=0)
                if conf > float(self.match_thr):
                    ids[i] = int(cid[j])
                    s[:i, j] = 0
                    s[i + 1:, j] = 0
        thr = float(self.init_thr if empty else self.new_thr)
        new = (ids == -2) & (sc > thr).cpu()
        k = int(new.sum())
        ids[new] = torch.arange(self.next_id, self.next_id + k)
        self.next_id += k
        left = torch.nonzero(ids == -2, as_tuple=False).squeeze(1)
        ious = _pair_iou(m[left].sigmoid() > 0.5, m.permute(1, 0, 2, 3).sigmoid() > 0.5)
        for a, r in enumerate(left):
            if (ious[a, :r] < float(self.post)).all():
                ids[r] = -1
        for a, tid in enumerate(ids.tolist()):
            if tid < 0:
                continue
            v = self.tracks.get(tid)
            if v is None:
                self.tracks[tid] = dict(embed=e[a], long_embed=[e[a]], long_score=[sc[a]], last_frame=frame_id,
                                        exist_frame=1)
            else:
                v["embed"] = (1 - self.m) * v["embed"] + self.m * e[a]
                v["long_embed"] = (v["long_embed"] + [e[a]])[-self.L:]
                v["long_score"] = (v["long_score"] + [sc[a]])[-self.L:]
                v["last_frame"] = frame_id
                v["exist_frame"] += 1
        for tid in [t for t, v in self.tracks.items() if frame_id - v["last_frame"] >= self.frames]:
            del self.tracks[tid]
        return rows, ids.tolist()
