"""Shared by tests/test_qdtrack_host.py, tests/test_gpu_qdtrack.py, tests/golden/make_qdtrack_golden.py and
tools/qdtrack_bench.py: seeded multi-frame BDD-like sequences for the QuasiDense tracker, a restatement of its
association step written from DESIGN.md section 3.19's semantics (not from the reference's code) that runs with torch on
any device, and a restatement of the reference's host-driven structure for timing.

Objects sit in the cells of a grid, so boxes of different objects never overlap; duplicates are shifted copies whose IoU
with their object's box is set by the shift ((w - dx) / (w + dx)), far from the thresholds.  Embeddings are unit vectors
times sqrt(scale): a detection of an object carries its object's vector plus a little noise.  Scores sit on a grid of
1/1000 + 1/2000, away from every score threshold.
"""
import hashlib

import numpy as np
import torch

# The reference's BDD call site (uninext_vid.py:323-336, with its config's init / obj score thresholds), the
# constructor's defaults (models/tracker.py:306-317), and the call site without backdrops.
BDD = dict(init_score_thr=0.5, obj_score_thr=0.3, match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1,
           memo_momentum=1.0, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3, nms_class_iou_thr=0.7, with_cats=True,
           match_metric="bisoftmax")
DEFAULTS = dict(init_score_thr=0.8, obj_score_thr=0.5, match_score_thr=0.5, memo_tracklet_frames=10,
                memo_backdrop_frames=1, memo_momentum=0.8, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3,
                nms_class_iou_thr=0.7, with_cats=True, match_metric="bisoftmax")
SETTINGS = {"bdd": BDD, "defaults": DEFAULTS, "bdd_nobackdrop": dict(BDD, memo_backdrop_frames=0)}
NUM_CLASSES, DIM = 8, 256


# ---- the restatement ------------------------------------------------------------------------------------------------
def box_iou(a, b):
    """mmcv's bbox_overlaps (mode "iou") of xyxy boxes a [m, 4] and b [n, 4], one torch operation at a time in the
    tensors' dtype: the union clamped at 1e-6 before the division."""
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:], b[None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = area_a[:, None] + area_b[None, :] - overlap
    return overlap / torch.max(union, union.new_tensor([1e-6]))


class Restated:
    """The association step of DESIGN.md section 3.19 with the tracklets in a dict.  ``margins`` collects, in float64,
    each decision's distance from flipping; ``seen`` the branches taken."""

    def __init__(self, init_score_thr, obj_score_thr, match_score_thr, memo_tracklet_frames, memo_backdrop_frames,
                 memo_momentum, nms_conf_thr, nms_backdrop_iou_thr, nms_class_iou_thr, **_ignored):
        f32 = np.float32
        self.init_thr, self.obj_thr, self.match_thr = f32(init_score_thr), f32(obj_score_thr), f32(match_score_thr)
        self.conf_thr, self.back_iou, self.class_iou = f32(nms_conf_thr), f32(nms_backdrop_iou_thr), f32(nms_class_iou_thr)
        self.frames, self.backdrop_frames, self.m = memo_tracklet_frames, memo_backdrop_frames, memo_momentum
        self.tracks = {}                       # id -> dict(embed, label, last_frame)
        self.backdrops = None                  # (labels [m], embeds [m, D]) of last frame, or None
        self.next_id = 0
        self.margins = []
        self.seen = set()

    def _margin(self, value64, thr):
        self.margins.append(abs(float(value64) - float(thr)))

    def step(self, boxes, scores, labels, embeds, frame_id):
        """boxes [n, 4] xyxy fp32, scores [n] fp32, labels [n] int, embeds [n, D] (all on one device) -> (order: the
        input row at each sorted position, keep: the kept sorted positions, ids of the kept rows)."""
        n = scores.shape[0]
        order = torch.sort(scores, descending=True, stable=True).indices
        b, sc, lab, e = boxes[order].float(), scores[order].float(), labels[order], embeds[order].float()
        iou = box_iou(b, b).cpu().numpy()
        iou64 = box_iou(b.double(), b.double()).cpu().numpy()
        s_np = sc.cpu().numpy()
        for thr in (self.obj_thr, self.init_thr):
            self.margins.append(np.abs(s_np.astype(np.float64) - float(thr)).min())
        pairs = iou64[np.triu_indices(n, 1)]
        for thr in (self.back_iou, self.class_iou):
            if pairs.size:
                self.margins.append(np.abs(pairs - float(thr)).min())
        # duplicate removal: any earlier row, removed or not
        keep = []
        for j in range(n):
            thr = self.back_iou if s_np[j] < self.obj_thr else self.class_iou
            if (iou[:j, j] > thr).any():
                self.seen.add("dup_class" if thr == self.class_iou else "dup_backdrop")
                if not any(iou[i, j] > thr for i in keep):
                    self.seen.add("dup_via_removed")
            else:
                keep.append(j)
        k = len(keep)
        kb, ks, kl, ke = b[keep], s_np[keep], lab[keep], e[keep]
        ids = [-1] * k
        if self.tracks:
            tids = sorted(self.tracks)
            memo_e = [self.tracks[t]["embed"].to(e.device) for t in tids]
            memo_l = [self.tracks[t]["label"] for t in tids]
            col_ids = list(tids)
            if self.backdrops is not None:
                memo_e += list(self.backdrops[1].to(e.device))
                memo_l += self.backdrops[0].tolist()
                col_ids += [-1] * len(self.backdrops[0])
            memo = torch.stack(memo_e)
            same = (kl.view(-1, 1).cpu() == torch.tensor(memo_l).view(1, -1))
            feats = ke @ memo.t()
            s_raw = ((feats.softmax(1) + feats.softmax(0)) / 2).cpu().numpy()
            s_all = ((feats.softmax(1) + feats.softmax(0)) / 2 * same.to(feats).to(feats.device)).cpu().numpy()
            f64 = ke.double() @ memo.double().t()
            s64_all = ((f64.softmax(1) + f64.softmax(0)) / 2).cpu().numpy() * same.numpy()
            if not same.all():
                self.seen.add("category_mask")
            taken = np.zeros(len(col_ids), bool)
            for i in range(k):
                s = np.where(taken, np.float32(0), s_all[i]).astype(np.float32)
                s64 = np.where(taken, 0.0, s64_all[i])
                c = int(np.argmax(s))
                self._margin(s64[c], self.match_thr)
                if s[c] > self.match_thr:
                    if len(s64) > 1:
                        self.margins.append(s64[c] - np.delete(s64, c).max())
                    if int(np.argmax(np.where(taken, 0, s_raw[i]))) != c:
                        self.seen.add("category_decides")
                    if col_ids[c] < 0:
                        self.seen.add("best_is_backdrop")
                    elif ks[i] > self.obj_thr:
                        ids[i] = col_ids[c]
                        taken[c] = True
                    else:
                        self._margin(s64[c], self.conf_thr)
                        if s[c] > self.conf_thr:
                            ids[i] = -2
                            self.seen.add("suppressed")
        for i in range(k):
            if ids[i] == -1 and ks[i] > self.init_thr:
                ids[i] = self.next_id
                self.next_id += 1
                self.seen.add("new")
        if any(i == -1 for i in ids):
            self.seen.add("left")
        kiou = iou[np.ix_(keep, keep)]
        back = [i for i in range(k) if ids[i] == -1 and not (kiou[:i, i] > self.back_iou).any()]
        self._update(ids, kl.cpu(), ke.cpu(), back, frame_id)
        return order.cpu().tolist(), keep, ids

    def _update(self, ids, labels, embeds, back, frame_id):
        for i, tid in enumerate(ids):
            if tid < 0:
                continue
            v = self.tracks.get(tid)
            if v is None:
                self.tracks[tid] = dict(embed=embeds[i], label=int(labels[i]), last_frame=frame_id)
            else:
                v["embed"] = (1 - self.m) * v["embed"] + self.m * embeds[i]
                v["label"] = int(labels[i])
                v["last_frame"] = frame_id
        self.backdrops = (labels[back].long(), embeds[back]) if self.backdrop_frames else None
        for tid in [t for t, v in self.tracks.items() if frame_id - v["last_frame"] >= self.frames]:
            del self.tracks[tid]
        if not self.tracks:
            self.seen.add("empty")


# ---- sequences ------------------------------------------------------------------------------------------------------
def _score(g, lo, hi):
    """A score in (lo, hi) on the grid k / 1000 + 1 / 2000."""
    return float(np.floor(g.uniform(lo, hi) * 1000) / 1000 + 0.0005)


class World:
    """Objects in the cells of a grid (cell 100 x 100 px, box about 60 x 60 inside it), each with a class and a base
    embedding of norm sqrt(scale)."""

    def __init__(self, num_objects, dim, seed, scale=24.0, cols=32):
        self.g = np.random.default_rng(seed)
        self.dim, self.cols, self.scale = dim, cols, scale
        base = self.g.standard_normal((num_objects, dim))
        self.base = base / np.linalg.norm(base, axis=1, keepdims=True) * np.sqrt(scale)
        self.label = self.g.integers(0, NUM_CLASSES, size=num_objects)

    def box(self, cell, shift=0.0):
        """The box of grid cell `cell`, jittered by whole pixels, moved right by `shift` of its width."""
        g = self.g
        x0, y0 = (cell % self.cols) * 100.0 + 20 + g.integers(0, 4), (cell // self.cols) * 100.0 + 20 + g.integers(0, 4)
        w = 60.0
        return [x0 + shift * w, y0, x0 + shift * w + w, y0 + w]

    def vector(self, norm=None):
        v = self.g.standard_normal(self.dim)
        return v / np.linalg.norm(v) * np.sqrt(self.scale if norm is None else norm)

    def frame(self, dets, perm=None):
        """dets: [(box, score, label, embed)] -> (boxes [n, 4], scores [n], labels [n] int64, embeds [n, D]), in the
        order perm (default: as given)."""
        if perm is not None:
            dets = [dets[i] for i in perm]
        boxes = torch.tensor([d[0] for d in dets], dtype=torch.float32)
        scores = torch.tensor([d[1] for d in dets], dtype=torch.float32)
        labels = torch.tensor([int(d[2]) for d in dets], dtype=torch.long)
        embeds = torch.from_numpy(np.stack([d[3] for d in dets]).astype(np.float32))
        return boxes, scores, labels, embeds


def golden_sequence(name, frames=20):
    """[(boxes, scores, labels, embeds)] for the setting `name` (its score thresholds place the scores), n <= 40:
    frames 0-7 track objects 0-9 with class-threshold duplicates, backdrop-threshold duplicates, a chain removed only
    through an already-removed row, a partial overlap left at -1 but not a backdrop, a lonely low-score row that becomes
    a backdrop and is matched to its own backdrop the frame after; objects 4, 5 and 6 are absent in frames 3-4, where a
    low-score row with object 4's embedding is suppressed (-2) and a row mixing objects 5 and 6 with object 6's class is
    matched to 6 by the category mask; frame 2 comes unsorted; frames 8-17 hold only three weak rows, so every tracklet
    expires after 10 absent frames; frames 18-19 start afresh."""
    s = SETTINGS[name]
    obj, init = s["obj_score_thr"], s["init_score_thr"]
    world = World(24, DIM, seed=sorted(SETTINGS).index(name) + 11)
    g = world.g
    world.label[5], world.label[6] = 2, 5                       # objects 5 and 6 differ in class
    lonely = world.vector()
    out = []
    for f in range(frames):
        dets = []
        if f < 8:
            present = [o for o in range(8 + (2 if f >= 5 else 0)) if not (f in (3, 4) and o in (4, 5, 6))]
            for o in present:
                dets.append((world.box(o), _score(g, max(init, obj) + 0.02, 0.98), world.label[o],
                             world.base[o] + 0.05 * world.vector(1.0)))
            hi = (obj + 0.01, min(init, 0.98) - 0.01)
            # a class-threshold duplicate of object 1 (IoU about 0.9, score >= obj)
            dets.append((world.box(1, 0.05), _score(g, *hi), world.label[1], world.base[1]))
            # a backdrop-threshold duplicate of object 2 (IoU 0.5, score < obj)
            dets.append((world.box(2, 1 / 3), _score(g, 0.02, obj - 0.01), world.label[2], world.vector(0.1)))
            # a chain beside object 3: Y (IoU 0.5 with 3) removed, Z (IoU 0.5 with Y, 0.2 with 3) removed through Y
            dets.append((world.box(3, 1 / 3), _score(g, 0.12, obj - 0.01), world.label[3], world.vector(0.1)))
            dets.append((world.box(3, 2 / 3), _score(g, 0.02, 0.1), world.label[3], world.vector(0.1)))
            # a partial overlap with object 7 (IoU 0.5, obj <= score <= init): kept, left at -1, not a backdrop
            dets.append((world.box(7, 1 / 3), _score(g, *hi), world.label[7], world.vector(0.3)))
            if f < 3:                                                # a lonely low-score row in its own cell
                dets.append((world.box(30), _score(g, 0.02, obj - 0.01), 1, lonely))
            if f in (3, 4):
                dets.append((world.box(44), _score(g, 0.02, obj - 0.01), world.label[4], world.base[4]))
                mix = 0.55 * world.base[5] + 0.45 * world.base[6]
                dets.append((world.box(45), _score(g, max(init, obj) + 0.02, 0.98), world.label[6], mix))
        elif f < 18:
            for i in range(3):
                dets.append((world.box(50 + i), _score(g, 0.02, obj - 0.01), int(g.integers(0, NUM_CLASSES)),
                             np.zeros(DIM)))
        else:
            for o in range(12, 20):
                dets.append((world.box(o), _score(g, max(init, obj) + 0.02, 0.98), world.label[o],
                             world.base[o] + 0.05 * world.vector(1.0)))
        ordered = sorted(range(len(dets)), key=lambda i: -dets[i][1])
        if f == 2:                                                  # one frame in an unsorted order
            ordered = list(g.permutation(len(dets)))
        out.append(world.frame(dets, ordered))
    return out


def random_sequence(seed, n, frames=4, dim=64):
    """Large frames for the GPU tests, up to n rows: frame 0 has n - 80 objects (all new tracklets); frame 1 has n - 24
    lonely low-score rows (nearly all backdrops) and 24 of the objects; later frames mix the objects (some absent, some
    suppressed at low score), new objects and duplicates, and stay within 1024 live tracklets."""
    objects = n - 80
    world = World(objects + n, dim, seed, scale=32.0)
    g = world.g
    out = []
    for f in range(frames):
        dets = []
        if f == 0:
            for o in range(objects):
                dets.append((world.box(o), _score(g, 0.55, 0.98), world.label[o], world.base[o]))
        elif f == 1:
            for o in range(24):
                dets.append((world.box(o), _score(g, 0.55, 0.98), world.label[o], world.base[o]))
            for c in range(24, n):
                dets.append((world.box(c), _score(g, 0.02, 0.28), world.label[objects + c],
                             world.base[objects + c]))
        else:
            for o in range(objects):
                u = g.random()
                if u < 0.7:
                    dets.append((world.box(o), _score(g, 0.55, 0.98), world.label[o], world.base[o]))
                    if u < 0.05:                                    # a duplicate (IoU about 0.9)
                        dets.append((world.box(o, 0.05), _score(g, 0.35, 0.45), world.label[o], world.base[o]))
                elif u < 0.8:
                    dets.append((world.box(o), _score(g, 0.02, 0.28), world.label[o], world.base[o]))
            for c in range(objects, n + 24):
                if len(dets) >= n:
                    break
                dets.append((world.box(c), _score(g, 0.55, 0.98) if g.random() < 0.25 else _score(g, 0.02, 0.28),
                             world.label[c], world.base[c]))
        dets = dets[:n]
        out.append(world.frame(dets, sorted(range(len(dets)), key=lambda i: -dets[i][1])))
    return out


def checksum(seq):
    """sha256 of a sequence's bytes: pins the generator's output."""
    h = hashlib.sha256()
    for frame in seq:
        for t in frame:
            h.update(t.numpy().tobytes())
    return h.hexdigest()[:16]


# ---- the reference's chain, for timing --------------------------------------------------------------------------------
class ReferenceChain(Restated):
    """The reference's host-driven structure on the tensors' device, for tools/qdtrack_bench.py: the sort, the
    duplicate removal as a loop over the rows with one host read each, the memo concatenated from per-tracklet entries
    and the backdrop list every frame, the matching loop with host reads per row, the new ids, the memory updated id by
    id and the backdrop loop with one host read per candidate.  Its ids are Restated's."""

    def step(self, boxes, scores, labels, embeds, frame_id):
        dev = boxes.device
        n = scores.shape[0]
        _, inds = scores.sort(descending=True, stable=True)
        b, sc, lab, e = boxes[inds], scores[inds], labels[inds], embeds[inds]
        valid = torch.ones(n, dtype=torch.bool, device=dev)
        ious = box_iou(b, b)
        for i in range(1, n):
            thr = float(self.back_iou) if sc[i] < float(self.obj_thr) else float(self.class_iou)
            if (ious[i, :i] > thr).any():
                valid[i] = False
        keep = torch.nonzero(valid.cpu()).squeeze(1).tolist()
        b, sc, lab, e = b[valid], sc[valid], lab[valid], e[valid]
        ids = torch.full((len(keep),), -1, dtype=torch.long)
        if self.tracks:
            memo_e = [self.tracks[t]["embed"][None] for t in self.tracks]
            memo_l = [self.tracks[t]["label"].view(1) for t in self.tracks]
            memo_ids = torch.tensor(list(self.tracks), dtype=torch.long)
            if self.backdrops is not None:
                memo_e.append(self.backdrops[1])
                memo_l.append(self.backdrops[0])
                memo_ids = torch.cat((memo_ids, torch.full((len(self.backdrops[0]),), -1, dtype=torch.long)))
            memo = torch.cat(memo_e)
            ml = torch.cat(memo_l)
            feats = torch.mm(e, memo.t())
            s = (feats.softmax(dim=1) + feats.softmax(dim=0)) / 2
            s *= (lab.view(-1, 1) == ml.view(1, -1)).float()
            for i in range(len(keep)):
                conf, c = torch.max(s[i, :], dim=0)
                tid = memo_ids[c]
                if conf > float(self.match_thr) and tid > -1:
                    if sc[i] > float(self.obj_thr):
                        ids[i] = tid
                        s[:i, c] = 0
                        s[i + 1:, c] = 0
                    elif conf > float(self.conf_thr):
                        ids[i] = -2
        new = (ids == -1) & (sc > float(self.init_thr)).cpu()
        m = int(new.sum())
        ids[new] = torch.arange(self.next_id, self.next_id + m)
        self.next_id += m
        for a, tid in enumerate(ids.tolist()):
            if tid < 0:
                continue
            v = self.tracks.get(tid)
            if v is None:
                self.tracks[tid] = dict(embed=e[a], label=lab[a], last_frame=frame_id)
            else:
                v["embed"] = (1 - self.m) * v["embed"] + self.m * e[a]
                v["label"] = lab[a]
                v["last_frame"] = frame_id
        cand = torch.nonzero(ids == -1).squeeze(1)
        bi = box_iou(b[cand.to(dev)], b)
        back = []
        for a, r in enumerate(cand.tolist()):
            if not (bi[a, :r] > float(self.back_iou)).any():
                back.append(r)
        self.backdrops = (lab[back], e[back]) if self.backdrop_frames else None
        for tid in [t for t, v in self.tracks.items() if frame_id - v["last_frame"] >= self.frames]:
            del self.tracks[tid]
        return inds.cpu().tolist(), keep, ids.tolist()
