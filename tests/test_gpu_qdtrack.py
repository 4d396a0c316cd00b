"""GPU tests of the QuasiDense tracker's association step (QuasiDenseTracker, msda_qdtrack_match_f32, DESIGN.md section
3.19): the reference's goldens through both entry points, large random sequences against the restatement of
tests/qdtrack_case.py run on CUDA, the IoU predicates bit for bit, the documented ties, the launch count, no host
synchronisation, the error word, and a whole BDD frame sequence from select_track_detections."""
import os

import numpy as np
import pytest
import torch

from tests import qdtrack_case as qc

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qdtrack")


def _tracker(name="bdd", **over):
    from uninext_b200.modules.tracker import QuasiDenseTracker
    return QuasiDenseTracker(**qc.SETTINGS[name], **over)


def _selected(boxes, scores, labels, embeds, seed=0):
    """The frame as select_track_detections gives it (rows in score order, stable) with its rows' embeddings scattered
    over Q = n + 5 queries: (dets, 0, pred_inst_embed [1, Q, D]) and the input row at each of dets' rows."""
    from uninext_b200.modules.detection_postprocess import TrackDetections
    n = scores.shape[0]
    q = min(n + 5, 1024)
    srt = torch.sort(scores, descending=True, stable=True).indices
    perm = torch.randperm(q, generator=torch.Generator().manual_seed(seed))
    pe = torch.randn(1, q, embeds.shape[1])
    pe[0, perm[:n]] = embeds[srt]
    sc, lb, bx = torch.zeros(1, q), torch.full((1, q), -1, dtype=torch.int32), torch.zeros(1, q, 4)
    qi = torch.full((1, q), -1, dtype=torch.int32)
    sc[0, :n], lb[0, :n], bx[0, :n], qi[0, :n] = scores[srt], labels[srt].int(), boxes[srt], perm[:n].int()
    dets = TrackDetections(sc.cuda(), lb.cuda(), bx.cuda(), qi.cuda(), torch.tensor([n], dtype=torch.int32).cuda())
    return (dets, 0, pe.cuda()), srt.tolist()


def _check_state(tr, z, f):
    st = tr.tracklets()
    assert sorted(st) == z[f"{f}/track_ids"].tolist(), f
    scale = max(float(np.abs(z[f"{f}/embed"]).max()) if z[f"{f}/embed"].size else 1.0, 1.0)
    for c, k in enumerate(sorted(st)):
        assert (st[k]["last_frame"], st[k]["label"]) == (z[f"{f}/last_frame"][c], z[f"{f}/label"][c])
        np.testing.assert_allclose(st[k]["embed"].numpy(), z[f"{f}/embed"][c], rtol=0, atol=1e-5 * scale)
    bd = tr.backdrops()
    assert bd["labels"].tolist() == z[f"{f}/back_labels"].tolist(), f
    if bd["labels"].numel():
        np.testing.assert_allclose(bd["embeds"].numpy(), z[f"{f}/back_embeds"], rtol=0, atol=1e-5 * scale)


@pytest.mark.parametrize("name", sorted(qc.SETTINGS))
def test_golden_sequences_through_match_and_match_selected(name):
    z = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    seq = qc.golden_sequence(name)
    assert str(z["checksum"]) == qc.checksum(seq)
    a, b = _tracker(name), _tracker(name)
    for f, (boxes, scores, labels, embeds) in enumerate(seq):
        n = scores.shape[0]
        bboxes = torch.cat((boxes, scores[:, None]), 1).cuda()
        indices = [3 * r + 7 for r in range(n)]
        ob, ol, ids, idx = a.match(bboxes, labels.cuda(), embeds.cuda(), f, indices)
        rows = z[f"{f}/rows"].tolist()
        assert ids.dtype == torch.int64 and not ids.is_cuda
        assert ids.tolist() == z[f"{f}/ids"].tolist(), f
        assert idx == z[f"{f}/indices"].tolist() and torch.equal(ob, bboxes[rows]) and ol.tolist() == labels[rows].tolist()
        args, srt = _selected(boxes, scores, labels, embeds, seed=f)
        res = b.match_selected(*args, f)
        trows, tids = b.read(res)
        got = res.ids.cpu()[:n].tolist()
        assert res.order.cpu()[:n].tolist() == list(range(n))                  # select_track_detections' order
        assert [srt[p] for p in range(n) if got[p] != -3] == rows
        assert [i for i in got if i != -3] == z[f"{f}/ids"].tolist()
        assert trows == [p for p in range(n) if got[p] > -1] and tids == [got[p] for p in trows]
        for tr in (a, b):
            _check_state(tr, z, f)
            assert tr.num_tracklets == a.num_tracklets


@pytest.mark.parametrize("name,n,seed", [("bdd", 1024, 1), ("defaults", 1024, 6), ("bdd_nobackdrop", 1000, 3),
                                         ("bdd", 300, 4)])
def test_random_sequences_match_the_restatement_on_cuda(name, n, seed):
    seq = qc.random_sequence(seed, n)
    ref = qc.Restated(**qc.SETTINGS[name])
    tr = _tracker(name)
    widest = 0
    for f, (boxes, scores, labels, embeds) in enumerate(seq):
        order, keep, want = ref.step(boxes.cuda(), scores.cuda(), labels.cuda(), embeds.cuda(), f)
        bd = tr.backdrops()["labels"].numel() if f else 0
        widest = max(widest, len(tr.tracklets()) + bd)
        args, srt = _selected(boxes, scores, labels, embeds, seed=seed * 100 + f)
        res = tr.match_selected(*args, f)
        tr.read(res)
        got = res.ids.cpu()[:scores.shape[0]].tolist()
        assert [p for p in range(len(got)) if got[p] != -3] == keep, f
        assert [got[p] for p in keep] == want, f
        assert sorted(tr.tracklets()) == sorted(ref.tracks)
    assert min(ref.margins) >= 1e-4, f"the generator left a decision within {min(ref.margins):.2e} of flipping"
    assert {"new", "left", "suppressed"} <= ref.seen and {"dup_class", "dup_backdrop"} & ref.seen
    if (name, n) == ("bdd", 1024):
        assert widest >= 1900


def _pair_frames():
    """(box a, box b, score b) pairs: degenerate, tiny, inverted and threshold-exact ones."""
    pairs = [
        ([0, 0, 10, 10], [0, 0, 10, 7], 0.35),          # IoU exactly fp32(0.7): not removed
        ([0, 0, 10, 10], [0, 0, 10, 3], 0.35),          # IoU 0.3 (and a backdrop test exactly at 0.3)
        ([0, 0, 10, 10], [0, 0, 10, 5], 0.3),           # score exactly at obj_score_thr: the class threshold
        ([0, 0, 10, 10], [0, 0, 10, 5], 0.2999),        # just below: the backdrop threshold
        ([0, 0, 0, 10], [0, 0, 0, 10], 0.2),            # zero width
        ([5, 5, 5, 5], [5, 5, 5, 5], 0.2),              # points
        ([0, 0, 1e-4, 1e-4], [0, 0, 1e-4, 1e-4], 0.2),  # union below 1e-6: IoU 0.01
        ([0, 0, 1e-3, 1e-3], [0, 0, 1e-3, 1e-3], 0.2),  # union 1e-6 and over
        ([0, 0, 2e-3, 1e-3], [0, 0, 1e-3, 1e-3], 0.2),
        ([10, 10, 0, 0], [10, 10, 0, 0], 0.2),          # inverted
        ([10, 10, 0, 0], [0, 0, 10, 10], 0.2),
        ([0, 10, 10, 0], [0, 10, 10, 0], 0.2),          # inverted in y only: negative areas
        ([0, 0, 10, -5], [0, 0, 10, 10], 0.2),
        ([-5, -5, 5, 5], [-4, -5, 6, 5], 0.2),
    ]
    g = torch.Generator().manual_seed(5)
    for _ in range(40):                                  # near-threshold random pairs
        a = (torch.rand(4, generator=g) * 20).tolist()
        b = (torch.tensor(a) + torch.randn(4, generator=g) * 3).tolist()
        pairs.append((a, b, 0.25 + float(torch.rand(1, generator=g)) * 0.1))
    return pairs


def test_iou_predicates_equal_the_fp32_mmcv_formula():
    """Two low-score rows per frame (no new ids, no tracklets): row 1 is removed exactly when the fp32 mmcv IoU on
    CUDA exceeds its threshold, and is a backdrop exactly when it is kept and the IoU does not exceed
    nms_backdrop_iou_thr."""
    tr = _tracker("bdd")
    obj = torch.tensor(0.3, dtype=torch.float32)
    for f, (a, b, s1) in enumerate(_pair_frames()):
        boxes = torch.tensor([a, b], dtype=torch.float32)
        scores = torch.tensor([0.45, s1], dtype=torch.float32)
        iou = float(qc.box_iou(boxes.cuda(), boxes.cuda())[0, 1])
        thr = 0.3 if scores[1] < obj else 0.7
        removed = iou > np.float32(thr)
        bboxes = torch.cat((boxes, scores[:, None]), 1).cuda()
        _, _, ids, _ = tr.match(bboxes, torch.zeros(2, dtype=torch.long).cuda(), torch.zeros(2, 8).cuda(), f, [0, 1])
        assert ids.tolist() == ([-1] if removed else [-1, -1]), (a, b, s1, iou)
        assert tr.backdrops()["labels"].numel() == 1 + (not removed and not iou > np.float32(0.3)), (a, b, iou)
    # the threshold-exact cases as documented
    exact = torch.tensor([[0, 0, 10, 10], [0, 0, 10, 7]], dtype=torch.float32).cuda()
    assert float(qc.box_iou(exact, exact)[0, 1]) == float(np.float32(0.7))


def test_ties_in_the_sort_and_the_argmax():
    tr = _tracker("bdd")
    e = torch.randn(1, 32) * 3
    # equal scores keep their row order; two tracklets with equal embeddings and labels
    boxes = torch.tensor([[0, 0, 10, 10], [100, 0, 110, 10], [200, 0, 210, 10]], dtype=torch.float32)
    scores = torch.tensor([0.8, 0.9, 0.8])
    bboxes = torch.cat((boxes, scores[:, None]), 1).cuda()
    feats = torch.cat((e, e, torch.randn(1, 32) * 3)).cuda()
    res = tr._run(bboxes[:, :4], bboxes[:, 4], torch.tensor([1, 1, 2]).cuda(), feats,
                  torch.arange(3, dtype=torch.int32).cuda(), torch.tensor([3], dtype=torch.int32).cuda(), 0)
    rows, ids = tr.read(res)
    assert res.order.tolist() == [1, 0, 2] and rows == [1, 0, 2] and ids == [0, 1, 2]
    # a row scoring the same against tracklets 0 and 1 takes the lower column: id 0
    _, _, ids, _ = tr.match(torch.tensor([[0, 0, 10, 10, 0.9]]).cuda(), torch.tensor([1]).cuda(), e.cuda(), 1, [0])
    assert ids.tolist() == [0]


def test_launch_count_is_constant_per_call():
    from uninext_b200 import _cabi
    from uninext_b200.modules.tracker import LAUNCHES
    lib = _cabi.load()
    tr = _tracker("bdd")
    for f, frame in enumerate(qc.golden_sequence("bdd")):
        args, _ = _selected(*frame)
        torch.cuda.synchronize()
        before = lib.msda_launch_count()
        res = tr.match_selected(*args, f)
        assert lib.msda_launch_count() - before == LAUNCHES == 8
        tr.read(res)


def test_second_match_selected_does_not_synchronise():
    seq = qc.golden_sequence("bdd")
    tr = _tracker("bdd")
    first, _ = _selected(*seq[0])
    second, _ = _selected(*seq[1])
    tr.read(tr.match_selected(*first, 0))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = tr.match_selected(*second, 1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    rows, ids = tr.read(res)
    assert ids and all(i >= 0 for i in ids)


def _state_copy(tr):
    return tr.state.clone(), tr.embed.clone(), tr.backdrop_embed.clone()


def test_overflow_and_bad_rows_raise_and_keep_the_state_before():
    seq = qc.golden_sequence("bdd")
    for kind in ("overflow", "bad_row"):
        tr = _tracker("bdd", max_tracklets=9)
        args, _ = _selected(*seq[0])
        tr.read(tr.match_selected(*args, 0))                           # 8 tracklets
        before = _state_copy(tr)
        args, _ = _selected(*seq[5], seed=5)                            # 10 objects: two new ones
        if kind == "bad_row":
            tr = _tracker("bdd")
            tr.read(tr.match_selected(*_selected(*seq[0])[0], 0))
            before = _state_copy(tr)
            args[0].query_index[0, 3] = args[2].shape[1]               # past the embeddings
        res = tr.match_selected(*args, 1)
        with pytest.raises(RuntimeError, match="max_tracklets=9" if kind == "overflow" else "outside"):
            tr.read(res)
        after = _state_copy(tr)
        assert torch.equal(after[0][3:], before[0][3:]) and torch.equal(after[0][:2], before[0][:2])
        assert torch.equal(after[1], before[1]) and torch.equal(after[2], before[2])
        with pytest.raises(RuntimeError):                              # sticky
            tr.read(tr.match_selected(*_selected(*seq[1])[0], 2))


def test_whole_bdd_frames_from_select_track_detections():
    """Q = 900 queries, the 8-class BDD map and the IoU branch, 20 frames: select_track_detections -> match_selected ->
    read gives the restated reference chain's (uninext_vid.py:1227-1257 with the reference's host-driven tracker)
    tracked queries and ids."""
    from tests import trackpost_case as tp
    from uninext_b200.modules.detection_postprocess import select_track_detections
    pmap = tp.MAPS["bdd"]()
    g = torch.Generator().manual_seed(9)
    base = torch.randn(900, 256, generator=g)
    base = (base / base.norm(dim=1, keepdim=True) * 5.0).cuda()
    objects = torch.randperm(900, generator=g)[:60].cuda()     # queries that see an object in every frame
    tr, ref = _tracker("bdd"), qc.ReferenceChain(**qc.BDD)
    tracked = 0
    for f in range(20):
        box_cls, box_pred, iou_pred = tp.make_inputs(1, 900, pmap, seed=300 + f, logit_shift=-7.0)
        box_cls[0, objects] += 9.0
        iou_pred[0, objects] = 4.0
        embed = base + 0.05 * torch.randn(900, 256, generator=g).cuda()
        indices, det_bboxes, det_labels = tp.mot_chain(box_cls[0], box_pred[0].clone(), iou_pred[0], pmap, (720, 1280),
                                                       0.1)
        indices = torch.as_tensor(indices).tolist()
        order, keep, ids = ref.step(det_bboxes[:, :4], det_bboxes[:, 4], det_labels, embed[indices], f)
        want_q = [indices[p] for p, i in zip(keep, ids) if i > -1]
        want_ids = [i for i in ids if i > -1]
        dets = select_track_detections(box_cls, box_pred, pmap, iou_pred, score_thres=0.1, nms_iou=0.7,
                                       box_format="xyxy_pixels", ori_sizes=[(720, 1280)])
        rows, got_ids = tr.read(tr.match_selected(dets, 0, embed[None], f))
        assert dets.query_index[0, rows].tolist() == want_q and got_ids == want_ids, f
        tracked += len(rows)
    assert tracked >= 20 * 50 and ref.next_id == tr.num_tracklets
