"""GPU tests (-m gpu) of the video trackers' detection selection (select_track_detections in
uninext_b200/modules/detection_postprocess.py, trackpost_select in csrc/msda_detpost.cuh) against both reference chains
restated in tests/trackpost_case.py (uninext_vid.py:1224-1250 inference_mot, :1380-1415 inference_vis, with torchvision's
batched_nms).

Inputs are tie-free (every token of class c carries the same value k * 2^-16, k distinct per (query, class)), so the
queries, labels, scores and boxes are compared bitwise and in order.  The NMS keep sets are also compared with an fp32
restatement of the kernel's arithmetic, exactly, and with torchvision's; pairs whose IoU lies within an fp32 ulp of the
threshold are counted and reported.  The NMS code is shared with postprocess_detections (csrc/msda_nms.cuh); its
outputs are compared bitwise with those the library gave before the code was shared (tests/golden/detpost/outputs.npz)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import torchvision

    from tests import test_gpu_detpost as dt
    from tests import trackpost_case as tc
    from uninext_b200 import _cabi
    from uninext_b200.modules.detection_postprocess import LAUNCHES, postprocess_detections, select_track_detections

NMS = {"mot": 0.7, "vis": 0.9}
FORMAT = {"mot": "xyxy_pixels", "vis": "cxcywh"}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detpost", "outputs.npz")


def run(path, box_cls, box_pred, pmap, iou_pred, thr, sizes=None):
    return select_track_detections(box_cls, box_pred, pmap, iou_pred, score_thres=thr, nms_iou=NMS[path],
                                   box_format=FORMAT[path], ori_sizes=sizes if path == "mot" else None)


def check_equal(got, want, b):
    n = int(got.count[b])
    assert n == want["query"].numel() >= 1
    assert torch.equal(got.query_index[b, :n].long(), want["query"]), "query_index"
    assert torch.equal(got.labels[b, :n].long(), want["labels"]), "labels"
    assert torch.equal(got.scores[b, :n], want["scores"]), "scores"
    assert torch.equal(got.boxes[b, :n], want["boxes"]), "boxes"
    if n < got.scores.shape[1]:              # detpost's fill values
        assert bool((got.scores[b, n:] == 0).all() and (got.labels[b, n:] == -1).all())
        assert bool((got.query_index[b, n:] == -1).all() and (got.boxes[b, n:] == 0).all())


def candidates(box_cls, pmap, iou_pred, b, thr):
    prob = tc.convert_grounding_to_od_logits(box_cls[b:b + 1], len(pmap), pmap)[0].sigmoid()
    if iou_pred is not None:
        prob = torch.sqrt(prob * iou_pred[b].sigmoid())
    sc, cl = torch.max(prob, 1)
    return sc, cl, int((sc > thr).sum())


# (name, path, B, Q, map, iou, thr, layout, logit_shift, iou_shift, ori sizes)
GRID = [(f"{p}_q{q}{'_iou' if iou else ''}_t{thr}", p, 1, q, "bdd" if p == "mot" else "ytvis", iou, thr, "random",
         -5.0 if p == "mot" else -6.0, 0.0, [(720, 1280)])
        for p in ("mot", "vis") for q in (300, 900) for iou in (True, False) for thr in (0.05, 0.1)]
CASES = GRID + [
    ("mot_no_candidate", "mot", 1, 900, "bdd", True, 0.1, "random", -12.0, 0.0, [(720, 1280)]),
    ("vis_no_candidate", "vis", 1, 300, "ytvis", False, 0.05, "random", -12.0, 0.0, None),
    ("mot_every_query", "mot", 1, 900, "bdd", True, 0.1, "random", 6.0, 8.0, [(720, 1280)]),
    ("vis_every_query", "vis", 1, 300, "ovis", False, 0.05, "random", 6.0, 0.0, None),
    ("mot_clustered", "mot", 1, 900, "bdd", True, 0.05, "clustered", -2.0, 0.0, [(720, 1280)]),
    ("vis_clustered", "vis", 1, 900, "ovis", True, 0.05, "clustered", -2.0, 0.0, None),
    ("mot_degenerate", "mot", 1, 300, "bdd", True, 0.05, "degenerate", -2.0, 0.0, [(720, 1280)]),
    ("vis_degenerate", "vis", 1, 300, "ytvis", True, 0.05, "degenerate", -4.0, 0.0, None),
    ("mot_3_frames_sizes", "mot", 3, 300, "bdd", True, 0.1, "random", -4.0, 0.0, [(720, 1280), (375, 1242), (1080, 1920)]),
    ("vis_3_frames", "vis", 3, 300, "ytvis", True, 0.1, "random", -5.0, 0.0, None),
    ("mot_q1024", "mot", 1, 1024, "bdd", True, 0.05, "clustered", 0.0, 0.0, [(720, 1280)]),
    ("vis_q1024", "vis", 1, 1024, "ovis", False, 0.1, "random", 0.0, 0.0, None),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_matches_chain(case):
    name, path, B, Q, mname, iou, thr, layout, shift, ishift, sizes = case
    pmap = tc.MAPS[mname]()
    box_cls, box_pred, iou_pred = tc.make_inputs(B, Q, pmap, 256, iou, seed=CASES.index(case), layout=layout,
                                                 logit_shift=shift, iou_shift=ishift)
    lib = _cabi.load()
    before = lib.msda_launch_count()
    got = run(path, box_cls, box_pred, pmap, iou_pred, thr, sizes)
    assert lib.msda_launch_count() - before == LAUNCHES == 2           # all frames, whether the fallback fires or not
    want = tc.chain(path, box_cls, box_pred, pmap, iou_pred, thr, sizes)
    n = [candidates(box_cls, pmap, iou_pred, b, thr)[2] for b in range(B)]
    for b in range(B):
        check_equal(got, want[b], b)
    if "no_candidate" in name:
        assert n == [0] * B and got.count.tolist() == [1] * B
    if "every_query" in name:
        assert n == [Q] * B
    print(f"{name}: {n} candidates of {Q}, kept {got.count.tolist()}")


def test_fallback_takes_the_lowest_query_on_exact_ties():
    """No candidate and several queries sharing the largest max_score: the lowest of them, without NMS."""
    pmap = {1: [0], 2: [1]}
    Q = 64
    box_cls = torch.full((1, Q, 4), -9.0, device="cuda")
    box_cls[0, [40, 17, 53], 1] = -5.0                                   # three equal maxima, class 1
    box_pred = torch.rand(1, Q, 4, generator=torch.Generator().manual_seed(3)).cuda()
    got = select_track_detections(box_cls, box_pred, pmap, score_thres=0.1, nms_iou=0.7, box_format="cxcywh")
    assert int(got.count[0]) == 1 and int(got.query_index[0, 0]) == 17 and int(got.labels[0, 0]) == 1
    assert torch.equal(got.boxes[0, 0], box_pred[0, 17])
    assert float(got.scores[0, 0]) == float(torch.tensor(-5.0, device="cuda").sigmoid())


# ---- NMS keep sets --------------------------------------------------------------------------------------------------
def near_pairs(boxes, scores, classes, thr):
    """Pairs of the candidates whose fp64 IoU after the coordinate trick lies within one fp32 ulp of thr."""
    bp = boxes.astype(np.float64)
    xyxy = np.stack([bp[:, 0] - 0.5 * bp[:, 2], bp[:, 1] - 0.5 * bp[:, 3], bp[:, 0] + 0.5 * bp[:, 2],
                     bp[:, 1] + 0.5 * bp[:, 3]], -1)
    bx = xyxy + (classes.astype(np.float64) * (xyxy.max() + 1))[:, None]
    left, right = np.maximum(bx[:, None, 0], bx[None, :, 0]), np.minimum(bx[:, None, 2], bx[None, :, 2])
    top, bottom = np.maximum(bx[:, None, 1], bx[None, :, 1]), np.minimum(bx[:, None, 3], bx[None, :, 3])
    inter = np.maximum(right - left, 0) * np.maximum(bottom - top, 0)
    area = (bx[:, 2] - bx[:, 0]) * (bx[:, 3] - bx[:, 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        iou = inter / (area[:, None] + area[None, :] - inter)
    t = np.float32(thr)
    return int(np.triu(np.abs(iou - float(t)) <= float(np.spacing(t)), 1).sum())


@pytest.mark.parametrize("layout", ["random", "clustered", "degenerate"])
@pytest.mark.parametrize("path", ["mot", "vis"])
@pytest.mark.parametrize("Q", [300, 900])
def test_nms_keep_sets(layout, path, Q):
    pmap = tc.MAPS["bdd" if path == "mot" else "ovis"]()
    thr = 0.05
    box_cls, box_pred, iou_pred = tc.make_inputs(1, Q, pmap, 256, True, seed=100 + Q + len(layout) + len(path),
                                                 layout=layout, logit_shift=-1.0)
    got = run(path, box_cls, box_pred, pmap, iou_pred, thr, [(480, 640)])
    mine = set(got.query_index[0, :int(got.count[0])].tolist())
    sc, cl, n = candidates(box_cls, pmap, iou_pred, 0, thr)
    assert n > 1
    cand = torch.nonzero(sc > thr).squeeze(1)
    bp, s, c = box_pred[0, cand].cpu().numpy(), sc[cand].cpu().numpy(), cl[cand].cpu().numpy()
    k32, _ = dt.restated_nms(bp, s, c, NMS[path], np.float32)
    ci = cand.cpu().numpy()
    want32 = {int(ci[k]) for k in k32}
    tv = set(cand[torchvision.ops.batched_nms(tc.box_cxcywh_to_xyxy(box_pred[0, cand]), sc[cand], cl[cand],
                                              NMS[path])].tolist())
    near = near_pairs(bp, s, c, NMS[path])
    print(f"{path} {layout} Q={Q}: {n} candidates, kept {len(mine)}; torchvision differs in {len(mine ^ tv)}; "
          f"{near} pairs with IoU within an fp32 ulp of {NMS[path]}")
    assert mine == want32                                    # the kernel's arithmetic, restated: the same decisions
    assert mine == tv or near > 0


# ---- runtime behaviour ----------------------------------------------------------------------------------------------
def test_no_host_sync_on_a_second_call():
    pmap = tc.MAPS["bdd"]()
    box_cls, box_pred, iou_pred = tc.make_inputs(2, 900, pmap, seed=21, logit_shift=-4.0)
    sizes = [(720, 1280), (375, 1242)]
    first = [run(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes) for p in ("mot", "vis")]   # caches map and sizes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = [run(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes) for p in ("mot", "vis")]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    for x, y in zip(first, second):
        for a, b in zip(x, y):
            assert torch.equal(a, b)


def test_cuda_graph_replay_on_new_inputs_and_after_cache_eviction():
    """A graph captured with a dict map and listed ori_sizes, replayed on new inputs copied in place, equals eager; also
    after the caches have dropped the device tensors it reads and their memory has been reused.  One of the new inputs
    has no candidate, so the fallback runs inside the graph."""
    from uninext_b200.modules import detection_postprocess as dp
    pmap = {c + 1: [3 * c, 3 * c + 1] for c in range(9)}               # a map no other test uses
    sizes = [(431, 613), (577, 1021)]
    box_cls, box_pred, iou_pred = tc.make_inputs(2, 900, pmap, seed=61, logit_shift=-3.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for p in ("mot", "vis"):
            run(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = {p: run(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes) for p in ("mot", "vis")}
    for step, (seed, shift) in enumerate(((62, -3.0), (63, -12.0), (64, 1.0))):
        if step == 1:
            dp._csr.cache_clear()
            dp._sizes.cache_clear()
            torch.cuda.empty_cache()
            junk = [torch.full((4096,), -7, dtype=torch.int32, device="cuda") for _ in range(64)]   # reuse freed blocks
        c2, p2, i2 = tc.make_inputs(2, 900, pmap, seed=seed, logit_shift=shift)
        box_cls.copy_(c2)
        box_pred.copy_(p2)
        iou_pred.copy_(i2)
        g.replay()
        torch.cuda.synchronize()
        for p in ("mot", "vis"):
            want = tc.chain(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes)
            for b in range(2):
                check_equal(outs[p], want[b], b)
            eager = run(p, box_cls, box_pred, pmap, iou_pred, 0.1, sizes)
            for a, e in zip(outs[p], eager):
                assert torch.equal(a, e)
        if shift < -10:
            assert outs["mot"].count.tolist() == [1, 1]
    del junk


def test_bad_arguments_raise():
    pmap = tc.MAPS["bdd"]()
    box_cls, box_pred, iou_pred = tc.make_inputs(1, 30, pmap, seed=1)
    kw = dict(score_thres=0.1, nms_iou=0.7)
    with pytest.raises(ValueError, match="box_format"):
        select_track_detections(box_cls, box_pred, pmap, iou_pred, box_format="xywh", **kw)
    with pytest.raises(ValueError, match="needs ori_sizes"):
        select_track_detections(box_cls, box_pred, pmap, iou_pred, box_format="xyxy_pixels", **kw)
    with pytest.raises(ValueError, match="ori_sizes"):
        select_track_detections(box_cls, box_pred, pmap, iou_pred, box_format="xyxy_pixels", ori_sizes=[(1, 2), (3, 4)],
                                **kw)
    with pytest.raises(ValueError, match="Q <= 1024"):
        big = torch.zeros(1, 1025, 256, device="cuda")
        select_track_detections(big, torch.zeros(1, 1025, 4, device="cuda"), pmap, box_format="cxcywh", **kw)
    with pytest.raises(ValueError, match="outside"):
        select_track_detections(box_cls[:, :, :10], box_pred, pmap, iou_pred, box_format="cxcywh", **kw)
    with pytest.raises(RuntimeError, match="CPU"):
        select_track_detections(box_cls, box_pred, pmap, iou_pred.cpu(), box_format="cxcywh", **kw)
    with pytest.raises(TypeError):
        select_track_detections(box_cls, box_pred, pmap, iou_pred, 0.1, 0.7, "cxcywh")      # keyword-only
    sizes = torch.tensor([[480, 640]], dtype=torch.int32, device="cuda")
    a = select_track_detections(box_cls, box_pred, pmap, iou_pred, box_format="xyxy_pixels", ori_sizes=sizes, **kw)
    b = select_track_detections(box_cls, box_pred, pmap, iou_pred, box_format="xyxy_pixels", ori_sizes=[(480, 640)], **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- postprocess_detections after the NMS code moved --------------------------------------------------------------
def golden_cases():
    """(name, call) of postprocess_detections on the inputs of tests/test_gpu_detpost.py: every chain case, arbitrary
    token values, exact ties.  tests/golden/make_detpost_golden.py stores their outputs."""
    out = []
    for case in dt.CASES:
        name, B, Q, mname, T, iou, nms, k, layout, sizes = case
        pmap = dt.MAPS[mname]()
        inputs = dt.make_inputs(B, Q, pmap, T, iou, seed=dt.CASES.index(case), layout=layout)
        out.append((name, lambda i=inputs, p=pmap, s=sizes, n=nms, kk=k: postprocess_detections(i[0], i[1], p, s, i[2],
                                                                                                  n, kk)))
    g = torch.Generator().manual_seed(5)
    arb = ((torch.randn(1, 300, 256, generator=g) * 3).cuda(), torch.rand(1, 300, 4, generator=g).cuda(),
           torch.randn(1, 300, 1, generator=g).cuda())
    for nms in (None, 0.7):
        out.append((f"arbitrary_tokens_{nms}", lambda nms=nms: postprocess_detections(arb[0], arb[1], dt.coco_like_map(),
                                                                                     [(480, 640)], arb[2], nms, 100)))
    g = torch.Generator().manual_seed(9)
    ties = (torch.randint(-1, 2, (1, 64, 256), generator=g).float().cuda(),
            torch.cat((torch.rand(1, 64, 2, generator=g), torch.full((1, 64, 2), 0.05)), -1).cuda())
    out.append(("exact_ties_nms", lambda: postprocess_detections(ties[0], ties[1], {c + 1: [c] for c in range(4)},
                                                                 [(100, 200)], None, 0.7, 256)))
    return out


def test_postprocess_detections_outputs_are_unchanged():
    stored = np.load(GOLDEN)
    for name, call in golden_cases():
        got = call()
        for field, t in zip(got._fields, got):
            assert np.array_equal(t.cpu().numpy(), stored[f"{name}/{field}"]), f"{name}: {field}"
