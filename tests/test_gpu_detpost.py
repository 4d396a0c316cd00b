"""GPU tests (-m gpu) of detection post-processing (uninext_b200/modules/detection_postprocess.py, kernels
csrc/msda_detpost.cuh) against the reference chain restated below as the reference writes it (uninext_img.py:393-472:
convert_grounding_to_od_logits, sigmoid / sqrt, torchvision's batched_nms, torch.topk, cxcywh -> xyxy, Boxes.scale).

Inputs are tie-free unless a case says otherwise: every token of class c carries the same value k * 2^-16 with k distinct
per (query, class), so the class mean is exact in any summation order and the scores are compared bitwise.  (With
arbitrary token values torch's CUDA mean may sum a class's tokens in another order than the CSR order;
test_scores_of_arbitrary_tokens checks the CSR-order arithmetic bitwise and the chain's scores to 2e-6 relative.)
The NMS keep sets are also compared with torchvision's and with fp32 and fp64 restatements of the greedy sweep; pairs
whose IoU lies within 1e-6 of the threshold are counted and reported."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import torchvision

    from uninext_b200 import _cabi
    from uninext_b200.modules.detection_postprocess import LAUNCHES, postprocess_detections
    from uninext_b200.modules.mask_postprocess import paste_masks

NEAR = 1e-6


def coco_like_map():
    """80 classes of 1 to 3 consecutive tokens, one separator token between classes (a COCO prompt's layout)."""
    pmap, t = {}, 1
    for c in range(80):
        n = 1 + (c % 7 == 3) + (c % 11 == 5)
        pmap[c + 1] = list(range(t, t + n))
        t += n + 1
    assert t <= 256
    return pmap


GROUNDING = {1: [0]}


# ---- the reference chain --------------------------------------------------------------------------------------------
def convert_grounding_to_od_logits(logits, num_classes, positive_map, score_agg="MEAN"):
    """uninext_img.py:598-613."""
    assert logits.ndim == 3
    assert positive_map is not None
    scores = torch.zeros(logits.shape[0], logits.shape[1], num_classes).to(logits.device)
    # 256 -> 80, average for each class
    # score aggregation method
    if score_agg == "MEAN": # True
        for label_j in positive_map:
            scores[:, :, label_j - 1] = logits[:, :, torch.LongTensor(positive_map[label_j])].mean(-1)
    else:
        raise NotImplementedError
    return scores


def box_cxcywh_to_xyxy(x):
    """util/box_ops.py."""
    x_c, y_c, w, h = x.unbind(-1)
    b = [(x_c - 0.5 * w), (y_c - 0.5 * h),
         (x_c + 0.5 * w), (y_c + 0.5 * h)]
    return torch.stack(b, dim=-1)


def chain(box_cls, box_pred, positive_map, image_sizes, iou_pred, nms_iou, max_num_inst):
    """uninext_img.py:389-472 per image (nms_iou None: the OTA-off branch), plus the query each result came from."""
    num_classes = len(positive_map)
    results = []
    for i in range(box_cls.shape[0]):
        logits_per_image = convert_grounding_to_od_logits(box_cls[i].unsqueeze(0), num_classes, positive_map)[0]
        prob = logits_per_image.sigmoid()
        if iou_pred is not None:
            prob = torch.sqrt(prob * iou_pred[i].sigmoid())
        box_pred_per_image = box_pred[i]
        keep_indices = torch.arange(box_cls.shape[1], device=box_cls.device)
        if nms_iou is not None:
            nms_scores, idxs = torch.max(prob, 1)
            boxes_before_nms = box_cxcywh_to_xyxy(box_pred_per_image)
            keep_indices = torchvision.ops.batched_nms(boxes_before_nms, nms_scores, idxs, nms_iou)
            prob = prob[keep_indices]
            box_pred_per_image = box_pred_per_image[keep_indices]
        num_inst = min(max_num_inst, len(prob.view(-1)))
        topk_values, topk_indexes = torch.topk(prob.view(-1), num_inst, dim=0)
        topk_boxes = torch.div(topk_indexes, logits_per_image.shape[1], rounding_mode='floor')
        labels = topk_indexes % logits_per_image.shape[1]
        boxes = box_cxcywh_to_xyxy(box_pred_per_image[topk_boxes])
        boxes[:, 0::2] *= image_sizes[i][1]                                  # Boxes.scale(scale_x=w, scale_y=h)
        boxes[:, 1::2] *= image_sizes[i][0]
        results.append(dict(scores=topk_values, labels=labels, query=keep_indices[topk_boxes], boxes=boxes,
                            keep=keep_indices))
    return results


# ---- inputs ---------------------------------------------------------------------------------------------------------
def make_inputs(B, Q, pmap, T=256, iou=True, seed=0, layout="random"):
    g = torch.Generator().manual_seed(seed)
    C = len(pmap)
    box_cls = torch.rand(B, Q, T, generator=g) * 8 - 4
    for b in range(B):                       # distinct exact class logits in [-4, 4)
        k = torch.randperm(1 << 19, generator=g)[:Q * C].reshape(Q, C) - (1 << 18)
        vals = k.float() * 2.0 ** -16
        for c, label in enumerate(sorted(pmap)):
            box_cls[b][:, pmap[label]] = vals[:, c:c + 1]
    cxcy = torch.rand(B, Q, 2, generator=g)
    wh = torch.rand(B, Q, 2, generator=g) * 0.4 + 0.02
    if layout == "clustered":                # 6 centres, jitter 0.01: heavy suppression
        centres = torch.rand(6, 2, generator=g)
        cxcy = centres[torch.randint(0, 6, (B, Q), generator=g)] + torch.randn(B, Q, 2, generator=g) * 0.01
        wh = 0.2 + torch.rand(B, Q, 2, generator=g) * 0.02
    elif layout == "degenerate":             # zero widths / heights, and boxes reaching below 0
        wh[:, ::5, 0] = 0.0
        wh[:, 1::5, 1] = 0.0
        cxcy[:, 2::5] = cxcy[:, 2::5] * 0.1 - 0.05
        wh[:, 2::5] = wh[:, 2::5] + 0.3
    box_pred = torch.cat((cxcy, wh), -1)
    iou_pred = torch.randn(B, Q, 1, generator=g) * 2 if iou else None
    cuda = lambda x: None if x is None else x.cuda()
    return cuda(box_cls), cuda(box_pred), cuda(iou_pred)


def check_equal(got, want, b):
    n = int(got.count[b])
    assert n == want["scores"].numel()
    assert torch.equal(got.query_index[b, :n].long(), want["query"]), "query_index"
    assert torch.equal(got.labels[b, :n].long(), want["labels"]), "labels"
    assert torch.equal(got.scores[b, :n], want["scores"]), "scores"
    assert torch.equal(got.boxes[b, :n], want["boxes"]), "boxes"
    k = got.scores.shape[1]
    if n < k:                                # documented fill values
        assert bool((got.scores[b, n:] == 0).all() and (got.labels[b, n:] == -1).all())
        assert bool((got.query_index[b, n:] == -1).all() and (got.boxes[b, n:] == 0).all())


# (name, B, Q, map, T, iou, nms, max_num_inst, layout, image sizes)
CASES = [
    ("coco_q300_iou_nms", 1, 300, "coco", 256, True, 0.7, 100, "random", [(480, 640)]),
    ("coco_q300_iou", 1, 300, "coco", 256, True, None, 100, "random", [(480, 640)]),
    ("coco_q300_nms", 1, 300, "coco", 256, False, 0.7, 100, "random", [(480, 640)]),
    ("coco_q300", 1, 300, "coco", 256, False, None, 100, "random", [(480, 640)]),
    ("coco_q900_iou_nms", 1, 900, "coco", 256, True, 0.7, 100, "random", [(800, 1333)]),
    ("coco_q900_iou", 1, 900, "coco", 256, True, None, 100, "random", [(800, 1333)]),
    ("coco_q900_nms", 1, 900, "coco", 256, False, 0.7, 100, "random", [(800, 1333)]),
    ("coco_q900", 1, 900, "coco", 256, False, None, 100, "random", [(800, 1333)]),
    ("grounding", 1, 900, "grounding", 256, True, 0.7, 1, "random", [(720, 1280)]),
    ("grounding_no_nms", 1, 900, "grounding", 256, True, None, 1, "random", [(720, 1280)]),
    ("one_class_few_kept", 1, 120, "one", 256, True, 0.7, 100, "clustered", [(480, 640)]),
    ("256_single_token_classes", 1, 900, "single256", 256, True, 0.7, 100, "random", [(800, 1333)]),
    ("256_single_token_classes_no_nms", 1, 900, "single256", 256, True, None, 100, "random", [(800, 1333)]),
    ("clustered", 1, 900, "coco", 256, True, 0.7, 100, "clustered", [(800, 1333)]),
    ("clustered_3_classes", 1, 900, "three", 256, True, 0.7, 100, "clustered", [(800, 1333)]),
    ("degenerate_boxes", 1, 300, "coco", 256, True, 0.7, 100, "degenerate", [(480, 640)]),
    ("batch4_sizes", 4, 300, "coco", 256, True, 0.7, 100, "random", [(480, 640), (800, 1333), (333, 500), (1024, 768)]),
    ("batch4_sizes_no_nms", 4, 300, "coco", 256, True, None, 100, "random", [(480, 640), (800, 1333), (333, 500), (1024, 768)]),
    ("short_prompt_T64", 2, 900, "three", 64, True, 0.7, 100, "random", [(480, 640), (640, 480)]),
    ("q1024_nms", 1, 1024, "coco", 256, True, 0.7, 100, "clustered", [(800, 1333)]),   # the largest NMS shared memory
]
MAPS = {"coco": coco_like_map, "grounding": lambda: GROUNDING, "one": lambda: {1: [3, 4]},
        "single256": lambda: {c + 1: [c] for c in range(256)}, "three": lambda: {1: [0, 1], 2: [3], 3: [5, 6, 7]}}


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_matches_chain(case):
    name, B, Q, mname, T, iou, nms, k, layout, sizes = case
    pmap = MAPS[mname]()
    box_cls, box_pred, iou_pred = make_inputs(B, Q, pmap, T, iou, seed=CASES.index(case), layout=layout)
    lib = _cabi.load()
    before = lib.msda_launch_count()
    got = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, nms, k)
    assert lib.msda_launch_count() - before == LAUNCHES == 2           # the whole batch
    want = chain(box_cls, box_pred, pmap, sizes, iou_pred, nms, k)
    for b in range(B):
        check_equal(got, want[b], b)
    if mname == "one":
        assert int(got.count[0]) < 100                                  # K * C < 100: count < 100, no error
    print(f"{name}: kept {[int(w['keep'].numel()) for w in want]} of {Q}, count {got.count.tolist()}")


# ---- NMS keep sets --------------------------------------------------------------------------------------------------
def restated_nms(box_pred, scores, classes, thr, dtype):
    """batched_nms's coordinate trick and torchvision's greedy sweep in numpy, every operation in `dtype`."""
    f = np.dtype(dtype).type
    bp = box_pred.astype(dtype)
    hw, hh = f(0.5) * bp[:, 2], f(0.5) * bp[:, 3]
    xyxy = np.stack([bp[:, 0] - hw, bp[:, 1] - hh, bp[:, 0] + hw, bp[:, 1] + hh], -1)
    off = classes.astype(dtype) * (xyxy.max() + f(1))
    bx = xyxy + off[:, None]
    order = np.argsort(-scores, kind="stable")
    bx = bx[order]
    left = np.maximum(bx[:, None, 0], bx[None, :, 0])
    right = np.minimum(bx[:, None, 2], bx[None, :, 2])
    top = np.maximum(bx[:, None, 1], bx[None, :, 1])
    bottom = np.minimum(bx[:, None, 3], bx[None, :, 3])
    inter = np.maximum(right - left, f(0)) * np.maximum(bottom - top, f(0))
    area = (bx[:, 2] - bx[:, 0]) * (bx[:, 3] - bx[:, 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        iou = inter / (area[:, None] + area[None, :] - inter)
    removed = np.zeros(len(order), bool)
    idx = np.arange(len(order))
    t = np.float32(thr) if dtype == np.float32 else float(np.float32(thr))       # torchvision compares with (float)thr
    keep = []
    for i in range(len(order)):
        if removed[i]:
            continue
        keep.append(order[i])
        removed |= (idx > i) & (iou[i] > t)
    near = int((np.triu(np.abs(iou.astype(np.float64) - float(np.float32(thr))) <= NEAR, 1)).sum())
    return set(int(x) for x in keep), near


@pytest.mark.parametrize("layout", ["random", "clustered", "degenerate"])
@pytest.mark.parametrize("Q", [300, 900])
def test_nms_keep_sets(layout, Q):
    pmap = coco_like_map() if layout != "clustered" else {1: [0, 1], 2: [3], 3: [5, 6, 7]}
    C = len(pmap)
    box_cls, box_pred, iou_pred = make_inputs(1, Q, pmap, 256, True, seed=Q + len(layout), layout=layout)
    got = postprocess_detections(box_cls, box_pred, pmap, [(480, 640)], iou_pred, 0.7, Q * C)   # every kept pair
    n = int(got.count[0])
    assert n % C == 0
    mine = set(got.query_index[0, :n].tolist())
    assert len(mine) == n // C
    want = chain(box_cls, box_pred, pmap, [(480, 640)], iou_pred, 0.7, Q * C)[0]
    tv = set(want["keep"].tolist())
    logits = convert_grounding_to_od_logits(box_cls, C, pmap)[0]
    prob = torch.sqrt(logits.sigmoid() * iou_pred[0].sigmoid())
    sc, cl = torch.max(prob, 1)
    bp, sc, cl = box_pred[0].cpu().numpy(), sc.cpu().numpy(), cl.cpu().numpy()
    k32, near32 = restated_nms(bp, sc, cl, 0.7, np.float32)
    k64, near64 = restated_nms(bp, sc, cl, 0.7, np.float64)
    print(f"{layout} Q={Q}: kept {len(mine)}; torchvision differs in {len(mine ^ tv)}, fp64 in {len(mine ^ k64)}; "
          f"{near64} pairs with IoU within {NEAR} of 0.7")
    assert mine == k32                                       # the kernel's arithmetic, restated: the same decisions
    assert mine == tv or near64 > 0
    assert mine == k64 or near64 > 0
    if layout == "clustered":
        assert len(mine) < Q // 4                            # heavy suppression


def test_scores_of_arbitrary_tokens():
    """Arbitrary token values.  Every (query, class) probability equals, bitwise, the documented arithmetic restated in
    torch (the class's tokens added in CSR order, times (float)1/n, sigmoid, sqrt), and is within 2e-6 relative of the
    chain's: torch's CUDA mean may add a class's tokens in another order, which moves the logit by an ulp.  The results
    come in the documented order; max_num_inst = Q*C also takes the sort through the workspace."""
    pmap = coco_like_map()
    g = torch.Generator().manual_seed(5)
    Q, C = 300, 80
    box_cls = (torch.randn(1, Q, 256, generator=g) * 3).cuda()
    box_pred = torch.rand(1, Q, 4, generator=g).cuda()
    iou_pred = torch.randn(1, Q, 1, generator=g).cuda()
    got = postprocess_detections(box_cls, box_pred, pmap, [(480, 640)], iou_pred, None, Q * C)
    prob = torch.sqrt(convert_grounding_to_od_logits(box_cls, C, pmap)[0].sigmoid() * iou_pred[0].sigmoid())
    csr = torch.empty(Q, C, device="cuda")
    for label, toks in pmap.items():
        acc = torch.zeros(Q, device="cuda")
        for t in toks:
            acc = acc + box_cls[0, :, t]
        csr[:, label - 1] = acc * float(np.float32(1) / np.float32(len(toks)))
    csr = torch.sqrt(csr.sigmoid() * iou_pred[0].sigmoid())
    assert int(got.count[0]) == Q * C
    q, c, s = got.query_index[0].long(), got.labels[0].long(), got.scores[0]
    assert torch.equal(torch.sort(q * C + c).values, torch.arange(Q * C, device="cuda"))
    assert torch.equal(s, csr[q, c])
    ref = prob[q, c]
    assert bool(((s - ref).abs() <= 2e-6 * ref).all())
    flat = q * C + c                                         # descending score, ties to the lower flat index
    assert bool(((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (flat[:-1] < flat[1:]))).all())
    print(f"{int((s != ref).sum())} of {Q * C} probabilities differ from the chain's, at most "
          f"{float(((s - ref).abs() / ref).max()):.2e} relative")


@pytest.mark.parametrize("nms", [None, 0.7])
def test_exact_ties_follow_the_documented_order(nms):
    """Token values from {-1, 0, 1}: many equal scores and equal per-query maxima.  Order: higher score first, then the
    lower kept rank (the stable score order of the NMS), then the lower class."""
    pmap = {c + 1: [c] for c in range(4)}
    g = torch.Generator().manual_seed(9)
    Q, C = 64, 4
    box_cls = torch.randint(-1, 2, (1, Q, 256), generator=g).float().cuda()
    box_pred = torch.cat((torch.rand(1, Q, 2, generator=g), torch.full((1, Q, 2), 0.05)), -1).cuda()
    got = postprocess_detections(box_cls, box_pred, pmap, [(100, 200)], None, nms, Q * C)
    prob = convert_grounding_to_od_logits(box_cls, C, pmap)[0].sigmoid()
    if nms is None:
        keep = torch.arange(Q, device="cuda")
    else:
        sc, cl = torch.max(prob, 1)
        keep = torchvision.ops.batched_nms(box_cxcywh_to_xyxy(box_pred[0]), sc, cl, nms)   # stable score order
    v = prob[keep].flatten().cpu().numpy()
    order = np.lexsort((np.arange(v.size), -v))
    n = int(got.count[0])
    assert n == v.size
    assert np.array_equal(got.scores[0, :n].cpu().numpy(), v[order])
    assert np.array_equal(got.labels[0, :n].cpu().numpy(), order % C)
    assert np.array_equal(got.query_index[0, :n].cpu().numpy(), keep.cpu().numpy()[order // C])


def test_no_host_sync_and_no_allocation_beyond_outputs():
    pmap = coco_like_map()
    box_cls, box_pred, iou_pred = make_inputs(2, 900, pmap, seed=21)
    sizes = [(480, 640), (800, 1333)]
    first = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred)     # caches the map and the sizes
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    n = ctypes.c_int64(0)
    _cabi.check(_cabi.load().msda_detpost_workspace(2, 900, 256, 80, 100, ctypes.byref(n)), "msda_detpost_workspace")
    blocks = lambda nbytes: (nbytes + 511) // 512 * 512                            # the caching allocator's rounding
    outs = sum(blocks(t.numel() * t.element_size()) for t in second)
    assert torch.cuda.memory_allocated() - base == outs                             # the workspace is freed on return
    assert torch.cuda.max_memory_allocated() - base == outs + blocks(n.value)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def test_cuda_graph_capture_and_replay():
    pmap = coco_like_map()
    box_cls, box_pred, iou_pred = make_inputs(2, 900, pmap, seed=31)
    sizes = [(480, 640), (800, 1333)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                                      # warm-up on a side stream
        for nms in (0.7, None):
            postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, nms)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ga = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, 0.7)
        gb = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, None)
    for seed in (32, 33):                                                           # new inputs, copied in place
        c2, p2, i2 = make_inputs(2, 900, pmap, seed=seed)
        box_cls.copy_(c2)
        box_pred.copy_(p2)
        iou_pred.copy_(i2)
        g.replay()
        torch.cuda.synchronize()
        for got, nms in ((ga, 0.7), (gb, None)):
            eager = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, nms)
            for a, b in zip(got, eager):
                assert torch.equal(a, b)


def test_captured_graph_survives_cache_eviction():
    """A graph captured with a dict map and listed image sizes reads the cached device tensors.  Dropping them from the
    caches (as the LRU does past its size) and reusing the freed memory must not change what the graph computes."""
    from uninext_b200.modules import detection_postprocess as dp
    pmap = {c + 1: [2 * c, 2 * c + 1] for c in range(7)}            # a map no other test uses
    sizes = [(417, 619), (523, 711)]
    box_cls, box_pred, iou_pred = make_inputs(2, 300, pmap, seed=51)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred)
    dp._csr.cache_clear()
    dp._sizes.cache_clear()
    torch.cuda.empty_cache()
    junk = [torch.full((4096,), -7, dtype=torch.int32, device="cuda") for _ in range(64)]   # reuse freed blocks
    c2, p2, i2 = make_inputs(2, 300, pmap, seed=52)
    box_cls.copy_(c2)
    box_pred.copy_(p2)
    iou_pred.copy_(i2)
    g.replay()
    torch.cuda.synchronize()
    want = chain(box_cls, box_pred, pmap, sizes, iou_pred, 0.7, 100)
    for b in range(2):
        check_equal(out, want[b], b)
    del junk


def test_then_paste_masks_gives_the_chain_masks():
    """postprocess_detections then paste_masks on the selected queries: the chain's final binary masks
    (uninext_img.py:474-479, then segmentation_postprocess's nearest resize), except pixels within 1e-6 of 0.5."""
    import torch.nn.functional as F
    pmap = coco_like_map()
    B, Q = 2, 300
    box_cls, box_pred, iou_pred = make_inputs(B, Q, pmap, seed=41)
    mask_pred = (torch.rand(B, Q, 1, 40, 60, generator=torch.Generator().manual_seed(42)) * 20 - 10).cuda()
    sizes, outs = [(150, 230), (160, 240)], [(300, 460), (120, 180)]
    got = postprocess_detections(box_cls, box_pred, pmap, sizes, iou_pred, 0.7, 100)
    want = chain(box_cls, box_pred, pmap, sizes, iou_pred, 0.7, 100)
    for b in range(B):
        n = int(got.count[b])
        masks = paste_masks(mask_pred[b][got.query_index[b, :n]], sizes[b], outs[b], 4, 0.5)
        mask_pred_i = mask_pred[b][want[b]["query"]]
        N, C, H, W = mask_pred_i.shape
        mask = F.interpolate(mask_pred_i, size=(H*4, W*4), mode='bilinear', align_corners=False)
        p = mask.sigmoid()
        mask = p > 0.5
        mask = mask[:,:,:sizes[b][0],:sizes[b][1]]
        mask = F.interpolate(mask.float(), size=outs[b], mode='nearest').squeeze(1).bool()
        p = F.interpolate(p[:, :, :sizes[b][0], :sizes[b][1]], size=outs[b], mode='nearest').squeeze(1)
        assert masks.shape == mask.shape
        assert int(((masks != mask) & ((p - 0.5).abs() > NEAR)).sum()) == 0


def test_bad_arguments_raise():
    pmap = coco_like_map()
    box_cls, box_pred, iou_pred = make_inputs(1, 30, pmap, seed=1)
    with pytest.raises(ValueError, match="max_num_inst"):
        postprocess_detections(box_cls, box_pred, pmap, [(10, 10)], iou_pred, 0.7, 30 * 80 + 1)
    with pytest.raises(ValueError, match="outside"):
        postprocess_detections(box_cls[:, :, :100], box_pred, pmap, [(10, 10)], iou_pred)   # tokens past T = 100
    with pytest.raises(ValueError, match="1..C"):
        postprocess_detections(box_cls, box_pred, {2: [0]}, [(10, 10)])
    with pytest.raises(ValueError, match="image sizes"):
        postprocess_detections(box_cls, box_pred, pmap, [(10, 10), (20, 20)])
    with pytest.raises(RuntimeError, match="CPU"):
        postprocess_detections(box_cls, box_pred, pmap, [(10, 10)], iou_pred.cpu())
    half = postprocess_detections(box_cls.half(), box_pred.half(), pmap, [(10, 10)], iou_pred.half())
    full = postprocess_detections(box_cls.half().float(), box_pred.half().float(), pmap, [(10, 10)], iou_pred.half().float())
    for a, b in zip(half, full):
        assert torch.equal(a, b)
