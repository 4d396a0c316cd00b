"""Shared by tests/test_gpu_trackpost.py and tools/trackpost_bench.py: prompt-shaped positive maps of the video datasets,
tie-free inputs, and the two reference chains of the video trackers restated line for line (uninext_vid.py:1224-1250
inference_mot, :1380-1415 inference_vis) up to the hand-over to tracker.match."""
import torch
import torchvision


def prompt_map(num_classes):
    """num_classes classes of 1 to 3 consecutive tokens, one separator token between classes (a class-name prompt)."""
    pmap, t = {}, 1
    for c in range(num_classes):
        n = 1 + (c % 5 == 2) + (c % 7 == 4)
        pmap[c + 1] = list(range(t, t + n))
        t += n + 1
    assert t <= 256
    return pmap


MAPS = {"ytvis": lambda: prompt_map(40), "ovis": lambda: prompt_map(25), "bdd": lambda: prompt_map(8)}


def make_inputs(B, Q, pmap, T=256, iou=True, seed=0, layout="random", logit_shift=0.0, iou_shift=0.0, device="cuda"):
    """box_cls [B, Q, T], box_pred [B, Q, 4], iou_pred [B, Q, 1] or None.  Every token of class c carries the same value
    k * 2^-16 + logit_shift, k distinct per (query, class): the class mean is exact and the scores tie-free."""
    g = torch.Generator().manual_seed(seed)
    box_cls = torch.rand(B, Q, T, generator=g) * 8 - 4
    C = len(pmap)
    for b in range(B):
        k = torch.randperm(1 << 19, generator=g)[:Q * C].reshape(Q, C) - (1 << 18)
        vals = k.float() * 2.0 ** -16 + logit_shift
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
    iou_pred = torch.randn(B, Q, 1, generator=g) * 2 + iou_shift if iou else None
    to = lambda x: None if x is None else x.to(device)
    return to(box_cls), to(box_pred), to(iou_pred)


# ---- the reference chains -------------------------------------------------------------------------------------------
def convert_grounding_to_od_logits(logits, num_classes, positive_map, score_agg="MEAN"):
    """uninext_vid.py's copy of uninext_img.py:598-613."""
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


def mot_chain(logits, output_boxes, output_iou, positive_map_label_to_token, ori_size, inference_select_thres):
    """uninext_vid.py:1227-1249 for one frame: (indices, det_bboxes, det_labels).  output_boxes is scaled in place, as
    the reference does: pass a copy."""
    num_classes = len(positive_map_label_to_token)
    logits = convert_grounding_to_od_logits(logits.unsqueeze(0), num_classes, positive_map_label_to_token)
    logits = logits[0]
    scores = logits.sigmoid()  #[300,42]
    if output_iou is not None:
        scores = torch.sqrt(scores * output_iou.sigmoid())
    max_score, output_labels = torch.max(scores,1)
    indices = torch.nonzero(max_score>inference_select_thres, as_tuple=False).squeeze(1)
    if len(indices) == 0:
        topkv, indices_top1 = torch.topk(scores.cpu().detach().max(1)[0],k=1)
        indices_top1 = indices_top1[torch.argmax(topkv)]
        indices = [indices_top1.tolist()]
    else:
        nms_scores,idxs = torch.max(scores[indices],1)
        boxes_before_nms = box_cxcywh_to_xyxy(output_boxes[indices])
        keep_indices = torchvision.ops.batched_nms(boxes_before_nms,nms_scores,idxs,0.7) #.tolist()
        indices = indices[keep_indices]
    box_score = torch.max(scores[indices],1)[0]
    # [0, 1] -> real coordinates
    output_boxes[:, 0::2] *= ori_size[1]
    output_boxes[:, 1::2] *= ori_size[0]
    det_bboxes = torch.cat([box_cxcywh_to_xyxy(output_boxes[indices]),box_score.unsqueeze(1)],dim=1)
    det_labels = torch.argmax(scores[indices],dim=1)
    return indices, det_bboxes, det_labels


def vis_chain(logits, output_boxes, output_iou, positive_map_label_to_token, inference_select_thres):
    """uninext_vid.py:1385-1412 for one frame: (indices, det_bboxes, det_labels)."""
    num_classes = len(positive_map_label_to_token)
    logits = convert_grounding_to_od_logits(logits.unsqueeze(0), num_classes, positive_map_label_to_token)
    logits = logits[0]
    if output_iou is not None:
        scores = torch.sqrt(logits.sigmoid() * output_iou.sigmoid()).cpu().detach()  #[300,42]
        max_score, _ = torch.max(torch.sqrt(logits.sigmoid() * output_iou.sigmoid()),1)
    else:
        scores = logits.sigmoid().cpu().detach()  #[300,42]
        max_score, _ = torch.max(logits.sigmoid(),1)
    indices = torch.nonzero(max_score>inference_select_thres, as_tuple=False).squeeze(1)
    if len(indices) == 0:
        topkv, indices_top1 = torch.topk(scores.max(1)[0],k=1)
        indices_top1 = indices_top1[torch.argmax(topkv)]
        indices = [indices_top1.tolist()]
    else:
        if output_iou is not None:
            nms_scores,idxs = torch.max(torch.sqrt(logits.sigmoid() * output_iou.sigmoid())[indices],1)
        else:
            nms_scores,idxs = torch.max(logits.sigmoid()[indices],1)
        boxes_before_nms = box_cxcywh_to_xyxy(output_boxes[indices])
        keep_indices = torchvision.ops.batched_nms(boxes_before_nms,nms_scores,idxs,0.9)#.tolist()
        indices = indices[keep_indices]
    if output_iou is not None:
        box_score = torch.max(torch.sqrt(logits.sigmoid() * output_iou.sigmoid())[indices],1)[0]
        det_labels = torch.argmax(torch.sqrt(logits.sigmoid() * output_iou.sigmoid())[indices],dim=1)
    else:
        box_score = torch.max(logits.sigmoid()[indices],1)[0]
        det_labels = torch.argmax(logits.sigmoid()[indices],dim=1)
    det_bboxes = torch.cat([output_boxes[indices],box_score.unsqueeze(1)],dim=1)
    return indices, det_bboxes, det_labels


def chain(path, box_cls, box_pred, pmap, iou_pred, score_thres, ori_sizes=None):
    """Both chains per frame b: [dict(query, scores, labels, boxes)], the boxes as the tracker receives them."""
    out = []
    for b in range(box_cls.shape[0]):
        iou = None if iou_pred is None else iou_pred[b]
        if path == "mot":
            idx, det, lab = mot_chain(box_cls[b], box_pred[b].clone(), iou, pmap, ori_sizes[b], score_thres)
        else:
            idx, det, lab = vis_chain(box_cls[b], box_pred[b], iou, pmap, score_thres)
        out.append(dict(query=torch.as_tensor(idx, device=box_cls.device).long().reshape(-1), scores=det[:, 4],
                        labels=lab, boxes=det[:, :4]))
    return out
