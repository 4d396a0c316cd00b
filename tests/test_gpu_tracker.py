"""GPU tests of the IDOL tracker's association step (IDOLTracker, msda_idol_match_f32, DESIGN.md section 3.18): the
reference's goldens through both entry points, large random sequences against the restatement of tests/tracker_case.py
run on CUDA, the binarisation and IoU predicates bit for bit, the launch count, no host synchronisation, and the
capacity overflow."""
import os

import numpy as np
import pytest
import torch

from tests import tracker_case as tc

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tracker")


def _tracker(flags=(True, True, True), **over):
    from uninext_b200.modules.tracker import IDOLTracker
    return IDOLTracker(**tc.settings(flags, **over))


def _dets(scores, q, perm):
    """A one-frame TrackDetections whose rows sit at query perm[r] of Q = q queries."""
    from uninext_b200.modules.detection_postprocess import TrackDetections
    n = scores.shape[0]
    sc = torch.zeros(1, q, device="cuda")
    sc[0, :n] = scores.cuda()
    qi = torch.full((1, q), -1, dtype=torch.int32, device="cuda")
    qi[0, :n] = perm[:n].to(torch.int32).cuda()
    return TrackDetections(sc, torch.zeros(1, q, dtype=torch.int32, device="cuda"), torch.zeros(1, q, 4, device="cuda"),
                           qi, torch.tensor([n], dtype=torch.int32, device="cuda"))


def _selected_inputs(scores, masks, embeds, seed=0):
    """The frame's rows scattered over Q = n + 5 queries (at most 1024): (dets, 0, pred_masks [1, Q, 1, h, w],
    pred_inst_embed), match_selected's arguments before frame_id."""
    n = scores.shape[0]
    q = min(n + 5, 1024)
    perm = torch.randperm(q, generator=torch.Generator().manual_seed(seed))
    pm = torch.randn(1, q, *masks.shape[1:]) * 4
    pe = torch.randn(1, q, embeds.shape[1])
    pm[0, perm[:n]] = masks
    pe[0, perm[:n]] = embeds
    return _dets(scores, q, perm), 0, pm.cuda(), pe.cuda()


@pytest.mark.parametrize("flag_index", range(len(tc.FLAG_SETS)))
def test_golden_sequences_through_match_and_match_selected(flag_index):
    flags = tc.FLAG_SETS[flag_index]
    name = "lm{}_fw{}_tw{}".format(*(int(x) for x in flags))
    z = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    seq = tc.golden_sequence(flag_index)
    assert str(z["checksum"]) == tc.checksum(seq)
    a, b = _tracker(flags), _tracker(flags)
    for f, (scores, masks, embeds) in enumerate(seq):
        n = scores.shape[0]
        bboxes = torch.cat((torch.rand(n, 4), scores[:, None]), 1).cuda()
        labels = torch.arange(n).cuda()
        indices = [3 * r + 7 for r in range(n)]
        ob, ol, ids, idx = a.match(bboxes, labels, masks.cuda(), embeds.cuda(), f, indices)
        keep = z[f"{f}/keep"].tolist()
        assert ids.dtype == torch.int64 and not ids.is_cuda
        assert ids.tolist() == z[f"{f}/ids"].tolist(), f
        assert idx == z[f"{f}/indices"].tolist() and ol.tolist() == keep and torch.equal(ob, bboxes[keep])
        res = b.match_selected(*_selected_inputs(scores, masks, embeds, seed=f), f)
        rows, tids = b.read(res)
        got = res.ids.cpu()[:n].tolist()
        assert [r for r in range(n) if got[r] != -3] == keep
        assert [got[r] for r in keep] == z[f"{f}/ids"].tolist()
        assert rows == [r for r in keep if got[r] > -1] and tids == [got[r] for r in rows]
        for tr in (a, b):
            st = tr.tracklets()
            assert sorted(st) == z[f"{f}/track_ids"].tolist() and tr.num_tracklets == a.num_tracklets
            for c, k in enumerate(sorted(st)):
                v = st[k]
                assert v["last_frame"] == z[f"{f}/last_frame"][c] and v["exist_frame"] == z[f"{f}/exist_frame"][c]
                ln = int(z[f"{f}/ring_len"][c])
                scale = float(np.abs(z[f"{f}/embed"]).max())
                assert v["long_embed"].shape[0] == ln
                np.testing.assert_allclose(v["embed"].numpy(), z[f"{f}/embed"][c], rtol=0, atol=1e-5 * scale)
                np.testing.assert_allclose(v["long_embed"].numpy(), z[f"{f}/long_embed"][c, :ln], rtol=0,
                                           atol=1e-5 * scale)
                np.testing.assert_allclose(v["long_score"].numpy(), z[f"{f}/long_score"][c, :ln], rtol=0, atol=1e-6)


# (n, h, w, flags, seed): YTVIS-sized and OVIS-sized masks
RANDOM_CASES = [(1024, 120, 216, (True, True, True), 1), (700, 180, 320, (False, True, False), 2),
                (250, 120, 216, (False, False, False), 3), (1024, 180, 320, (True, False, False), 4),
                (100, 180, 320, (True, True, True), 5)]


@pytest.mark.parametrize("n,h,w,flags,seed", RANDOM_CASES)
def test_random_sequences_match_the_restatement_on_cuda(n, h, w, flags, seed):
    seq = tc.random_sequence(seed, n, h, w)
    ref = tc.Restated(**tc.settings(flags))
    tr = _tracker(flags)
    for f, (scores, masks, embeds) in enumerate(seq):
        keep, want = ref.step(scores.cuda(), masks[:, 0].cuda(), embeds.cuda(), f)
        res = tr.match_selected(*_selected_inputs(scores, masks, embeds, seed=seed * 100 + f), f)
        rows, _ = tr.read(res)
        got = res.ids.cpu()[:scores.shape[0]].tolist()
        assert [r for r in range(len(got)) if got[r] != -3] == keep, f
        assert [got[r] for r in keep] == want, f
        assert sorted(tr.tracklets()) == sorted(ref.tracks)
    assert min(ref.margins) >= 1e-4, f"the generator left a decision within {min(ref.margins):.2e} of flipping"


def _singletons(values, h=40, w=72):
    """Row 0 empty, then one row per value: the value at its own pixel, -10 elsewhere."""
    n = len(values) + 1
    m = torch.full((n, 1, h * w), -10.0)
    m[torch.arange(1, n), 0, torch.arange(len(values))] = values
    return m.reshape(n, 1, h, w)


def test_binarisation_is_torch_cuda_sigmoid_bit_for_bit():
    """A row whose one pixel is on is kept (IoU 0 with the others); rows with no pixel on have IoU 1 with the empty
    row 0 and are removed.  So the keep set shows every bit."""
    tiny = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, 5.96e-8, -5.96e-8, 6e-8, 1.2e-7,
                         -1.2e-7, 1e-10, float("inf"), float("-inf"), float("nan")])
    x = torch.cat((tiny, torch.linspace(-2e-7, 2e-7, 4001), torch.linspace(-1e-3, 1e-3, 2001),
                   torch.linspace(-20, 20, 2001)))
    x = torch.cat((x, torch.nextafter(x, torch.tensor(1.0)), torch.nextafter(x, torch.tensor(-1.0))))
    want_all = (x.cuda().sigmoid() > 0.5).cpu()
    tr = _tracker()
    for c in range(0, x.numel(), 1000):
        v = x[c:c + 1000]
        m = _singletons(v)
        n = m.shape[0]
        scores = torch.full((n,), 0.1005)                       # below every score threshold: no tracklet
        res = tr.match_selected(*_selected_inputs(scores, m, torch.zeros(n, 8)), 0)
        tr.read(res)
        ids = res.ids.cpu()[:n]
        pos = torch.arange(n)[1:]
        got = ids[1:] != -3
        assert torch.equal(got, want_all[c:c + 1000]), [float(v[i]) for i in torch.nonzero(got != want_all[c:c + 1000])[:5]]
        assert ids[0] != -3 and pos.numel() == v.numel()


def _frame_of_sets(sets, hw=(180, 320)):
    h, w = hw
    n = len(sets)
    m = torch.full((n, h * w), -5.0)
    for r, s in enumerate(sets):
        m[r, torch.as_tensor(s, dtype=torch.long)] = 5.0
    return m.reshape(n, 1, h, w)


def test_iou_predicates_equal_the_fp32_formula_from_int64_counts():
    g = torch.Generator().manual_seed(7)
    h, w = 120, 216
    # exact ties: IoU 4096 / 8192 = 0.5 (not > 0.5: kept) and fp32(1000 / 20000) = fp32(0.05) (not < 0.05: stays -2)
    sets = [list(range(0, 8192)), list(range(0, 4096)), list(range(10000, 30000)), list(range(10000, 11000))]
    m = _frame_of_sets(sets)
    scores = torch.tensor([0.1505, 0.1405, 0.1305, 0.1205])
    tr = _tracker()
    res = tr.match_selected(*_selected_inputs(scores, m, torch.zeros(4, 8)), 0)
    tr.read(res)
    assert res.ids.cpu()[:4].tolist() == [-1, -2, -1, -2]
    # random overlapping masks: keep sets and backdrops equal the restatement's fp32 formula exactly
    for seed in range(3):
        n = 300
        base = torch.rand(24, h * w, generator=g) < 0.3
        pick = torch.randint(0, 24, (n,), generator=g)
        noise = torch.rand(n, h * w, generator=g) < torch.rand(n, 1, generator=g) * 0.6
        on = base[pick] ^ noise
        logits = torch.where(on, 3.0, -3.0).reshape(n, 1, h, w)
        scores = torch.sort(torch.rand(n, generator=g) * 0.15 + 0.02, descending=True).values
        ref = tc.Restated(**tc.settings((True, True, True)))
        keep, want = ref.step(scores, logits[:, 0].cuda(), torch.zeros(n, 8).cuda(), 0)
        tr = _tracker()
        res = tr.match_selected(*_selected_inputs(scores, logits, torch.zeros(n, 8), seed=seed), 0)
        tr.read(res)
        got = res.ids.cpu()[:n].tolist()
        assert [r for r in range(n) if got[r] != -3] == keep
        assert [got[r] for r in keep] == want
        assert -1 in want and -2 in want and len(keep) < n


def test_launch_count_is_constant_per_call():
    from uninext_b200 import _cabi
    from uninext_b200.modules.tracker import LAUNCHES
    lib = _cabi.load()
    tr = _tracker()
    for f, (scores, masks, embeds) in enumerate(tc.golden_sequence(0)):
        args = _selected_inputs(scores, masks, embeds)
        torch.cuda.synchronize()
        before = lib.msda_launch_count()
        res = tr.match_selected(*args, f)
        assert lib.msda_launch_count() - before == LAUNCHES == 8
        tr.read(res)


def test_second_match_selected_does_not_synchronise():
    seq = tc.golden_sequence(1)
    tr = _tracker()
    first = _selected_inputs(*seq[0])
    second = _selected_inputs(*seq[1])
    tr.read(tr.match_selected(*first, 0))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = tr.match_selected(*second, 1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    rows, ids = tr.read(res)
    assert ids and all(i >= 0 for i in ids)


def test_overflow_raises_and_keeps_no_partial_state():
    world = tc.World(12, 40, 72, 16, seed=3)
    dets = [(o, "full", 0.9005 - 0.01 * o, None) for o in range(9)]
    scores, masks, embeds = world.frame(dets)
    tr = _tracker(max_tracklets=8)
    res = tr.match_selected(*_selected_inputs(scores, masks, embeds), 0)
    with pytest.raises(RuntimeError, match="max_tracklets=8"):
        tr.read(res)
    assert tr.tracklets() == {} and tr.num_tracklets == 0
    small = world.frame(dets[:2])
    with pytest.raises(RuntimeError, match="max_tracklets"):
        tr.match(torch.cat((torch.rand(2, 4), small[0][:, None]), 1).cuda(), torch.zeros(2).cuda(), small[1].cuda(),
                 small[2].cuda(), 1, [0, 1])
