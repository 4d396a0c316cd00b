"""GPU tests (-m gpu) of mask pasting (uninext_b200/modules/mask_postprocess.py, kernel csrc/msda_maskpaste.cuh) against
the reference's torch chain, restated below as the reference writes it: binary masks equal everywhere except pixels whose
reference probability lies within 1e-6 of the threshold, probabilities within 1e-6, every output element written, one
launch per call, no allocation beyond the output, CUDA-graph capture, and an output past 2^31 elements."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.modules.mask_postprocess import paste_masks

NEAR = 1e-6


def chain_image(mask_pred_i, image_size, output_size, mask_stride, mask_thres):
    """uninext_img.py:474-479, then segmentation_postprocess (models/ddetrs.py:1060-1064)."""
    N, C, H, W = mask_pred_i.shape
    mask = F.interpolate(mask_pred_i, size=(H*mask_stride, W*mask_stride), mode='bilinear', align_corners=False)
    mask = mask.sigmoid() > mask_thres
    mask = mask[:,:,:image_size[0],:image_size[1]]
    mask = F.interpolate(mask.float(), size=(output_size[0], output_size[1]), mode='nearest')
    mask = mask.squeeze(1).byte()
    return mask


def chain_video(track_masks, image_size, ori_size, output_h, output_w):
    """uninext_vid.py:620-622 (probabilities; :1264-1266 and :1335-1337 then take `> 0.5`)."""
    track_masks = F.interpolate(track_masks,  size=(output_h*4, output_w*4) ,mode="bilinear", align_corners=False).sigmoid()
    track_masks = track_masks[:, :, :image_size[0],:image_size[1]] # crop the padding area
    track_masks = F.interpolate(track_masks, size=(ori_size[0], ori_size[1]), mode='nearest') # (1, 1, H, W)
    return track_masks[:, 0]


def chain_probs(logits4, image_size, output_size, stride):
    """The video chain at any stride (the reference's is 4)."""
    n, c, h, w = logits4.shape
    m = F.interpolate(logits4, size=(h * stride, w * stride), mode="bilinear", align_corners=False).sigmoid()
    m = m[:, :, :image_size[0], :image_size[1]]
    return F.interpolate(m, size=(output_size[0], output_size[1]), mode="nearest")[:, 0]


def make_logits(i, hs, ws, seed=0, dtype=torch.float32):
    """Logits spanning +-30, ~5% exactly 0, plus a 2x2 block of zeros (interpolates to exactly 0: p == 0.5)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(i, 1, hs, ws, generator=g) * 60 - 30
    x[torch.rand(i, 1, hs, ws, generator=g) < 0.05] = 0.0
    x[:, :, :2, :2] = 0.0
    x[:, :, hs // 2:, ws // 3:] *= 0.02              # a band near 0, where the threshold decisions are made
    return x.to("cuda", dtype)


# (I, Hs, Ws, stride, crop (h, w), output (H_out, W_out))
CASES = [
    (3, 200, 336, 4, (800, 1333), (480, 640)),        # downsampling, UNINEXT's padded 800x1344 input
    (3, 25, 42, 4, (97, 163), (250, 400)),            # upsampling, crop not a multiple of the stride
    (1, 1, 7, 4, (3, 25), (5, 50)),                   # Hs = 1
    (3, 9, 1, 4, (33, 2), (40, 3)),                   # Ws = 1
    (3, 10, 12, 4, (37, 45), (1, 1)),                 # 1x1 output
    (100, 200, 336, 4, (800, 1333), (480, 640)),
    (300, 50, 84, 4, (199, 333), (427, 641)),
    (5, 12, 20, 8, (90, 157), (120, 200)),            # stride 8
    (4, 13, 17, 3, (37, 50), (61, 77)),               # stride 3: scale 1/3 is not exact in fp32
    (2, 30, 40, 4, (120, 160), (120, 160)),           # output = crop (uninext_vid.py:1187-1192)
]


def _ids(c):
    return f"I{c[0]}_{c[1]}x{c[2]}_s{c[3]}_crop{c[4][0]}x{c[4][1]}_out{c[5][0]}x{c[5][1]}"


@pytest.mark.parametrize("case", CASES, ids=_ids)
@pytest.mark.parametrize("threshold", [0.5, 0.3])
def test_binary_matches_chain(case, threshold):
    i, hs, ws, stride, crop, outs = case
    x = make_logits(i, hs, ws, seed=i + hs)
    lib = _cabi.load()
    before = lib.msda_launch_count()
    got = paste_masks(x, crop, outs, stride, threshold)
    assert lib.msda_launch_count() == before + 1
    assert got.dtype == torch.bool and got.shape == (i, *outs)
    if stride == 4:
        want = chain_image(x, crop, outs, stride, threshold).bool()
    else:
        want = chain_probs(x, crop, outs, stride) > threshold
    p_ref = chain_probs(x, crop, outs, stride)
    near = (p_ref - threshold).abs() <= NEAR
    bad = (got != want) & ~near
    print(f"{_ids(case)} thr {threshold}: {int(near.sum())} of {near.numel()} pixels within {NEAR} of the threshold, "
          f"{int(((got != want) & near).sum())} of them differ")
    assert int(bad.sum()) == 0, f"{int(bad.sum())} pixels differ away from the threshold"


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_probabilities_match_chain(case):
    i, hs, ws, stride, crop, outs = case
    x = make_logits(i, hs, ws, seed=7 * i + ws)
    got = paste_masks(x, crop, outs, stride, threshold=None)
    assert got.dtype == torch.float32 and got.shape == (i, *outs)
    want = chain_video(x, crop, outs, hs, ws) if stride == 4 else chain_probs(x, crop, outs, stride)
    assert (got - want).abs().max().item() <= 1e-6
    if stride == 4:                                                   # uninext_vid.py:1264-1266: nearest, then > 0.5
        b = paste_masks(x, crop, outs, stride, 0.5)
        assert int(((b != (want > 0.5)) & ((want - 0.5).abs() > NEAR)).sum()) == 0


def test_input_forms_dtype_and_empty():
    x = make_logits(3, 25, 42, seed=3)
    a = paste_masks(x, (97, 163), (250, 400))
    assert torch.equal(a, paste_masks(x[:, 0], (97, 163), (250, 400)))
    xh = x.half()
    got = paste_masks(xh, (97, 163), (250, 400), threshold=None)
    want = chain_video(xh.float(), (97, 163), (250, 400), 25, 42)           # the chain's .float() of the input
    assert (got - want).abs().max().item() <= 1e-6
    lib = _cabi.load()
    before = lib.msda_launch_count()
    for thr, dt in ((0.5, torch.bool), (None, torch.float32)):
        e = paste_masks(x[:0], (97, 163), (250, 400), threshold=thr)
        assert e.shape == (0, 250, 400) and e.dtype == dt and e.is_cuda
    assert lib.msda_launch_count() == before


@pytest.mark.parametrize("binary", [1, 0])
@pytest.mark.parametrize("outs", [(427, 641), (480, 640)], ids=["scalar", "vector"])
def test_every_element_is_written(binary, outs):
    x = make_logits(5, 50, 84, seed=5)[:, 0].contiguous()
    if binary:
        out = torch.full((5, *outs), 0xAB, dtype=torch.uint8, device="cuda")
    else:
        out = torch.full((5, *outs), float("nan"), dtype=torch.float32, device="cuda")
    _cabi.call("msda_mask_paste_f32", x, 5, 50, 84, 4, 199, 333, outs[0], outs[1], 0.5, binary, out, device=x.device)
    if binary:
        assert bool(((out == 0) | (out == 1)).all())
        assert torch.equal(out.bool(), paste_masks(x, (199, 333), outs))
    else:
        assert bool(torch.isfinite(out).all()) and bool(((out >= 0) & (out <= 1)).all())


@pytest.mark.parametrize("threshold", [0.5, None])
def test_peak_allocation_is_the_output(threshold):
    x = make_logits(100, 200, 336, seed=11)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = paste_masks(x, (800, 1333), (480, 640), threshold=threshold)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - base
    assert torch.cuda.max_memory_allocated() - base == grown          # nothing beyond the output's block
    nbytes = out.numel() * out.element_size()
    del out
    same_size = torch.empty(nbytes, dtype=torch.uint8, device="cuda")   # what the caching allocator grants that many bytes
    assert torch.cuda.memory_allocated() - base == grown
    del same_size


def test_cuda_graph_capture_and_replay():
    x = make_logits(100, 200, 336, seed=13)
    eager_b = paste_masks(x, (800, 1333), (480, 640))
    eager_p = paste_masks(x, (800, 1333), (480, 640), threshold=None)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                         # warm-up on a side stream, as torch asks
        paste_masks(x, (800, 1333), (480, 640))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gb = paste_masks(x, (800, 1333), (480, 640))
        gp = paste_masks(x, (800, 1333), (480, 640), threshold=None)
    gb.zero_()
    gp.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gb, eager_b) and torch.equal(gp, eager_p)
    x.copy_(make_logits(100, 200, 336, seed=14))                      # new inputs, same graph
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gb, paste_masks(x, (800, 1333), (480, 640)))


def test_output_past_2_31_elements():
    """300 x 2160 x 3840 = 2.49e9 bytes: sampled rows of instances near the end, whose offsets pass 2^31, against the
    chain run on that instance alone."""
    i, hs, ws, crop, outs = 300, 200, 336, (800, 1333), (2160, 3840)
    x = make_logits(i, hs, ws, seed=17)
    got = paste_masks(x, crop, outs)
    assert got.numel() > 2 ** 31
    torch.cuda.synchronize()
    for k in (0, 150, 259, 299):
        want = chain_image(x[k:k + 1], crop, outs, 4, 0.5)[0].bool()
        p_ref = chain_probs(x[k:k + 1], crop, outs, 4)[0]
        for r in (0, 1, 1079, 2158, 2159):
            bad = (got[k, r] != want[r]) & ((p_ref[r] - 0.5).abs() > NEAR)
            assert int(bad.sum()) == 0, (k, r)
    del got
    torch.cuda.empty_cache()


def test_bad_arguments_raise():
    x = make_logits(2, 10, 12)
    with pytest.raises(ValueError):
        paste_masks(x, (41, 45), (10, 10))                             # crop taller than stride * Hs
    with pytest.raises(ValueError):
        paste_masks(x, (40, 45), (0, 10))
    with pytest.raises(ValueError):
        paste_masks(x.reshape(2, 2, 5, 12), (20, 45), (10, 10))
    lib = _cabi.load()
    assert lib.msda_mask_paste_f32(x.data_ptr(), 2, 10, 12, 4, 41, 45, 10, 10, 0.5, 1, x.data_ptr(), None) == -1
    assert lib.msda_mask_paste_f32(None, 2, 10, 12, 4, 40, 45, 10, 10, 0.5, 1, ctypes.c_void_p(x.data_ptr()), None) == -1
