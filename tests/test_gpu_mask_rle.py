"""GPU tests (-m gpu) of COCO run-length encoding (uninext_b200/modules/mask_postprocess.py: paste_masks_rle,
encode_masks_rle; kernels csrc/msda_maskrle.cuh).  encode_masks_rle is compared byte for byte with the restatement in
tests/coco_rle.py on paste_masks outputs and on edge masks; paste_masks_rle with encode_masks_rle(paste_masks(...)),
with no tolerance, since both evaluate pixels through the same device code.  Also: a 24000 x 24000 mask, offsets past
2^31, pycocotools when it is installed, fixed launch and synchronisation counts, and the peak allocation."""
import gc
import os
import warnings

import numpy as np
import pytest
import torch

from tests.coco_rle import encode_np
from tests.test_gpu_mask_paste import CASES, _ids, make_logits

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.modules.mask_postprocess import encode_masks_rle, paste_masks, paste_masks_rle

LAUNCHES = 7                                     # pass 1, cub's scan (2), pass 2, pass 3 (3)


def restated(masks):
    m = masks.cpu().numpy()
    return [encode_np(m[k]) for k in range(m.shape[0])]


def assert_same(got, want):
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g["size"] == w["size"], k
        assert g["counts"] == w["counts"], (k, g["counts"][:40], w["counts"][:40])


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_encode_of_pasted_masks_matches_restatement(case):
    i, hs, ws, stride, crop, outs = case
    m = paste_masks(make_logits(i, hs, ws, seed=i + hs), crop, outs, stride, 0.5)
    got = encode_masks_rle(m)
    assert_same(got, restated(m))
    assert all(isinstance(r["counts"], bytes) and r["size"] == list(outs) for r in got)


def _edge_masks():
    h, w = 37, 29
    z = torch.zeros(3, h, w, dtype=torch.bool)
    first, last = z.clone(), z.clone()
    first[:, 0, 0] = True
    last[:, -1, -1] = True
    cross = z.clone()                               # runs that run over column ends into the next column
    cross[0, h - 5:, 3] = True
    cross[0, :7, 4] = True
    cross[1, :, 10:13] = True
    cross[2, h - 1, :] = True
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    checker = ((yy + xx) % 2 == 0).expand(3, h, w).clone()
    return {"zeros": z, "ones": ~z, "first_pixel": first, "last_pixel": last, "cross_columns": cross,
            "checkerboard": checker, "checker_inverse": ~checker,
            "1x1_set": torch.ones(2, 1, 1, dtype=torch.bool), "1x1_clear": torch.zeros(2, 1, 1, dtype=torch.bool),
            "1xW": torch.rand(3, 1, 1000, generator=torch.Generator().manual_seed(1)) > 0.5,
            "Hx1": torch.rand(3, 1000, 1, generator=torch.Generator().manual_seed(2)) > 0.5,
            "checker_big": ((torch.arange(1080)[:, None] + torch.arange(1920)[None]) % 2 == 1).expand(4, 1080, 1920)
                           .clone()}


@pytest.mark.parametrize("name", list(_edge_masks()))
@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8])
def test_edge_masks(name, dtype):
    m = _edge_masks()[name].to(dtype)
    if dtype == torch.uint8:
        m = m * 7                                   # any nonzero byte is a set pixel
    assert_same(encode_masks_rle(m.cuda()), restated(m))


def test_known_answers():
    two = lambda rows: torch.tensor(rows, dtype=torch.bool, device="cuda")[None]
    assert encode_masks_rle(two([[0, 0], [0, 0]]))[0] == {"size": [2, 2], "counts": b"4"}
    assert encode_masks_rle(two([[1, 1], [1, 1]]))[0] == {"size": [2, 2], "counts": b"04"}
    assert encode_masks_rle(two([[0, 1], [1, 0]]))[0] == {"size": [2, 2], "counts": b"121"}


@pytest.mark.parametrize("offset", [1, 3, 5, 16])
@pytest.mark.parametrize("w", [64, 61])
def test_unaligned_views(offset, w):
    """Contiguous views whose storage starts 1..16 bytes into a buffer, with rows a multiple of 4 bytes or not."""
    i, h = 5, 70
    g = torch.Generator(device="cuda").manual_seed(offset + w)
    buf = (torch.rand(i * h * w + offset, device="cuda", generator=g) > 0.6).to(torch.uint8)
    m = buf[offset:].view(i, h, w)
    assert m.is_contiguous() and m.data_ptr() % 16 == offset % 16
    assert_same(encode_masks_rle(m), restated(m))
    assert_same(encode_masks_rle(m.view(torch.bool)), restated(m))


def test_non_contiguous_input():
    m = torch.rand(6, 50, 40, device="cuda") > 0.5
    assert_same(encode_masks_rle(m[::2, :, 5:]), restated(m[::2, :, 5:]))
    assert_same(encode_masks_rle(m.transpose(1, 2)), restated(m.transpose(1, 2)))


# (I, Hs, Ws, stride, crop, output)
FUSED = [
    (1, 25, 42, 4, (97, 163), (250, 400)),          # upsampled, crop not a multiple of the stride
    (100, 200, 336, 4, (800, 1333), (480, 640)),   # downsampled, COCO evaluation
    (300, 50, 84, 4, (199, 333), (427, 641)),
    (5, 12, 20, 8, (90, 157), (120, 200)),          # stride 8
    (4, 13, 17, 3, (37, 50), (61, 77)),             # stride 3
    (3, 9, 1, 4, (33, 2), (40, 3)),
    (3, 10, 12, 4, (37, 45), (1, 1)),
    (10, 90, 160, 4, (360, 640), (720, 1280)),      # video tracks
]


@pytest.mark.parametrize("case", FUSED, ids=_ids)
@pytest.mark.parametrize("threshold", [0.5, 0.3])
def test_fused_equals_paste_then_encode(case, threshold):
    i, hs, ws, stride, crop, outs = case
    x = make_logits(i, hs, ws, seed=3 * i + ws)
    got = paste_masks_rle(x, crop, outs, stride, threshold)
    assert_same(got, encode_masks_rle(paste_masks(x, crop, outs, stride, threshold)))


def test_empty_and_input_forms():
    x = make_logits(3, 25, 42, seed=3)
    lib = _cabi.load()
    before = lib.msda_launch_count()
    assert paste_masks_rle(x[:0], (97, 163), (250, 400)) == []
    assert encode_masks_rle(torch.zeros(0, 20, 30, dtype=torch.bool, device="cuda")) == []
    assert lib.msda_launch_count() == before
    a = paste_masks_rle(x, (97, 163), (250, 400))
    assert a == paste_masks_rle(x[:, 0], (97, 163), (250, 400))
    assert paste_masks_rle(x.half(), (97, 163), (250, 400)) == encode_masks_rle(paste_masks(x.half(), (97, 163),
                                                                                            (250, 400)))


def test_24000_square_constant_mask():
    """One instance of constant negative logits pasted to 24000 x 24000: one run of 576e6 zeros, the 7-character case,
    and a column scan over 24000 columns, without a full-size mask on the host."""
    x = torch.full((1, 1, 1, 1), -3.0, device="cuda")
    got = paste_masks_rle(x, (4, 4), (24000, 24000))
    assert got == [{"size": [24000, 24000], "counts": b"PPTZUa0"}]
    ones = paste_masks_rle(-x, (4, 4), (24000, 24000))
    assert ones == [{"size": [24000, 24000], "counts": b"0PPTZUa0"}]


def test_offsets_past_2_31():
    """300 x 2160 x 3840 = 2.49e9 pixels: instances near the end, whose pixel offsets pass 2^31, against the same instance
    pasted and encoded alone."""
    i, hs, ws, crop, outs = 300, 200, 336, (800, 1333), (2160, 3840)
    x = make_logits(i, hs, ws, seed=17)
    fused = paste_masks_rle(x, crop, outs)
    m = paste_masks(x, crop, outs)
    assert m.numel() > 2 ** 31
    from_masks = encode_masks_rle(m)
    del m
    torch.cuda.empty_cache()
    for k in (0, 150, 259, 298, 299):
        alone = paste_masks(x[k:k + 1], crop, outs)
        want = restated(alone)[0]
        assert fused[k] == want and from_masks[k] == want, k


def test_pycocotools_agrees():
    mask_util = pytest.importorskip("pycocotools.mask")
    x = make_logits(20, 50, 84, seed=21)
    m = paste_masks(x, (199, 333), (427, 641))
    got = paste_masks_rle(x, (199, 333), (427, 641))
    host = m.cpu().numpy().astype(np.uint8)
    for k in range(host.shape[0]):
        want = mask_util.encode(np.asfortranarray(host[k][:, :, None]))[0]
        assert got[k]["size"] == list(want["size"]) and got[k]["counts"] == want["counts"], k
    edge = _edge_masks()
    for name in ("zeros", "ones", "first_pixel", "last_pixel", "checkerboard"):
        e = edge[name].to(torch.uint8).numpy()
        want = [mask_util.encode(np.asfortranarray(e[k][:, :, None]))[0] for k in range(e.shape[0])]
        got = encode_masks_rle(edge[name].cuda())
        assert [g["counts"] for g in got] == [w["counts"] for w in want], name


@pytest.mark.parametrize("shape", [(1, 25, 42, (97, 163), (250, 400)), (300, 50, 84, (199, 333), (427, 641)),
                                   (2, 200, 336, (800, 1333), (1080, 1920))])
def test_launches_per_call_are_fixed(shape):
    i, hs, ws, crop, outs = shape
    x = make_logits(i, hs, ws, seed=5)
    lib = _cabi.load()
    before = lib.msda_launch_count()
    paste_masks_rle(x, crop, outs)
    assert lib.msda_launch_count() - before == LAUNCHES
    m = paste_masks(x, crop, outs)
    before = lib.msda_launch_count()
    encode_masks_rle(m)
    assert lib.msda_launch_count() - before == LAUNCHES


def _syncs(fn):
    """The synchronising CUDA operations torch reports while fn runs, as 'file:line'."""
    gc.collect()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return [f"{os.path.basename(w.filename)}:{w.lineno}" for w in caught
            if "called a synchronizing CUDA operation" in str(w.message)]


@pytest.mark.parametrize("i", [1, 300])
def test_two_host_synchronisations(i):
    x = make_logits(i, 50, 84, seed=9)
    m = paste_masks(x, (199, 333), (427, 641))
    paste_masks_rle(x, (199, 333), (427, 641))                   # warm-up: first-call work is not part of the count
    encode_masks_rle(m)
    fused, masks = _syncs(lambda: paste_masks_rle(x, (199, 333), (427, 641))), _syncs(lambda: encode_masks_rle(m))
    assert len(fused) == 2 and len(masks) == 2, (fused, masks)


def _peak(fn):
    """The peak of the bytes requested from the caching allocator during fn, above what was requested before it (the
    allocator may hand out a cached block up to 1 MiB larger than asked for, which says nothing about the call)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_stats()["requested_bytes.all.current"]
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.memory_stats()["requested_bytes.all.peak"] - base, out


def _bound(i, h, w, out):
    """The workspace (bitmap, column counts, scan storage), 4 B per boundary, 7 B per count and the [I + 1] offsets."""
    import ctypes
    n = ctypes.c_int64(0)
    _cabi.check(_cabi.load().msda_mask_rle_workspace(i, h, w, ctypes.byref(n)), "msda_mask_rle_workspace")
    counts = sum(len(_decode_len(r["counts"])) for r in out)
    bitmap = i * ((h + 31) // 32) * w * 4
    return n.value + 4 * (counts - i) + 8 * (i + 1) + 7 * counts, bitmap


def _decode_len(s):
    """The values of an RLE string (their number is the number of counts)."""
    vals, p = [], 0
    while p < len(s):
        while s[p] - 48 & 0x20:
            p += 1
        p += 1
        vals.append(p)
    return vals


@pytest.mark.parametrize("case", [c for c in FUSED if c[0] >= 10], ids=_ids)
def test_peak_allocation_on_random_logits(case):
    i, hs, ws, stride, crop, outs = case
    x = make_logits(i, hs, ws, seed=i)
    paste_masks_rle(x, crop, outs, stride)
    peak, out = _peak(lambda: paste_masks_rle(x, crop, outs, stride))
    bound, _ = _bound(i, *outs, out)
    print(f"{_ids(case)}: peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB")
    assert peak <= bound


def blob_logits(i, hs, ws, seed=0):
    """Mask-like logits: a few smooth blobs per instance, positive inside, negative outside."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(hs, dtype=torch.float32), torch.arange(ws, dtype=torch.float32),
                            indexing="ij")
    out = torch.full((i, hs, ws), -8.0)
    for k in range(i):
        for _ in range(int(torch.randint(1, 4, (1,), generator=g))):
            cy, cx = float(torch.rand(1, generator=g)) * hs, float(torch.rand(1, generator=g)) * ws
            r = 3 + float(torch.rand(1, generator=g)) * hs / 4
            out[k] = torch.maximum(out[k], 8.0 * (1 - ((yy - cy) ** 2 + (xx - cx) ** 2) / r ** 2))
    return out.cuda()


def test_peak_on_mask_like_logits_is_a_quarter_of_the_byte_mask():
    i, outs = 300, (1080, 1920)
    x = blob_logits(i, 200, 336, seed=4)
    paste_masks_rle(x, (800, 1333), outs)
    peak, out = _peak(lambda: paste_masks_rle(x, (800, 1333), outs))
    bound, bitmap = _bound(i, *outs, out)
    byte_mask = i * outs[0] * outs[1]
    print(f"mask-like 300 -> 1080x1920: peak {peak / 2**20:.1f} MiB, bitmap {bitmap / 2**20:.1f} MiB, "
          f"byte mask {byte_mask / 2**20:.1f} MiB")
    assert peak <= bound and peak < 0.25 * byte_mask
    assert_same(out, encode_masks_rle(paste_masks(x, (800, 1333), outs)))
