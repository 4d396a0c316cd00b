"""The encoder's input preparation, the pyramid geometry and the two-stage selection against plain references on ragged
pyramids: levels smaller than one 32-position tile, H * W one above or below a multiple of 32 or not a multiple of 4,
1 x W, H x 1 and 1 x 1 levels, L = 1 and L = 8 (msda_flatten.h's largest), N = 1 and N = 3, channel counts around the
32-channel tiles, and padding masks that are not rectangles: random interior holes, a first row and a first column
unlike the interior (get_valid_ratio reads only those), and one image whose coarsest level is all padding.

    flatten_levels          forward and the input gradients bit for bit the reference's torch chain, grad_level_embed
                            within 1e-6 of scale of the fp64 sum, every gradient subset; through the C ABI every output
                            element written and nothing around it
    valid ratios            bit for bit get_valid_ratio on CUDA, a 0 ratio for the fully padded level
    get_reference_points    bit for bit the torch chain on CUDA (inf and NaN where ratios are 0), fp64 within 4 ulps
    proposals               keep and +inf exact, finite values within 1e-6 of scale of the CPU chain and of fp64
    get_sine_pos_embed      forward and backward against fp64 autograd of the formula; odd widths raise
    two_stage_select        restated_fp64 at S = 1, 63, 64, 65 and past 2048, N = 1 and 5, k on both sides of the
                            on-chip sort, one image all padding; bit-identical on a repeated run

The tests without the gpu marker check the fixtures and the fp64 restatements on the CPU."""
import ctypes
import math

import pytest
import torch

from tests.test_gpu_dino_transformer import reference_chain
from uninext_b200.modules.deformable_transformer import (gen_encoder_output_proposals, get_reference_points,
                                                         get_sine_pos_embed)

DEV = "cuda"
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


# ---- the ragged pyramids ---------------------------------------------------------------------------------------------
# (shapes, N).  l8: 37 x 41 is wider and taller than a warp's stride, 9 x 7 = 63 (% 32 = 31), 1 x 33 (% 32 = 1),
# 5 x 1, 3 x 6 = 18 (< 32, % 4 = 2), 1 x 1, 2 x 5, 1 x 3.  l6 has the same kinds of levels at L = 6, N = 1.
CASES = {
    "l8_n3": (((37, 41), (9, 7), (1, 33), (5, 1), (3, 6), (1, 1), (2, 5), (1, 3)), 3),
    "l6_n1": (((34, 40), (23, 25), (11, 3), (7, 1), (1, 29), (1, 1)), 1),
    "l1_n3": (((33, 35),), 3),
    "l1_1x1_n1": (((1, 1),), 1),
}


def make_masks(shapes, n, seed=0):
    """[N, H, W] bool per level, True = padded.  Per image and level: a valid top-left rectangle, interior positions
    flipped at random (holes in it, islands outside), then a first row and a first column drawn on their own; image 0
    keeps its first position, so that a level has a nonzero ratio; with L > 1 the last image's coarsest level is all
    padding."""
    g = torch.Generator().manual_seed(seed)
    masks = []
    for lvl, (h, w) in enumerate(shapes):
        m = torch.zeros(n, h, w, dtype=torch.bool)
        for b in range(n):
            vh, vw = int(torch.randint(1, h + 1, (1,), generator=g)), int(torch.randint(1, w + 1, (1,), generator=g))
            m[b, vh:, :] = True
            m[b, :, vw:] = True
            m[b, 1:, 1:] ^= torch.rand(h - 1, w - 1, generator=g) < 0.2
            m[b, 0, :] = torch.rand(w, generator=g) < 0.3
            m[b, :, 0] = torch.rand(h, generator=g) < 0.3
            m[0, 0, 0] = False
            if len(shapes) > 1 and b == n - 1 and lvl == len(shapes) - 1:
                m[b] = True
        masks.append(m)
    return masks


def flat_mask(masks):
    return torch.cat([m.flatten(1) for m in masks], 1)


def pyramid_inputs(name, c, le_rows=None, seed=0):
    """(shapes, srcs, masks, pos_embeds, level_embed) on the GPU; level_embed has le_rows >= L rows."""
    shapes, n = CASES[name]
    g = torch.Generator().manual_seed(seed)
    srcs = [torch.randn(n, c, h, w, generator=g).to(DEV) for h, w in shapes]
    pos = [torch.randn(n, c, h, w, generator=g).to(DEV) for h, w in shapes]
    le = torch.randn(le_rows or len(shapes), c, generator=g).to(DEV)
    return shapes, srcs, [m.to(DEV) for m in make_masks(shapes, n, seed)], pos, le


def starts_of(shapes):
    out = [0]
    for h, w in shapes:
        out.append(out[-1] + h * w)
    return out


# ---- fp64 restatements -----------------------------------------------------------------------------------------------
def valid_counts64(masks):
    """[N, L, 2] fp64 (valid W, valid H): the unpadded positions of each level's first row and first column."""
    return torch.stack([torch.stack(((~m[:, 0, :]).sum(1), (~m[:, :, 0]).sum(1)), -1) for m in masks], 1).double()


def pixel_grid64(shapes, device):
    """Per flattened position: (x + 0.5, y + 0.5), (W, H) and the level, fp64."""
    xy, wh, lvl = [], [], []
    for i, (h, w) in enumerate(shapes):
        yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
        xy.append(torch.stack((xx.flatten(), yy.flatten()), -1) + 0.5)
        wh.append(torch.tensor([[float(w), float(h)]], dtype=torch.float64).expand(h * w, 2))
        lvl.append(torch.full((h * w,), i, dtype=torch.long))
    return torch.cat(xy).to(device), torch.cat(wh).to(device), torch.cat(lvl).to(device)


def ref_points64(shapes, vr):
    """get_reference_points (deformable_transformer_dino.py:289-301) in fp64: [N, S, L, 2]."""
    xy, wh, lvl = pixel_grid64(shapes, vr.device)
    vr = vr.double()
    return (xy[None] / (vr[:, lvl] * wh[None]))[:, :, None] * vr[:, None]


def proposals64(shapes, masks, base_scale):
    """The geometry of gen_encoder_output_proposals in fp64, without the drop: logit of ((x + .5) / valid W,
    (y + .5) / valid H, s 2^l, s 2^l) -> [N, S, 4]."""
    xy, _, lvl = pixel_grid64(shapes, masks[0].device)
    counts = valid_counts64(masks)
    size = (base_scale * 2.0 ** lvl.double())[None, :, None].expand(counts.shape[0], -1, 2)
    p = torch.cat((xy[None] / counts[:, lvl], size), -1)
    return torch.log(p / (1 - p))


def sine64(pos, F, temperature, exchange_xy):
    """get_sine_pos_embed's documented formula in fp64: [R, n] -> [R, n * F]; component k, feature j = sin (j even) or
    cos (j odd) of pos_k 2 pi / T^(2 floor(j / 2) / F), components 0 and 1 swapped when exchange_xy and n >= 2."""
    j = torch.arange(F, dtype=torch.float64, device=pos.device)
    a = pos[..., None] * (2 * math.pi) / temperature ** (2 * torch.div(j, 2, rounding_mode="floor") / F)
    emb = torch.where(j.remainder(2) == 0, a.sin(), a.cos())
    order = list(range(pos.shape[-1]))
    if exchange_xy and len(order) >= 2:
        order[0], order[1] = 1, 0
    return emb[:, order].flatten(1)


# ---- CPU: the fixtures and the restatements --------------------------------------------------------------------------
def test_pyramids_have_the_edges_they_are_meant_to():
    for name, (shapes, n) in CASES.items():
        if len(shapes) == 1:
            continue
        hw = [h * w for h, w in shapes]
        assert any(v < 32 for v in hw) and any(v % 32 in (1, 31) for v in hw) and any(v % 4 for v in hw), name
        assert any(h == 1 and w > 1 for h, w in shapes) and any(w == 1 and h > 1 for h, w in shapes), name
        assert (1, 1) in shapes and any(h > 32 and w > 32 for h, w in shapes), name
        masks = make_masks(shapes, n)
        assert masks[-1][-1].all(), name
        # counting the last column instead of the first, or the second row instead of the first, changes a count
        first_col = [(~m[:, :, 0]).sum(1) for m in masks]
        assert any(not torch.equal(c, (~m[:, :, -1]).sum(1)) for c, m in zip(first_col, masks)), name
        assert any(not torch.equal((~m[:, 0, :]).sum(1), (~m[:, 1, :]).sum(1)) for m in masks if m.shape[1] > 1), name
        # and the masks are no rectangles: some padded position has an unpadded one below it and to its right
        assert any((m[:, :-1, :-1] & ~m[:, 1:, 1:]).any() for m in masks), name


@pytest.mark.parametrize("name", list(CASES))
def test_fp64_restatements_match_the_cpu_chains(name):
    """The fp64 restatements above agree with the module's CPU chains (fp32), so a kernel that matches them matches
    the reference's formulas."""
    shapes, n = CASES[name]
    masks = make_masks(shapes, n)
    vr = torch.stack([torch.stack(((~m[:, 0, :]).sum(1).float() / m.shape[2], (~m[:, :, 0]).sum(1).float() / m.shape[1]),
                                  -1) for m in masks], 1)
    w_vr = valid_counts64(masks) / torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
    assert ((vr.double() - w_vr).abs() <= 2.0 ** -24 * w_vr).all()
    want, got = ref_points64(shapes, vr), get_reference_points(shapes, vr)
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(got))
    assert ((got[fin].double() - want[fin]).abs() <= 4 * 2.0 ** -24 * want[fin].abs()).all()
    prop, keep = gen_encoder_output_proposals(flat_mask(masks), shapes)
    w = proposals64(shapes, masks, 0.05)
    k = keep[..., 0]
    assert k.any() and (prop[k].double() - w[k]).abs().max() <= 1e-6 * w[k].abs().max()
    pos = torch.rand(50, 3, generator=torch.Generator().manual_seed(0))
    for F, t, xy in ((128, 10000, True), (34, 20, False)):
        assert (get_sine_pos_embed(pos, F, t, xy).double() - sine64(pos.double(), F, t, xy)).abs().max() < 1e-5


def test_odd_sine_width_raises():
    for dev in ["cpu"] + (["cuda"] if torch.cuda.is_available() else []):
        with pytest.raises(ValueError, match="even"):
            get_sine_pos_embed(torch.rand(4, 2, device=dev), 33)


# ---- flatten_levels ------------------------------------------------------------------------------------------------
def _flatten_arm(fn, srcs, masks, pos, le, want, feed):
    """fn on fresh leaves; want: which of 'src', 'pos', 'le' require grad; feed: which outputs (0 = src_flatten,
    2 = lvl_pos_embed_flatten) the loss reads.  -> (outputs, src grads, pos grads, level_embed grad, pos cotangent)."""
    s = [t.clone().requires_grad_("src" in want) for t in srcs]
    p = [t.clone().requires_grad_("pos" in want) for t in pos]
    e = le.clone().requires_grad_("le" in want)
    out = fn(s, masks, p, e)
    g = torch.Generator(device=DEV).manual_seed(1)
    cots = {i: torch.randn(out[i].shape, device=DEV, generator=g) for i in (0, 2)}
    fed = [(out[i], cots[i]) for i in feed if out[i].requires_grad]
    if fed:
        torch.autograd.backward([o for o, _ in fed], [c for _, c in fed])
    return out, [t.grad for t in s], [t.grad for t in p], e.grad, cots[2]


def _same_grad(a, b):
    """Bit-equal gradients; a leaf the reference's loss does not reach (None) may get zeros from the kernel."""
    if b is None:
        return a is None or not a.any()
    return a is not None and torch.equal(a, b)


def _check_flatten(shapes, srcs, masks, pos, le, want, feed):
    ko, ks, kp, ke, cot = _flatten_arm(_flatten, srcs, masks, pos, le, want, feed)
    ro, rs, rp, re, _ = _flatten_arm(reference_chain, srcs, masks, pos, le, want, feed)
    for i, (a, b) in enumerate(zip(ko, ro)):
        assert a.dtype == b.dtype and torch.equal(a, b), i
    assert all(_same_grad(a, b) for a, b in zip(ks, rs)) and all(_same_grad(a, b) for a, b in zip(kp, rp))
    if re is None:
        assert _same_grad(ke, None)
        return
    # grad_level_embed: the fp64 sum over images and each level's positions; rows past L embed no level.  fp32 sums of
    # 32 partials at a time stay far inside 1e-6 of the largest sum.
    st = starts_of(shapes)
    want_le = torch.zeros(le.shape, dtype=torch.float64, device=DEV)
    for lvl, (a, b) in enumerate(zip(st[:-1], st[1:])):
        want_le[lvl] = cot[:, a:b].double().sum((0, 1))
    assert ke.shape == le.shape and torch.equal(ke[len(shapes):], torch.zeros_like(ke[len(shapes):]))
    assert (ke.double() - want_le).abs().max().item() <= 1e-6 * want_le.abs().max().item()


def _flatten(*args):
    from uninext_b200.modules.dino_transformer import flatten_levels
    return flatten_levels(*args)


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("c", [4, 28, 32, 36, 260, 1024])
def test_flatten_levels_against_the_reference_chain(name, c):
    """Forward, valid ratios and all three gradients.  The ratios compare bit for bit: the reference divides on the
    device by the level size, which torch does as a multiply by its fp32 reciprocal, as flatten_levels does."""
    shapes, srcs, masks, pos, le = pyramid_inputs(name, c)
    _check_flatten(shapes, srcs, masks, pos, le, {"src", "pos", "le"}, (0, 2))
    if len(shapes) > 1:
        vr = _flatten(srcs, masks, pos, le)[5]
        assert (vr[-1, -1] == 0).all() and (vr[:, :-1] > 0).any()


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", ["l8_n3", "l6_n1"])
@pytest.mark.parametrize("want", [("src",), ("pos",), ("le",), ("src", "pos", "le"), ("src", "le")])
def test_flatten_levels_gradient_subsets(name, want):
    """Each subset of the leaves requiring grad (("src", "le"): pos_embeds do not), with both outputs in the loss and
    with only one (autograd gives the other's gradient as None, materialised as zeros), and a level_embed with more
    rows than levels."""
    shapes, srcs, masks, pos, le = pyramid_inputs(name, 36, le_rows=len(CASES[name][0]) + 3)
    for feed in ((0, 2), (0,), (2,)):
        _check_flatten(shapes, srcs, masks, pos, le, set(want), feed)


def _guarded(numel, dtype, fill, guard):
    """A buffer of numel elements with `guard` elements of `fill` on each side; -> (whole buffer, the inner view)."""
    buf = torch.full((numel + 2 * guard,), fill, dtype=dtype, device=DEV)
    return buf, buf[guard:guard + numel]


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("c", [4, 36])
def test_flatten_abi_writes_every_output_element_and_nothing_else(name, c):
    """Outputs, gradients and the workspace pre-filled with NaN (the mask with 0x5a) inside larger buffers: after the
    calls no NaN is left inside, the values are the reference chain's, and the 128 bytes on each side are untouched."""
    from uninext_b200 import _cabi
    shapes, srcs, masks, pos, le = pyramid_inputs(name, c)
    n, nl, s = srcs[0].shape[0], len(shapes), sum(h * w for h, w in shapes)
    hs, ws = (ctypes.c_int * nl)(*[h for h, _ in shapes]), (ctypes.c_int * nl)(*[w for _, w in shapes])
    nan, G = float("nan"), 32
    sf, sf_in = _guarded(n * s * c, torch.float32, nan, G)
    pf, pf_in = _guarded(n * s * c, torch.float32, nan, G)
    mf, mf_in = _guarded(n * s, torch.uint8, 0x5a, 4 * G)
    m8 = [m.view(torch.uint8) for m in masks]
    _cabi.call("msda_flatten_levels_forward_f32", _ptrs(srcs), _ptrs(pos), _ptrs(m8), hs, ws, nl, n, c, le, sf_in,
               pf_in, mf_in, device=le.device)
    src_flat, mask_flat, pos_flat = reference_chain(srcs, masks, pos, le)[:3]
    assert torch.equal(sf_in.view(n, s, c), src_flat) and torch.equal(pf_in.view(n, s, c), pos_flat)
    assert torch.equal(mf_in.view(n, s), mask_flat.view(torch.uint8))
    for buf in (sf, pf):
        assert torch.isnan(buf[:G]).all() and torch.isnan(buf[-G:]).all()
    assert (mf[:4 * G] == 0x5a).all() and (mf[-4 * G:] == 0x5a).all()

    g = torch.Generator(device=DEV).manual_seed(2)
    g_src, g_pos = (torch.randn(n, s, c, device=DEV, generator=g) for _ in range(2))
    gs = [_guarded(n * c * h * w, torch.float32, nan, G) for h, w in shapes]
    gp = [_guarded(n * c * h * w, torch.float32, nan, G) for h, w in shapes]
    ge, ge_in = _guarded(nl * c, torch.float32, nan, G)
    nbytes = _cabi.workspace("msda_flatten_levels_workspace", hs, ws, nl, n, c)
    work = torch.full((nbytes // 4,), nan, device=DEV)
    _cabi.call("msda_flatten_levels_backward_f32", g_src, g_pos, hs, ws, nl, n, c, _ptrs([v for _, v in gs]),
               _ptrs([v for _, v in gp]), ge_in, work, nbytes, device=g_src.device)
    st = starts_of(shapes)
    for lvl, (h, w) in enumerate(shapes):
        for g_flat, (buf, inner) in ((g_src, gs[lvl]), (g_pos, gp[lvl])):
            want = g_flat[:, st[lvl]:st[lvl + 1]].transpose(1, 2).reshape(n, c, h, w)
            assert torch.equal(inner.view(n, c, h, w), want), lvl
            assert torch.isnan(buf[:G]).all() and torch.isnan(buf[-G:]).all()
    want_le = torch.stack([g_pos[:, a:b].double().sum((0, 1)) for a, b in zip(st[:-1], st[1:])])
    assert (ge_in.view(nl, c).double() - want_le).abs().max().item() <= 1e-6 * want_le.abs().max().item()
    assert torch.isnan(ge[:G]).all() and torch.isnan(ge[-G:]).all()


# ---- geometry ------------------------------------------------------------------------------------------------------
def _ratios(name):
    shapes, srcs, masks, pos, le = pyramid_inputs(name, 4)
    return shapes, masks, _flatten(srcs, masks, pos, le)[5]


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", list(CASES))
def test_reference_points_against_the_torch_chain_and_fp64(name):
    """msda_encoder_ref_points at every position of every level: bit for bit the torch chain on the same device (with
    the same inf and NaN where a ratio is 0), and within 4 ulps of fp64 (three fp32 roundings) where finite."""
    shapes, _, vr = _ratios(name)
    got = get_reference_points(shapes, vr)
    xy, wh, lvl = (t.float() if t.is_floating_point() else t for t in pixel_grid64(shapes, DEV))
    chain = (xy[None] / (vr[:, lvl] * wh[None]))[:, :, None] * vr[:, None]
    nan = torch.isnan(chain)
    assert got.shape == chain.shape and torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan], chain[~nan])
    if len(shapes) > 1:
        assert nan.any() and torch.isinf(got).any()         # the fully padded level
    want = ref_points64(shapes, vr)
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(got)) and fin.any()
    assert ((got[fin].double() - want[fin]).abs() <= 4 * 2.0 ** -24 * want[fin].abs()).all()


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("base_scale", [0.05, 0.03, 0.005])
def test_encoder_proposals_against_the_cpu_chain_and_fp64(name, base_scale):
    """keep and the +inf pattern exactly the CPU chain's; finite values within 1e-6 of scale of it and of fp64 (the
    logit of an fp32 ratio: a few fp32 roundings of values below 5).  At 0.05 levels 5 .. 7 (0.05 2^l >= 0.99) are all
    dropped; at 0.005 levels 0 and 1 (sizes below 0.01) are."""
    shapes, n = CASES[name]
    masks = make_masks(shapes, n)
    m = flat_mask(masks)
    prop, keep = gen_encoder_output_proposals(m.to(DEV), shapes, base_scale)
    w_prop, w_keep = gen_encoder_output_proposals(m, shapes, base_scale)
    assert torch.equal(keep.cpu(), w_keep) and torch.equal(torch.isinf(prop).cpu(), torch.isinf(w_prop))
    assert torch.equal(torch.isinf(w_prop), ~w_keep.expand_as(w_prop))
    st = starts_of(shapes)
    sized = [0.01 < base_scale * 2 ** l < 0.99 for l in range(len(shapes))]
    for l, ok in enumerate(sized):
        if not ok:
            assert not keep[:, st[l]:st[l + 1]].any(), l
    k = w_keep[..., 0]
    assert k.any() == any(sized)                # a single level of size 0.005 keeps nothing
    if k.any():
        got, cpu, want = prop.cpu()[k].double(), w_prop[k].double(), proposals64(shapes, masks, base_scale)[k]
        scale = want.abs().max().item()
        assert (got - cpu).abs().max().item() <= 1e-6 * scale and (got - want).abs().max().item() <= 1e-6 * scale
    if name == "l8_n3" and base_scale == 0.05:
        assert not keep[:, st[5]:].any() and keep[:, :st[5]].any()


# ---- get_sine_pos_embed ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("F", [2, 30, 32, 34, 64, 128, 200])
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_sine_pos_embed_against_fp64_autograd(F, n):
    """Forward within 1e-5 absolute (the argument reaches 2 pi, and powf, the fp32 2 pi and sinf each round once);
    backward within 1e-4 of scale (a sum of F products of such terms).  exchange_xy on and off (with n = 1 it swaps
    nothing), temperature 20 and 10000, R from 1 to 100003 positions."""
    combos = [(False, 20, 1), (True, 10000, 33), (False, 10000, 1000), (True, 20, 100003)]
    g = torch.Generator(device=DEV).manual_seed(F * 10 + n)
    for xy, t, r in combos:
        pos = torch.rand(r, n, device=DEV, generator=g).requires_grad_(True)
        out = get_sine_pos_embed(pos, F, t, xy)
        p64 = pos.detach().double().requires_grad_(True)
        want = sine64(p64, F, t, xy)
        assert out.shape == want.shape == (r, n * F)
        assert (out.double() - want).abs().max().item() <= 1e-5, (xy, t, r)
        cot = torch.randn(out.shape, device=DEV, generator=g)
        out.backward(cot)
        want.backward(cot.double())
        scale = p64.grad.abs().max().item()
        assert (pos.grad.double() - p64.grad).abs().max().item() <= 1e-4 * scale, (xy, t, r)


# ---- two_stage_select ------------------------------------------------------------------------------------------------
# S = 63 / 64 / 65: one head-backward tile short of, at and one row past kTsRows = 64; 2083: 33 tiles, and k = 2048 /
# 2049 on either side of the on-chip sort (kTsSmemSort = 2048), k = S in the workspace sort.
TS_SHAPES = {1: ((1, 1),), 63: ((6, 8), (3, 4), (1, 3)), 64: ((6, 8), (3, 4), (2, 2)), 65: ((6, 8), (3, 4), (5, 1)),
             2083: ((40, 48), (13, 12), (7, 1))}
TS_PARAMS = [(s, n, k) for s in TS_SHAPES for n in (1, 5) for k in sorted({1, s} | ({2048, 2049} if s > 2049 else set()))]


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("s,n,k", TS_PARAMS)
def test_two_stage_select_small_and_odd_sizes(s, n, k):
    """restated_fp64 with test_user_sizes_against_fp64's tolerances and tie rules.  With N = 5 the last image is all
    padding: every row of it reads b_e, all its logits tie (ascending rows are selected) and its proposals are +inf."""
    from tests.test_gpu_two_stage import check_against_fp64, make_problem, run_fused
    shapes = TS_SHAPES[s]
    mask = flat_mask(make_masks(shapes, n, seed=s))
    if n > 1:
        mask[-1] = True
    assert mask.shape == (n, s) and (~mask).any()
    _, mods, x = make_problem(shapes, mask, ("still", "vl")[TS_PARAMS.index((s, n, k)) % 2], seed=s)
    out, g_mem, grads, cot = check_against_fp64(shapes, mods, x, k)
    if n > 1:
        assert torch.equal(out[3][-1], torch.arange(k, device=DEV)) and (out[2][-1] == 1).all()
    again = run_fused(shapes, mods, x, k, cot)
    a = [*out, g_mem, *grads.values()]
    b = [*again[0], again[1], *again[2].values()]
    assert all(torch.equal(u, v) for u, v in zip(a, b))
