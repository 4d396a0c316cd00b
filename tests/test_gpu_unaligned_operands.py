"""GPU tests (-m gpu): the kernels around the op and the CondInst head on operands that are contiguous but not 16-byte
aligned -- views ``buf[k:k + n]`` with a storage offset of k = 0..3 floats, which ``contiguous()`` / ``reshape`` pass on
unchanged -- against plain fp64 restatements of the same maths.  Tolerances as in test_gpu_fused.py (1e-5 of scale for
values, 1e-4 for reduced gradients) and test_gpu_condinst.py (2e-4 for the dynamic mask head, 1e-6 / 1e-5 for
aligned_bilinear).  Also: aligned_bilinear at factors 3 and 8 (generic kernels) and at widths > 512 (the factor-2
kernels' multi-sweep column loop), and the raw C ABI refusing misaligned pointers without touching its outputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.functions.fused import add_layer_norm, linear_colsum, sampling_prologue
    from uninext_b200.modules.dynamic_mask_head import aligned_bilinear, dynamic_mask_with_coords

DEV = "cuda"
OFFSETS = [0, 1, 2, 3]                          # storage offsets in floats: data_ptr() % 16 == 0, 4, 8, 12
BADARG = -1                                     # MSDA_E_BADARG


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _at(k, *shape, gen, scale=1.0, requires_grad=False):
    """A contiguous [shape] view starting k floats into a fresh buffer (random values), and the buffer (a leaf: gradients
    of the view land in buf.grad[k:k + n])."""
    n = 1
    for s in shape:
        n *= s
    buf = (torch.randn(n + 4, generator=gen) * scale).to(DEV).requires_grad_(requires_grad)
    t = buf[k:k + n].view(*shape)
    assert t.is_contiguous() and t.data_ptr() % 16 == 4 * k
    return t, buf


def _grad_of(view, buf):
    k = view.storage_offset()
    return buf.grad[k:k + view.numel()].view(view.shape)


def _lib():
    return _cabi.load()


# ---- add_layer_norm ------------------------------------------------------------------------------------------------------

def _layer_norm_fp64(a, b, norm, gy):
    a64 = a.detach().double().requires_grad_(True)
    b64 = None if b is None else b.detach().double().requires_grad_(True)
    w64 = norm.weight.detach().double().requires_grad_(True)
    bb64 = norm.bias.detach().double().requires_grad_(True)
    y64 = F.layer_norm(a64 if b64 is None else a64 + b64, (a.shape[-1],), w64, bb64, norm.eps)
    y64.backward(gy.double())
    return y64, a64.grad, None if b64 is None else b64.grad, w64.grad, bb64.grad


def _norm(cols, gen):
    norm = torch.nn.LayerNorm(cols).to(DEV)
    with torch.no_grad():
        norm.weight.copy_(1.0 + 0.2 * torch.randn(cols, generator=gen))
        norm.bias.copy_(0.2 * torch.randn(cols, generator=gen))
    return norm


@pytest.mark.parametrize("with_b", [True, False])
@pytest.mark.parametrize("cols", [128, 384])
@pytest.mark.parametrize("k", OFFSETS)
def test_add_layer_norm_unaligned_gradient(k, cols, with_b):
    """Aligned inputs (the kernels run forward), upstream gradient at offset k: the backward copies it to an aligned
    buffer instead of handing a misaligned pointer to the float4 kernel."""
    gen = torch.Generator().manual_seed(10 + k)
    rows = 77
    norm = _norm(cols, gen)
    a = torch.randn(rows, cols, generator=gen).to(DEV).requires_grad_(True)
    b = torch.randn(rows, cols, generator=gen).to(DEV).requires_grad_(True) if with_b else None
    gy, _ = _at(k, rows, cols, gen=gen)
    lib = _lib()
    n0 = lib.msda_launch_count()
    y = add_layer_norm(a, b, norm)
    n1 = lib.msda_launch_count()
    seen = []
    y.register_hook(lambda g: seen.append(g.data_ptr() % 16))
    y.backward(gy)
    assert seen == [4 * k]                                      # the backward received the offset gradient ...
    assert n1 > n0 and lib.msda_launch_count() > n1             # ... and forward and backward both ran the kernels
    want = _layer_norm_fp64(a, b, norm, gy)
    assert _rel(y, want[0]) < 1e-5 and _rel(a.grad, want[1]) < 1e-5
    if with_b:
        assert _rel(b.grad, want[2]) < 1e-5
    assert _rel(norm.weight.grad, want[3]) < 1e-4 and _rel(norm.bias.grad, want[4]) < 1e-4


@pytest.mark.parametrize("with_b", [True, False])
@pytest.mark.parametrize("cols", [128, 384])
@pytest.mark.parametrize("k", OFFSETS)
def test_add_layer_norm_unaligned_inputs(k, cols, with_b):
    """Inputs and upstream gradient at offset k: aligned inputs run the kernels, misaligned ones the stock ops -- the
    same numbers either way."""
    gen = torch.Generator().manual_seed(20 + k)
    rows = 50
    norm = _norm(cols, gen)
    a, abuf = _at(k, rows, cols, gen=gen, requires_grad=True)
    b, bbuf = _at(k, rows, cols, gen=gen, requires_grad=True) if with_b else (None, None)
    gy, _ = _at(k, rows, cols, gen=gen)
    y = add_layer_norm(a, b, norm)
    y.backward(gy)
    want = _layer_norm_fp64(a, b, norm, gy)
    assert _rel(y, want[0]) < 1e-5 and _rel(_grad_of(a, abuf), want[1]) < 1e-5
    if with_b:
        assert _rel(_grad_of(b, bbuf), want[2]) < 1e-5
    assert _rel(norm.weight.grad, want[3]) < 1e-4 and _rel(norm.bias.grad, want[4]) < 1e-4


@pytest.mark.parametrize("cols", [128, 384])
@pytest.mark.parametrize("lead", [1, 3, 5])
def test_add_layer_norm_gradient_from_cat_of_flattened_tensors(lead, cols):
    """loss = (cat([t0.flatten(), y.flatten()]) * w).sum() with an odd t0.numel(): autograd hands the backward a
    contiguous slice of the cat's gradient that starts 4 * lead bytes past an aligned block."""
    gen = torch.Generator().manual_seed(30 + lead)
    rows = 40
    norm = _norm(cols, gen)
    a = torch.randn(2, rows, cols, generator=gen).to(DEV).requires_grad_(True)
    t0 = torch.randn(lead, generator=gen).to(DEV).requires_grad_(True)
    w = torch.randn(lead + a.numel(), generator=gen).to(DEV)
    y = add_layer_norm(a, None, norm)
    seen = []
    y.register_hook(lambda g: seen.append(g.data_ptr() % 16))
    (torch.cat([t0.reshape(-1), y.reshape(-1)]) * w).sum().backward()
    assert seen == [4 * lead % 16] and seen[0] != 0
    want = _layer_norm_fp64(a, None, norm, w[lead:].view(a.shape))
    assert _rel(a.grad, want[1]) < 1e-5
    assert _rel(norm.weight.grad, want[3]) < 1e-4 and _rel(norm.bias.grad, want[4]) < 1e-4
    assert torch.equal(t0.grad, w[:lead])


# ---- sampling_prologue -----------------------------------------------------------------------------------------------------

# one L*P of each group width of msda_prologue_fwd / _bwd (4, 8, 16, 32 lanes per (row, head))
PROLOGUE = [(2, 1, 3, 3), (4, 2, 4, 4), (2, 4, 4, 2), (4, 4, 8, 2)]         # refdim, L, P, M


@pytest.mark.parametrize("k", OFFSETS)
@pytest.mark.parametrize("refdim,L,P,M", PROLOGUE)
def test_sampling_prologue_unaligned(refdim, L, P, M, k):
    """query, reference points and both upstream gradients at offset k; grad_loc is read as float2, so k = 1, 3 must be
    copied and k = 2 (8-byte aligned) may be read in place."""
    gen = torch.Generator().manual_seed(40 + 4 * L + P + k)
    rows, C = 93, 64
    off = torch.nn.Linear(C, M * L * P * 2).to(DEV)
    att = torch.nn.Linear(C, M * L * P).to(DEV)
    q, qbuf = _at(k, 2, rows, C, gen=gen, requires_grad=True)
    ref = torch.rand(2 * rows * L * refdim + 4, generator=gen).to(DEV)[k:k + 2 * rows * L * refdim].view(2, rows, L, refdim)
    shapes = torch.randint(2, 60, (L, 2), generator=gen).to(DEV)
    g_loc, _ = _at(k, 2, rows, M, L, P, 2, gen=gen)
    g_att, _ = _at(k, 2, rows, M, L, P, gen=gen)
    loc, attn = sampling_prologue(q, off, att, ref, shapes, M, L, P)
    seen = []
    loc.register_hook(lambda g: seen.append(g.data_ptr() % 16))
    torch.autograd.backward([loc, attn], [g_loc, g_att])
    assert seen == [4 * k]                                      # the kernel's wrapper received the offset gradient
    # the module's composition (ms_deform_attn.py:99-109) in fp64
    dd = lambda t: t.detach().double().requires_grad_(True)
    q64, ow, ob, aw, ab = (dd(t) for t in (q, off.weight, off.bias, att.weight, att.bias))
    o = F.linear(q64, ow, ob).view(2, rows, M, L, P, 2)
    a = F.softmax(F.linear(q64, aw, ab).view(2, rows, M, L * P), -1).view(2, rows, M, L, P)
    r = ref.double()
    if refdim == 2:
        wh = torch.stack([shapes[..., 1], shapes[..., 0]], -1).double()
        lc = r[:, :, None, :, None, :] + o / wh[None, None, None, :, None, :]
    else:
        lc = r[:, :, None, :, None, :2] + o / P * r[:, :, None, :, None, 2:] * 0.5
    (lc * g_loc.double()).sum().add((a * g_att.double()).sum()).backward()
    assert _rel(loc, lc) < 1e-5 and _rel(attn, a) < 1e-5
    assert _rel(_grad_of(q, qbuf), q64.grad) < 1e-4
    for got, want in ((off.weight.grad, ow.grad), (off.bias.grad, ob.grad), (att.weight.grad, aw.grad),
                      (att.bias.grad, ab.grad)):
        assert _rel(got, want) < 1e-4


# ---- linear_colsum(relu=True) --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", OFFSETS)
def test_linear_relu_backward_unaligned_gradient(k):
    """An upstream gradient at offset k reaches the ReLU backward: misaligned, it takes threshold_backward + colsum (as
    colsum() itself does) instead of raising."""
    gen = torch.Generator().manual_seed(50 + k)
    lin = torch.nn.Linear(256, 384).to(DEV)
    x = torch.randn(3, 77, 256, generator=gen).to(DEV).requires_grad_(True)
    gy, _ = _at(k, 3, 77, 384, gen=gen)
    y = linear_colsum(x, lin, relu=True)
    seen = []
    y.register_hook(lambda g: seen.append(g.data_ptr() % 16))
    y.backward(gy)
    assert seen == [4 * k]
    x64, w64, b64 = (t.detach().double().requires_grad_(True) for t in (x, lin.weight, lin.bias))
    y64 = torch.relu(F.linear(x64, w64, b64))
    y64.backward(gy.double())
    assert _rel(y, y64) < 1e-5
    assert _rel(x.grad, x64.grad) < 1e-4 and _rel(lin.weight.grad, w64.grad) < 1e-4 and _rel(lin.bias.grad, b64.grad) < 1e-4


# ---- CondInst dynamic mask head ------------------------------------------------------------------------------------------

def _aligned_bilinear_fp64(x, f):
    """ddetrs.py:921-942 in fp64: replicate-pad by one, align_corners bilinear to (f*h + 1, f*w + 1), shift by f // 2."""
    *lead, h, w = x.shape
    t = F.pad(x.reshape(1, -1, h, w), (0, 1, 0, 1), mode="replicate")
    t = F.interpolate(t, size=(f * h + 1, f * w + 1), mode="bilinear", align_corners=True)
    t = F.pad(t, (f // 2, 0, f // 2, 0), mode="replicate")
    return t[..., :f * h, :f * w].reshape(*lead, f * h, f * w)


def _dynamic_mask_fp64(feats, refs, params, num_insts, stride, factor):
    """The 3-layer dynamic MLP from the parameter layout of include/msda_b200.h -- w1[8][10] | w2[8][8] | w3[8] | b1[8] |
    b2[8] | b3, inputs (rel_x, rel_y, feat_0..7), rel = ref - (pixel * stride + stride // 2) -- then aligned_bilinear."""
    n, c, h, w = feats.shape
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    loc = torch.stack([xs, ys]).double() * stride + stride // 2                                   # [2, h, w]
    logits, s = [], 0
    for b, cnt in enumerate(num_insts):
        p, r = params[s:s + cnt], refs[s:s + cnt]
        s += cnt
        x = torch.cat([r[:, :, None, None] - loc, feats[b].expand(cnt, c, h, w)], 1)             # [cnt, 10, h, w]
        w1, w2, w3 = p[:, :80].view(cnt, 8, 10), p[:, 80:144].view(cnt, 8, 8), p[:, 144:152].view(cnt, 1, 8)
        b1, b2, b3 = p[:, 152:160], p[:, 160:168], p[:, 168:169]
        x = torch.relu(torch.einsum("noc,nchw->nohw", w1, x) + b1[..., None, None])
        x = torch.relu(torch.einsum("noc,nchw->nohw", w2, x) + b2[..., None, None])
        logits.append((torch.einsum("noc,nchw->nohw", w3, x) + b3[..., None, None])[:, 0])
    return _aligned_bilinear_fp64(torch.cat(logits), factor)[None]


@pytest.mark.parametrize("k", OFFSETS)
@pytest.mark.parametrize("num_insts,hw", [([5, 3], (12, 20)), ([4, 0, 19], (9, 11)), ([21], (25, 42)), ([2, 6], (1, 7))])
def test_dynamic_mask_head_unaligned_features(num_insts, hw, k):
    """Mask features, reference points and parameters at offset k, with H*W % 4 == 0 (the shape that takes 16-byte
    accesses when the features are aligned) and H*W % 4 != 0; forward and all three gradients."""
    gen = torch.Generator().manual_seed(60 + k)
    n, (h, w), total, stride = len(num_insts), hw, sum(num_insts), 8
    feats, fbuf = _at(k, n, 8, h, w, gen=gen, requires_grad=True)
    refs, rbuf = _at(k, 1, total, 2, gen=gen, requires_grad=True)
    with torch.no_grad():
        rbuf.uniform_(0, 8.0 * max(h, w))
    params, pbuf = _at(k, 1, total, 169, gen=gen, scale=0.3, requires_grad=True)
    out = dynamic_mask_with_coords(feats, refs, params, num_insts, stride, True, 4)
    go = torch.randn(out.shape, generator=gen).to(DEV)
    out.backward(go)
    f64, r64, p64 = (t.detach().double().requires_grad_(True) for t in (feats, refs, params))
    want = _dynamic_mask_fp64(f64, r64.view(total, 2), p64.view(total, 169), num_insts, stride, 2)
    want.backward(go.double())
    assert _rel(out, want) < 2e-4
    assert _rel(_grad_of(feats, fbuf), f64.grad) < 2e-4
    assert _rel(_grad_of(params, pbuf), p64.grad) < 2e-4
    assert _rel(_grad_of(refs, rbuf), r64.grad) < 1e-3         # piecewise-linear through two ReLUs, as test_gpu_condinst.py


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("hw", [(12, 20), (9, 11)])
def test_condinst_forward_abi_unaligned_feats_and_logits(hw, k):
    """msda_condinst_forward_f32 with feats and logits both at offset k: the scalar path gives bit for bit what the
    16-byte path gives on aligned copies (the same FMAs in the same order)."""
    gen = torch.Generator().manual_seed(70 + k)
    h, w = hw
    num_insts = [6, 11]
    total = sum(num_insts)
    feats, _ = _at(k, 2, 8, h, w, gen=gen)
    params = (torch.randn(total, 169, generator=gen) * 0.3).to(DEV)
    refs = (torch.rand(total, 2, generator=gen) * 8.0 * max(h, w)).to(DEV)
    starts = torch.tensor([0, num_insts[0], total], dtype=torch.int32, device=DEV)
    lib = _lib()
    stream = torch.cuda.current_stream().cuda_stream
    outbuf = torch.full((total * h * w + 4,), float("nan"), device=DEV)
    logits = outbuf[k:k + total * h * w]
    assert logits.data_ptr() % 16 == 4 * k
    ref_logits = torch.empty(total * h * w, device=DEV)
    for f, o in ((feats, logits), (feats.clone(), ref_logits)):
        assert lib.msda_condinst_forward_f32(f.data_ptr(), params.data_ptr(), refs.data_ptr(), starts.data_ptr(), 2, h, w,
                                             total, max(num_insts), 8, 1, o.data_ptr(), stream) == 0
    torch.cuda.synchronize()
    assert torch.equal(logits, ref_logits)
    assert outbuf[:k].isnan().all() and outbuf[k + total * h * w:].isnan().all()        # nothing written outside


# ---- aligned_bilinear ------------------------------------------------------------------------------------------------------

# factors 3 and 8: generic kernels (odd f for 3); factor 2 with w > 512: more than 256 column groups per row, i.e. the
# multi-sweep column loop of aligned_bilinear2_fwd (2w / 4 > 256) and aligned_bilinear2_bwd (w / 2 > 256)
BILINEAR = [(3, (2, 9, 13)), (3, (1, 1, 1)), (3, (3, 20, 34)), (8, (2, 7, 10)), (8, (1, 3, 1)), (2, (2, 5, 600)),
            (2, (1, 3, 1030)), (4, (1, 4, 520))]


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("factor,shape", BILINEAR)
def test_aligned_bilinear_matches_fp64(factor, shape, k):
    """Input and upstream gradient at offset k (k = 1: the backward reads grad_out through the generic kernel)."""
    gen = torch.Generator().manual_seed(80 + factor)
    x, xbuf = _at(k, *shape, gen=gen, requires_grad=True)
    out = aligned_bilinear(x, factor)
    go, _ = _at(k, *out.shape, gen=gen)
    out.backward(go)
    x64 = x.detach().double().requires_grad_(True)
    want = _aligned_bilinear_fp64(x64, factor)
    want.backward(go.double())
    assert _rel(out, want) < 1e-6
    assert _rel(_grad_of(x, xbuf), x64.grad) < 1e-5


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("factor,shape", [(2, (2, 5, 600)), (2, (3, 6, 8)), (4, (2, 9, 13)), (3, (2, 4, 8))])
def test_aligned_bilinear_abi_unaligned_out_and_grad_out(factor, shape, k):
    """out and grad_out at offset k through the C ABI: the forward takes the one-output-per-thread kernel (VEC = 1), the
    backward the generic gather (grad_out not 16-byte aligned), grad_in at offset k too."""
    gen = torch.Generator().manual_seed(90 + k)
    planes, h, w = shape
    oh, ow = h * factor, w * factor
    x = torch.randn(*shape, generator=gen).to(DEV)
    lib = _lib()
    stream = torch.cuda.current_stream().cuda_stream
    obuf = torch.full((planes * oh * ow + 4,), float("nan"), device=DEV)
    out = obuf[k:k + planes * oh * ow]
    assert lib.msda_aligned_bilinear_forward_f32(x.data_ptr(), planes, h, w, factor, out.data_ptr(), stream) == 0
    go, _ = _at(k, planes, oh, ow, gen=gen)
    gbuf = torch.full((planes * h * w + 4,), float("nan"), device=DEV)
    gin = gbuf[k:k + planes * h * w]
    assert lib.msda_aligned_bilinear_backward_f32(go.data_ptr(), planes, h, w, factor, gin.data_ptr(), stream) == 0
    torch.cuda.synchronize()
    x64 = x.double().requires_grad_(True)
    want = _aligned_bilinear_fp64(x64, factor)
    want.backward(go.double())
    assert _rel(out.view(planes, oh, ow), want) < 1e-6
    assert _rel(gin.view(shape), x64.grad) < 1e-5
    for buf, n in ((obuf, planes * oh * ow), (gbuf, planes * h * w)):
        assert buf[:k].isnan().all() and buf[k + n:].isnan().all()


# ---- raw C ABI: misaligned pointers are refused before anything is enqueued ---------------------------------------------

def _sentinel(n):
    return torch.full((n + 4,), 12345.0, device=DEV)


def test_abi_refuses_misaligned_operands_and_leaves_outputs_untouched():
    lib = _lib()
    stream = torch.cuda.current_stream().cuda_stream
    rows, cols, R, M, L, P = 20, 256, 10, 2, 2, 4
    src = torch.randn(rows * cols * 8 + 64, device=DEV)
    inp = lambda k: src.data_ptr() + 4 * k                     # readable input at a float offset k
    shapes = torch.tensor([[8, 9], [4, 5]], dtype=torch.int64, device=DEV)
    outs = {name: _sentinel(n) for name, n in (("y", rows * cols), ("z", rows * cols), ("mean", rows), ("rstd", rows),
                                               ("dz", rows * cols), ("dgamma", cols), ("dbeta", cols),
                                               ("loc", R * M * L * P * 2), ("attn", R * M * L * P),
                                               ("gproj", R * M * L * P * 3), ("g2", rows * cols), ("colsum", cols))}
    o = lambda name, k=0: outs[name].data_ptr() + 4 * k
    calls = {
        "add_layernorm_forward a": lambda: lib.msda_add_layernorm_forward_f32(
            inp(1), inp(0), inp(0), inp(0), rows, cols, 1e-5, o("z"), o("y"), o("mean"), o("rstd"), stream),
        "add_layernorm_forward y": lambda: lib.msda_add_layernorm_forward_f32(
            inp(0), None, inp(0), inp(0), rows, cols, 1e-5, None, o("y", 2), o("mean"), o("rstd"), stream),
        "add_layernorm_forward z": lambda: lib.msda_add_layernorm_forward_f32(
            inp(0), inp(0), inp(0), inp(0), rows, cols, 1e-5, o("z", 3), o("y"), o("mean"), o("rstd"), stream),
        "layernorm_backward dy": lambda: lib.msda_layernorm_backward_f32(
            inp(1), inp(0), inp(0), inp(0), inp(0), rows, cols, o("dz"), o("dgamma"), o("dbeta"), stream),
        "layernorm_backward dz": lambda: lib.msda_layernorm_backward_f32(
            inp(0), inp(0), inp(0), inp(0), inp(0), rows, cols, o("dz", 1), o("dgamma"), o("dbeta"), stream),
        "layernorm_backward dbeta": lambda: lib.msda_layernorm_backward_f32(
            inp(0), inp(0), inp(0), inp(0), inp(0), rows, cols, o("dz"), o("dgamma"), o("dbeta", 2), stream),
        "prologue_forward loc": lambda: lib.msda_prologue_forward_f32(
            inp(0), inp(0), shapes.data_ptr(), R, M, L, P, 2, o("loc", 1), o("attn"), stream),
        "prologue_backward grad_loc": lambda: lib.msda_prologue_backward_f32(
            inp(3), inp(0), inp(0), inp(0), shapes.data_ptr(), R, M, L, P, 2, o("gproj"), stream),
        "relu_backward_colsum g": lambda: lib.msda_relu_backward_colsum_f32(
            inp(1), inp(0), rows, cols, o("g2"), o("colsum"), stream),
        "colsum out": lambda: lib.msda_colsum_f32(inp(0), rows, cols, o("colsum", 2), stream),
    }
    before = lib.msda_launch_count()
    for what, call in calls.items():
        assert call() == BADARG, what
    torch.cuda.synchronize()
    assert lib.msda_launch_count() == before
    for name, t in outs.items():
        assert (t == 12345.0).all(), name
