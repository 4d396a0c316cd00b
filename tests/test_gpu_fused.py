"""GPU tests of the one-pass kernels around the op (prologue, column sum, add+LayerNorm) against the plain PyTorch
composition they replace (fp32; tolerance 1e-5 relative to scale for values, 1e-4 for reduced gradients)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200.functions.fused import add_layer_norm, colsum, linear_colsum, sampling_prologue
    from uninext_b200.modules import MSDeformAttn

DEV = "cuda"


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("rows,cols", [(1, 4), (37, 128), (44646, 256), (44646, 384), (600, 2048), (301, 1200), (5, 8)])
def test_colsum(rows, cols):
    torch.manual_seed(0)
    x = torch.randn(rows, cols, device=DEV)
    assert _rel(colsum(x), x.double().sum(0)) < 1e-5


@pytest.mark.parametrize("rows,cols,with_b", [(3, 128, True), (1000, 256, True), (44646, 256, True), (777, 512, False),
                                              (50, 384, True)])
def test_add_layer_norm_matches_torch(rows, cols, with_b):
    torch.manual_seed(1)
    norm = torch.nn.LayerNorm(cols).to(DEV)
    with torch.no_grad():
        norm.weight.normal_(1.0, 0.2); norm.bias.normal_(0, 0.2)
    a = torch.randn(2, rows, cols, device=DEV, requires_grad=True)
    b = torch.randn(2, rows, cols, device=DEV, requires_grad=True) if with_b else None
    gy = torch.randn(2, rows, cols, device=DEV)
    y = add_layer_norm(a, b, norm)
    y.backward(gy)
    got = (y.detach(), a.grad.clone(), None if b is None else b.grad.clone(), norm.weight.grad.clone(), norm.bias.grad.clone())
    a.grad = None; norm.weight.grad = None; norm.bias.grad = None
    if b is not None:
        b.grad = None
    a64, b64 = a.detach().double().requires_grad_(True), (None if b is None else b.detach().double().requires_grad_(True))
    z = a64 if b64 is None else a64 + b64
    w64 = norm.weight.detach().double().requires_grad_(True); bb64 = norm.bias.detach().double().requires_grad_(True)
    y64 = F.layer_norm(z, (cols,), w64, bb64, norm.eps)
    y64.backward(gy.double())
    assert _rel(got[0], y64) < 1e-5
    assert _rel(got[1], a64.grad) < 1e-5
    if b is not None:
        assert _rel(got[2], b64.grad) < 1e-5
    assert _rel(got[3], w64.grad) < 1e-4 and _rel(got[4], bb64.grad) < 1e-4


@pytest.mark.parametrize("refdim,L,P,M,rows", [(2, 4, 4, 8, 1000), (4, 4, 4, 8, 301), (2, 2, 3, 5, 77), (4, 8, 4, 2, 64),
                                               (2, 1, 1, 3, 9)])
def test_sampling_prologue_matches_module_math(refdim, L, P, M, rows):
    torch.manual_seed(2)
    C = 64
    off = torch.nn.Linear(C, M * L * P * 2).to(DEV)
    att = torch.nn.Linear(C, M * L * P).to(DEV)
    q = torch.randn(2, rows, C, device=DEV, requires_grad=True)
    shapes = torch.randint(2, 60, (L, 2), device=DEV)
    ref = torch.rand(2, rows, L, refdim, device=DEV)
    g_loc = torch.randn(2, rows, M, L, P, 2, device=DEV)
    g_att = torch.randn(2, rows, M, L, P, device=DEV)
    loc, w = sampling_prologue(q, off, att, ref, shapes, M, L, P)
    (loc * g_loc).sum().add((w * g_att).sum()).backward()
    got = (loc.detach(), w.detach(), q.grad.clone(), off.weight.grad.clone(), off.bias.grad.clone(),
           att.weight.grad.clone(), att.bias.grad.clone())
    for t in (q, off.weight, off.bias, att.weight, att.bias):
        t.grad = None
    # the reference composition (ms_deform_attn.py:99-109), in fp64
    dd = lambda t: t.detach().double()
    q64 = dd(q).requires_grad_(True)
    ow, ob, aw, ab = (dd(t).requires_grad_(True) for t in (off.weight, off.bias, att.weight, att.bias))
    o = F.linear(q64, ow, ob).view(2, rows, M, L, P, 2)
    a = F.softmax(F.linear(q64, aw, ab).view(2, rows, M, L * P), -1).view(2, rows, M, L, P)
    r = ref.double()
    if refdim == 2:
        norm = torch.stack([shapes[..., 1], shapes[..., 0]], -1).double()
        lc = r[:, :, None, :, None, :] + o / norm[None, None, None, :, None, :]
    else:
        lc = r[:, :, None, :, None, :2] + o / P * r[:, :, None, :, None, 2:] * 0.5
    (lc * g_loc.double()).sum().add((a * g_att.double()).sum()).backward()
    assert _rel(got[0], lc) < 1e-5 and _rel(got[1], a) < 1e-5
    assert _rel(got[2], q64.grad) < 1e-4
    for g, t in zip(got[3:], (ow, ob, aw, ab)):
        assert _rel(g, t.grad) < 1e-4


def test_add_layer_norm_under_autocast_is_fp32_like_torch():
    torch.manual_seed(8)
    norm = torch.nn.LayerNorm(256).to(DEV)
    a = torch.randn(4, 300, 256, device=DEV).bfloat16().requires_grad_(True)
    b = torch.randn(4, 300, 256, device=DEV).bfloat16().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = add_layer_norm(a, b, norm)
        y_ref = norm(a + b)
    assert y.dtype == torch.float32 and y_ref.dtype == torch.float32
    assert _rel(y, y_ref) < 2e-2                      # torch adds in bf16 first; ours adds the fp32 casts
    y.float().square().mean().backward()
    assert a.grad.dtype == torch.bfloat16 and torch.isfinite(a.grad.float()).all() and norm.weight.grad is not None


def test_linear_colsum_matches_linear():
    torch.manual_seed(3)
    lin = torch.nn.Linear(256, 384).to(DEV)
    x = torch.randn(3, 500, 256, device=DEV, requires_grad=True)
    gy = torch.randn(3, 500, 384, device=DEV)
    y = linear_colsum(x, lin); y.backward(gy)
    got = (y.detach(), x.grad.clone(), lin.weight.grad.clone(), lin.bias.grad.clone())
    x.grad = None; lin.weight.grad = None; lin.bias.grad = None
    y2 = lin(x); y2.backward(gy)
    assert torch.allclose(got[0], y2, rtol=1e-4, atol=1e-4)
    assert _rel(got[1], x.grad) < 1e-3 and _rel(got[2], lin.weight.grad) < 1e-3 and _rel(got[3], lin.bias.grad) < 1e-4


def test_linear_relu_and_split_k_weight_grad():
    from uninext_b200.functions.fused import weight_grad
    torch.manual_seed(5)
    lin = torch.nn.Linear(256, 512).to(DEV)
    x = torch.randn(2, 9000, 256, device=DEV, requires_grad=True)          # 18000 rows -> split-K path (256*512 outputs)
    gy = torch.randn(2, 9000, 512, device=DEV)
    y = linear_colsum(x, lin, relu=True); y.backward(gy)
    got = (y.detach(), x.grad.clone(), lin.weight.grad.clone(), lin.bias.grad.clone())
    x.grad = None; lin.weight.grad = None; lin.bias.grad = None
    y2 = torch.relu(lin(x)); y2.backward(gy)
    assert torch.allclose(got[0], y2, rtol=1e-4, atol=1e-4)
    assert _rel(got[1], x.grad) < 1e-3 and _rel(got[2], lin.weight.grad) < 1e-3 and _rel(got[3], lin.bias.grad) < 1e-4
    g2, x2 = torch.randn(44646, 384, device=DEV), torch.randn(44646, 256, device=DEV)
    assert _rel(weight_grad(g2, x2), g2.double().t() @ x2.double()) < 1e-4


@pytest.mark.parametrize("m,n,k", [(128, 256, 256), (1, 32, 32), (300, 256, 256), (1000, 384, 256), (44646, 256, 256),
                                   (44646, 384, 256), (513, 512, 64), (77, 32, 96), (200, 448, 128), (129, 64, 512)])
def test_tcgen05_linear_matches_fp64_within_tf32(m, n, k):
    """Hand-written TF32 GEMM (sm_90a wgmma, TMA-fed): TF32 operands (10-bit mantissa), fp32 accumulate."""
    from uninext_b200.functions.fused import tcgen05_linear, tcgen05_linear_ok
    torch.manual_seed(6)
    a = torch.randn(m, k, device=DEV)
    w = torch.randn(n, k, device=DEV) * 0.1
    b = torch.randn(n, device=DEV)
    assert tcgen05_linear_ok(a, w)
    for bias in (b, None):
        got = tcgen05_linear(a, w, bias)
        want = a.double() @ w.double().t() + (0 if bias is None else bias.double())
        assert _rel(got, want) < 2e-3
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:                                            # and as close to cuBLAS' TF32 result as TF32 rounding allows
        assert _rel(tcgen05_linear(a, w, b), torch.addmm(b, a, w.t())) < 2e-3
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def test_module_with_tcgen05_gemms():
    from uninext_b200.workloads import CONFIGS, level_tensors
    from uninext_b200.modules.deformable_layers import encoder_reference_points
    cfg = CONFIGS["cfg1"]
    ss, lsi = level_tensors(cfg.shapes, DEV)
    torch.manual_seed(7)
    a, b = MSDeformAttn(gemm="tcgen05").to(DEV), MSDeformAttn(gemm="cublas").to(DEV)
    with torch.no_grad():
        a.sampling_offsets.weight.normal_(0, 0.02); a.attention_weights.weight.normal_(0, 0.05)
    b.load_state_dict(a.state_dict())
    src = torch.randn(2, cfg.S, 256, device=DEV)
    ref = encoder_reference_points(cfg.shapes, torch.ones(2, 4, 2, device=DEV), DEV)
    outs = []
    for mod in (a, b):
        x = src.clone().requires_grad_(True)
        y = mod(x, ref, x, ss, lsi, None)
        y.square().mean().backward()
        outs.append((y.detach(), x.grad))
    # TF32 (10-bit mantissa) products vs fp32 products: the forward stays within 1e-2 of scale; in the backward a 1e-3
    # relative change of the sampling offsets moves ~0.4 % of the taps into the neighbouring bilinear cell, whose location
    # gradient differs by O(1), so the input gradient is compared in the L2 sense.
    assert _rel(outs[0][0], outs[1][0]) < 1e-2
    l2 = ((outs[0][1] - outs[1][1]).double().norm() / outs[1][1].double().norm()).item()
    assert l2 < 3e-2 and _rel(outs[0][1], outs[1][1]) < 0.2


def test_fused_and_unfused_module_agree():
    from uninext_b200.workloads import CONFIGS, level_tensors
    from uninext_b200.modules.deformable_layers import encoder_reference_points
    cfg = CONFIGS["cfg1"]
    ss, lsi = level_tensors(cfg.shapes, DEV)
    torch.manual_seed(4)
    a, b = MSDeformAttn(fused=True).to(DEV), MSDeformAttn(fused=False).to(DEV)
    with torch.no_grad():
        a.sampling_offsets.weight.normal_(0, 0.02); a.attention_weights.weight.normal_(0, 0.05)
    b.load_state_dict(a.state_dict())
    src = torch.randn(2, cfg.S, 256, device=DEV)
    ref = encoder_reference_points(cfg.shapes, torch.ones(2, 4, 2, device=DEV), DEV)
    mask = torch.zeros(2, cfg.S, dtype=torch.bool, device=DEV); mask[1, -50:] = True
    outs = []
    for mod in (a, b):
        x = src.clone().requires_grad_(True)
        y = mod(x, ref, x, ss, lsi, mask)
        y.square().mean().backward()
        outs.append((y.detach(), x.grad, {k: p.grad for k, p in mod.named_parameters()}))
    assert _rel(outs[0][0], outs[1][0]) < 1e-4 and _rel(outs[0][1], outs[1][1]) < 1e-3
    for k in outs[0][2]:
        assert _rel(outs[0][2][k], outs[1][2][k]) < 1e-3, k


@pytest.mark.parametrize("m,n,k,use_mask,relu", [(128, 256, 256, False, False), (300, 256, 256, True, False), (1, 64, 32, False, True),
                                                   (1000, 192, 128, True, True), (44646, 256, 256, True, False)])
def test_tcgen05_w_stationary_linear_with_fused_tail(m, n, k, use_mask, relu):
    """msda_linear_tf32_ex: C = A W^T + bias with the padding-mask zeroing (ms_deform_attn.py:96-97) and ReLU in the epilogue."""
    from uninext_b200.functions.fused import tcgen05_linear_ex, tcgen05_ws_ok
    g = torch.Generator().manual_seed(m + n)
    a = torch.randn(m, k, generator=g).to(DEV)
    w = (torch.randn(n, k, generator=g) * 0.1).to(DEV)
    b = torch.randn(n, generator=g).to(DEV)
    mask = (torch.rand(m, generator=g) < 0.3).to(DEV) if use_mask else None
    assert tcgen05_ws_ok(a, w)
    got = tcgen05_linear_ex(a, w, b, mask, relu)
    want = a.double() @ w.double().t() + b.double()
    if relu:
        want = want.clamp_min(0)
    if mask is not None:
        want = want.masked_fill(mask[:, None], 0.0)
        assert (got[mask] == 0).all()                      # masked rows are exact zeros, not small numbers
    assert _rel(got, want) < 2e-3                            # TF32 products, fp32 accumulation


def test_module_tcgen05_gemm_with_fused_mask():
    """gemm="tcgen05": value_proj runs on the W-stationary tcgen05 kernel with bias and padding mask fused (no masked_fill
    launch) and stays within TF32 distance of the fp32 result; gemm="auto" (default) follows allow_tf32 / MSDA_GEMM_AUTO."""
    from uninext_b200 import _cabi
    from uninext_b200.workloads import CONFIGS, level_tensors
    from uninext_b200.modules.deformable_layers import encoder_reference_points
    cfg = CONFIGS["cfg1"]
    ss, lsi = level_tensors(cfg.shapes, DEV)
    torch.manual_seed(9)
    assert MSDeformAttn().gemm == "auto"
    mod = MSDeformAttn(gemm="tcgen05").to(DEV)
    src = torch.randn(2, cfg.S, 256, device=DEV)
    ref = encoder_reference_points(cfg.shapes, torch.ones(2, 4, 2, device=DEV), DEV)
    mask = torch.zeros(2, cfg.S, dtype=torch.bool, device=DEV); mask[1, -200:] = True
    lib = _cabi.load()
    old = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        mod.gemm = "cublas"
        want = mod(src, ref, src, ss, lsi, mask)
        mod.gemm = "tcgen05"
        x = src.clone().requires_grad_(True)
        got = mod(x, ref, x, ss, lsi, mask)
        got.square().mean().backward()
        assert torch.isfinite(x.grad).all()
        # gemm="auto": cuBLAS, except value_proj WITH a padding mask under allow_tf32 (fused mask epilogue beats GEMM + masked_fill)
        mod.gemm = "auto"
        auto_fp32 = mod(src, ref, src, ss, lsi, mask)
        torch.backends.cuda.matmul.allow_tf32 = True
        auto_tf32 = mod(src, ref, src, ss, lsi, mask)
        auto_nomask = mod(src, ref, src, ss, lsi, None)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert _rel(got, want) < 1e-2
    assert torch.equal(auto_fp32, want)                                 # strict fp32: the cuBLAS path, bit for bit
    assert _rel(auto_tf32, want) < 1e-2 and torch.isfinite(auto_nomask).all()
    assert (auto_tf32[1, -200:] - auto_fp32[1, -200:]).abs().max() < 1e-2
