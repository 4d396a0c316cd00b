"""GPU tests of the fused image-text attention in bf16 mode (msda_vlfuse_bf16.cuh): taken for bf16 q, k, vv and vl.

Accuracy is judged against bf16 products: the yardstick restates the kernels' formulas in torch with every product
operand rounded to bf16, fp32 accumulation and the outputs rounded to bf16 (``_bf16_model``, the bf16 counterpart of
``_tf32_model`` in test_gpu_vlfuse_tf32.py).  For each output, the fused error against the fp64 restatement, on the
bf16-valued inputs, must stay within 2x the yardstick's error plus 1e-3."""
import os
import time

import numpy as np
import pytest
import torch

from tests import vlfuse_case as vc
from tests.test_gpu_vlfuse import CASES, _fwd_bwd, _inputs, _restate, _seed, _vlf_kernels
from tests.test_gpu_vlfuse_tf32 import tf32
from uninext_b200.modules import vl_fusion as vf

pytestmark = pytest.mark.gpu
NAMES = ("O_v", "O_l", "dQ", "dK", "dVv", "dVl")
BF16 = {"vlf_bf16_fwd_rows", "vlf_bf16_fwd_cols", "vlf_bf16_bwd_rows", "vlf_bf16_bwd_cols"}
TC = {"vlf_tc_fwd_rows", "vlf_tc_fwd_cols", "vlf_tc_bwd_rows", "vlf_tc_bwd_cols"}
SIMT = {"vlf_fwd_rows", "vlf_fwd_cols", "vlf_bwd_rows", "vlf_bwd_cols"}
SHARED = {"vlf_colstats", "vlf_reduce", "vlf_bwd_delta"}
UNINEXT_SHAPES = [(2, 8, 22323, 256, 256), (1, 8, 22323, 20, 256)]   # cfg2 with T = 256; cfg5 (20-token prompt)


def _bf(t):
    return t.to(torch.bfloat16).float()


class _Operand(torch.autograd.Function):
    """A product's operand: rounded to bf16 on the way in; its gradient passes unchanged."""
    @staticmethod
    def forward(ctx, t):
        return _bf(t)

    @staticmethod
    def backward(ctx, g):
        return g


class _Product(torch.autograd.Function):
    """A product's result: unchanged on the way out; its gradient, an operand of the backward products, is rounded."""
    @staticmethod
    def forward(ctx, t):
        return t.clone()

    @staticmethod
    def backward(ctx, g):
        return _bf(g)


class _Attend(torch.autograd.Function):
    """O = bf16(drop(softmax(logits)) V) over the last axis of `logits` [b, h, i, j], V [b, j, h, d], with bf16 products
    and the kernels' softmax backward: dlogits = P o (dP - delta), delta = rowsum(dO o O) in fp32 over the bf16 O and
    dO.  dV is rounded to bf16 (an output)."""
    @staticmethod
    def forward(ctx, logits, v, keep):
        p = logits.softmax(dim=-1)
        pd = p * keep
        o = _bf(torch.einsum("bhij,bjhd->bihd", _bf(pd), _bf(v)))
        ctx.save_for_backward(p, pd, v, keep, o)
        return o

    @staticmethod
    def backward(ctx, go):
        p, pd, v, keep, o = ctx.saved_tensors
        go = _bf(go)
        g = torch.einsum("bihd,bjhd->bhij", go, _bf(v)) * keep
        delta = (go * o).sum(-1).permute(0, 2, 1).unsqueeze(-1)
        return p * (g - delta), _bf(torch.einsum("bhij,bihd->bjhd", _bf(pd), go)), None


class _RoundGrad(torch.autograd.Function):
    """Identity whose gradient is rounded to bf16: dQ and dK are outputs of the kernels."""
    @staticmethod
    def forward(ctx, t):
        return t.clone()

    @staticmethod
    def backward(ctx, g):
        return _bf(g)


def _bf16_model(q, k, vv, vl, bias, cmin, cmax, masks=None, p=0.0):
    """The kernels' formulas on fp32 copies of bf16 tensors: every product operand rounded to bf16, fp32 accumulation,
    every output rounded to bf16.  Run with TF32 not allowed."""
    q, k = _RoundGrad.apply(q), _RoundGrad.apply(k)
    x = _Product.apply(torch.einsum("bshd,bthd->bhst", _Operand.apply(q), _Operand.apply(k)))
    xc = x.clamp(min=-50000) if cmin else x
    xc = xc.clamp(max=50000) if cmax else xc
    y = xc.transpose(2, 3)
    if masks is None:
        keep_v = keep_l = torch.ones((), device=q.device)
    else:
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
        keep_v, keep_l = masks[0] * scale, masks[1] * scale
    o_v = _Attend.apply(xc + bias[:, None, None, :] if bias is not None else xc, vl, keep_v)
    o_l = _Attend.apply(y - y.max(dim=-1, keepdim=True)[0].detach(), vv, keep_l)
    return o_v, o_l


def _err(g, w):
    return ((g.double() - w).abs().max() / w.abs().max().clamp_min(1e-30)).item()


def _bf16_inputs(*shape, bias_kind=None, big=False, seed=0):
    """``_inputs`` rounded to bf16: (q, k, vv, vl) as bf16 tensors, the text bias fp32."""
    q, k, vv, vl, bias = _inputs(*shape, bias_kind, big, seed)
    return (*(t.to(torch.bfloat16) for t in (q, k, vv, vl)), bias)


def _check_bf16(q, k, vv, vl, bias, cmin, cmax, seed=None, p=0.0, absolute=None):
    """q, k, vv, vl: bf16.  Returns the fused errors against fp64."""
    go_v, go_l = torch.randn(q.shape, device="cuda").to(torch.bfloat16), torch.randn(k.shape, device="cuda").to(torch.bfloat16)
    masks = None
    if p > 0:
        B, S, H, _ = q.shape
        masks = vf.dropout_masks(seed, B, H, S, k.shape[1], p)
    got = _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, cmin, cmax, p, p > 0, seed=seed), q, k, vv, vl, go_v, go_l)
    assert all(t.dtype == torch.bfloat16 for t in got), [t.dtype for t in got]
    f32 = [t.float() for t in (q, k, vv, vl)]
    with tf32(False):
        model = _fwd_bwd(lambda *a: _bf16_model(*a, bias, cmin, cmax, masks, p), *f32, go_v.float(), go_l.float())
    want = _fwd_bwd(lambda *a: _restate(*a, bias, cmin, cmax, masks, p), *(t.double() for t in (q, k, vv, vl)),
                    go_v.double(), go_l.double())
    errs = {}
    for name, g, m, w in zip(NAMES, got, model, want):
        e, em = _err(g, w), _err(m, w)
        assert e <= 2 * em + 1e-3, (name, e, em)
        if absolute is not None:
            assert e < absolute, (name, e, em)
        errs[name] = e
    return errs


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_bf16_within_bf16_product_error(case):
    *shape, cmin, cmax, bias_kind, big = case
    q, k, vv, vl, bias = _bf16_inputs(*shape, bias_kind=bias_kind, big=big)
    # the project's bf16 tolerance at the UNINEXT shapes; single-element softmaxes (T = 1, S = 1) carry the dO-rounding
    # residue the yardstick reproduces, so only the relative bound applies there
    _check_bf16(q, k, vv, vl, bias, cmin, cmax, absolute=1e-2 if tuple(shape) in UNINEXT_SHAPES else None)


def test_bf16_cfg5_shape_within_bf16_tolerance():
    q, k, vv, vl, bias = _bf16_inputs(*UNINEXT_SHAPES[1], bias_kind="partial")
    _check_bf16(q, k, vv, vl, bias, True, True, absolute=1e-2)


def test_bf16_dropout_matches_yardstick_with_exported_masks():
    q, k, vv, vl, bias = _bf16_inputs(2, 4, 1000, 40, 128, bias_kind="partial")
    _check_bf16(q, k, vv, vl, bias, True, True, seed=_seed(1234), p=0.1)
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    run = lambda: _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=_seed(1234)),
                           q, k, vv, vl, go_v, go_l)
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_bf16_runs_are_bit_identical():
    q, k, vv, vl, bias = _bf16_inputs(2, 8, 5000, 256, 256, bias_kind="partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    run = lambda: _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=_seed(99)),
                           q, k, vv, vl, go_v, go_l)
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _train_step(seed):
    torch.manual_seed(seed)
    block = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6,
                                op_dtype=torch.bfloat16).cuda().train()
    v = torch.randn(2, 2125, 256, device="cuda", requires_grad=True)
    l = torch.randn(2, 17, 768, device="cuda", requires_grad=True)
    mask = torch.ones(2, 17, dtype=torch.int64, device="cuda")
    mask[1, 9:] = 0
    out_v, out_l = block(v, l, mask)
    (out_v.square().sum() + out_l.square().sum()).backward()
    return [out_v, out_l, v.grad, l.grad] + [p.grad for p in block.parameters()]


def test_bf16_training_step_repeats_under_manual_seed():
    a, b = _train_step(3), _train_step(3)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    c = _train_step(4)
    assert not torch.equal(a[0], c[0])


def test_bf16_core_runs_under_deterministic_algorithms():
    q, k, vv, vl, bias = _bf16_inputs(1, 8, 700, 40, 256, bias_kind="partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    run = lambda: _fwd_bwd(lambda *x: vf.vl_attention(*x, bias, True, True, 0.1, True, seed=_seed(3)), q, k, vv, vl,
                           go_v, go_l)
    torch.use_deterministic_algorithms(True)
    try:
        a = run()           # raises if anything on the path alerts
    finally:
        torch.use_deterministic_algorithms(False)
    b = run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_bf16_cuda_graph_replay_equals_eager_and_redraws_the_seed():
    q, k, vv, vl, bias = _bf16_inputs(1, 8, 700, 40, 256, bias_kind="partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, vv, vl)]

    def step():
        seed = vf.draw_seed("cuda")
        o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True, seed=seed)
        grads = torch.autograd.grad((o_v, o_l), leaves, (go_v, go_l))
        return [seed, o_v, o_l, *grads]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    seeds = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        seed = static[0].clone()
        seeds.append(seed.item())
        eager = _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=seed), q, k, vv, vl,
                         go_v, go_l)
        assert all(torch.equal(x, y) for x, y in zip(static[1:], eager))
    assert seeds[0] != seeds[1]


@pytest.mark.parametrize("T,stable,dtype,allow_tf32,want", [
    (17, False, torch.bfloat16, False, BF16 | SHARED), (256, False, torch.bfloat16, False, BF16 | SHARED),
    (17, False, torch.bfloat16, True, BF16 | SHARED), (256, False, torch.bfloat16, True, BF16 | SHARED),
    (17, False, torch.float32, False, SIMT | SHARED), (17, False, torch.float32, True, TC | SHARED),
    (257, False, torch.bfloat16, False, set()), (17, True, torch.bfloat16, False, set())])
def test_profiler_shows_which_kernels_run(T, stable, dtype, allow_tf32, want):
    q, k, vv, vl, _ = _inputs(1, 8, 300, T, 256, None)
    leaves = [t.to(dtype).requires_grad_(True) for t in (q, k, vv, vl)]

    def fn():
        o_v, o_l = vf.vl_attention(*leaves, None, True, True, 0.0, False, stable)
        (o_v.float().sum() + o_l.float().sum()).backward()

    with tf32(allow_tf32):
        fn()
        for _ in range(4):      # a window that misses records is profiled again; the path is fixed by the inputs
            names, launched = _vlf_kernels(fn)
            if want <= names:
                break
            time.sleep(0.5)
    assert launched == (3 * 9 if want else 0), launched
    assert names == want, names
    assert all(t.grad.dtype == dtype for t in leaves)


def test_bf16_peak_memory_stays_below_one_bf16_logits_copy():
    B, H, S, T, D = 2, 8, 22323, 256, 256
    q, k, vv, vl, bias = _bf16_inputs(B, H, S, T, D, bias_kind="partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True)
    torch.autograd.backward((o_v, o_l), (go_v, go_l))
    torch.cuda.synchronize()
    outputs = sum(t.numel() * 2 for t in (o_v, o_l, *(x.grad for x in leaves)))
    extra = torch.cuda.max_memory_allocated() - base - outputs
    assert extra < B * H * S * T * 2, extra / 2 ** 20


# The l_proj bias gradient is the sum of dK over all text tokens.  The vision softmax's part of that sum cancels exactly
# (every row of its dS sums to zero), so the gradient is a small residue of much larger terms, and rounding dS to bf16
# leaves an error of a few 1e-2 of it.  The bf16 torch composition shows the same; this key is held to 2x its error.
CANCELLING = {"grad.attn.l_proj.bias"}


@pytest.mark.parametrize("autocast", [False, True], ids=["fp32", "autocast"])
@pytest.mark.parametrize("name", sorted(vc.CASES))
def test_bf16_block_matches_reference_fixture(name, autocast):
    """BiAttentionBlock(op_dtype=bf16) against the reference block's fp32 results: within 1e-2 of each result's scale,
    except the cancelling sums above, which stay within 2x the error of the bf16 torch composition in the same block."""
    import tests.test_vlfuse_reference as ref
    want = dict(np.load(os.path.join(ref.GOLDEN, f"vlfuse_{name}.npz")))
    want.pop("state_dict_keys")
    block = lambda: vf.BiAttentionBlock(vc.V_DIM, vc.L_DIM, vc.EMBED, vc.HEADS, dropout=0.1, drop_path=0.0,
                                        init_values=1.0 / 6, op_dtype=torch.bfloat16)
    seen = []
    orig_attention, orig_supported = vf.vl_attention, vf.fused_supported

    def spy(*a, **kw):
        out = orig_attention(*a, **kw)
        seen.append((a[0].dtype, out[0].dtype))
        return out
    vf.vl_attention = spy
    try:
        with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
            fused_block = block()
            got = vc.run(fused_block, name, "cuda")
            vf.fused_supported = lambda *a, **kw: False
            comp = vc.run(block(), name, "cuda")
    finally:
        vf.vl_attention, vf.fused_supported = orig_attention, orig_supported
    assert seen == [(torch.bfloat16, torch.bfloat16)] * 2, seen
    assert all(p.dtype == torch.float32 and p.grad.dtype == torch.float32 for p in fused_block.parameters())
    for key, w in want.items():
        scale = max(np.abs(w).max(), 1e-30)
        e = np.abs(got[key].astype(np.float64) - w).max() / scale
        ec = np.abs(comp[key].astype(np.float64) - w).max() / scale
        if key in CANCELLING:
            assert e <= max(2 * ec, 1e-2), (name, key, e, ec)
        else:
            assert e < 1e-2, (name, key, e, ec)


def test_bf16_block_output_and_gradient_dtypes():
    torch.manual_seed(0)
    block = vf.BiAttentionBlock(256, 768, 2048, 8, op_dtype=torch.bfloat16).cuda().train()
    v = torch.randn(2, 300, 256, device="cuda", requires_grad=True)
    l = torch.randn(2, 17, 768, device="cuda", requires_grad=True)
    for autocast in (False, True):
        with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
            out_v, out_l = block(v, l)
        assert out_v.dtype == out_l.dtype == torch.float32, (autocast, out_v.dtype, out_l.dtype)
        (out_v.float().sum() + out_l.float().sum()).backward()
        assert v.grad.dtype == l.grad.dtype == torch.float32
        assert all(p.grad.dtype == torch.float32 for p in block.parameters())
