"""GPU tests of the fused image-text attention in TF32 mode (msda_vlfuse_tc.cuh): taken when torch allows TF32 matmuls.

Accuracy is judged against TF32 products: for each output, the fused TF32 error against the fp64 restatement must stay
within 2x the error of the same maths in fp32 torch ops, plus 1e-4.  That yardstick's error is the larger of torch's own
run under TF32 and a run with every product operand rounded to TF32 explicitly, because cuBLAS runs fp32 SGEMMs for
some shapes (small or unaligned T) even when TF32 is allowed.  In-process tests switch TF32
only through ``torch.backends.cuda.matmul.allow_tf32``; the newer ``fp32_precision`` API runs in subprocesses, because
once it is used, later ``allow_tf32`` reads in that process raise."""
import os
import subprocess
import sys
import textwrap
import time
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from tests import vlfuse_case as vc
from tests.test_gpu_vlfuse import CASES, _fwd_bwd, _inputs, _restate, _seed, _vlf_kernels
from uninext_b200.modules import vl_fusion as vf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("O_v", "O_l", "dQ", "dK", "dVv", "dVl")
TC = {"vlf_tc_fwd_rows", "vlf_tc_fwd_cols", "vlf_tc_bwd_rows", "vlf_tc_bwd_cols"}
SIMT = {"vlf_fwd_rows", "vlf_fwd_cols", "vlf_bwd_rows", "vlf_bwd_cols"}
SHARED = {"vlf_colstats", "vlf_reduce", "vlf_bwd_delta"}


@contextmanager
def tf32(on=True):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = on
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def _torch_tf32(q, k, vv, vl, bias, cmin, cmax, masks=None, p=0.0):
    """The restatement's maths in fp32 torch ops; under TF32, cuBLAS may run their einsums on tensor cores."""
    if masks is None:
        return vf.vl_attention_torch(q, k, vv, vl, bias, cmin, cmax)
    x = torch.einsum("bshd,bthd->bhst", q, k)
    xc = x.clamp(min=-50000) if cmin else x
    xc = xc.clamp(max=50000) if cmax else xc
    y = xc.transpose(2, 3)
    p_l = (y - y.max(dim=-1, keepdim=True)[0]).softmax(dim=-1)
    p_v = (xc + bias[:, None, None, :] if bias is not None else xc).softmax(dim=-1)
    scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    p_v, p_l = p_v * masks[0] * scale, p_l * masks[1] * scale
    return torch.einsum("bhst,bthd->bshd", p_v, vl), torch.einsum("bhts,bshd->bthd", p_l, vv)


def _rna(t):
    """fp32 -> the nearest TF32 value (ties away from zero), as cvt.rna.tf32.f32 rounds."""
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


class _Operand(torch.autograd.Function):
    """A product's operand: rounded to TF32 on the way in; its gradient passes unchanged."""
    @staticmethod
    def forward(ctx, t):
        return _rna(t)

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
        return _rna(g)


class _Attend(torch.autograd.Function):
    """O = drop(softmax(logits)) V over the last axis of `logits` [b, h, i, j], V [b, j, h, d], with TF32 products and
    the kernels' softmax backward: dlogits = P o (dP - delta), delta = rowsum(dO o O) in fp32."""
    @staticmethod
    def forward(ctx, logits, v, keep):
        p = logits.softmax(dim=-1)
        pd = p * keep
        o = torch.einsum("bhij,bjhd->bihd", _rna(pd), _rna(v))
        ctx.save_for_backward(p, pd, v, keep, o)
        return o

    @staticmethod
    def backward(ctx, go):
        p, pd, v, keep, o = ctx.saved_tensors
        g = torch.einsum("bihd,bjhd->bhij", _rna(go), _rna(v)) * keep
        delta = (go * o).sum(-1).permute(0, 2, 1).unsqueeze(-1)
        return p * (g - delta), torch.einsum("bhij,bihd->bjhd", _rna(pd), _rna(go)), None


def _tf32_model(q, k, vv, vl, bias, cmin, cmax, masks=None, p=0.0):
    """The kernels' formulas with every operand of every product, forward and backward, rounded once to TF32 and fp32
    accumulation: the TF32 arithmetic whatever kernel cuBLAS picks (for small or unaligned T it runs fp32 SGEMMs even
    under allow_tf32, so torch's own TF32 result can be plain fp32).  Run with allow_tf32 off.  delta = rowsum(dO o O)
    matters where a softmax is over one element (T = 1, or S = 1 for the text side): there the exact gradient through
    it is zero, and the TF32 rounding of dO in dP is left over against the fp32 delta."""
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


def _check_tf32(q, k, vv, vl, bias, cmin, cmax, seed=None, p=0.0):
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    masks = None
    if p > 0:
        B, S, H, _ = q.shape
        masks = vf.dropout_masks(seed, B, H, S, k.shape[1], p)
    with tf32():
        got = _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, cmin, cmax, p, p > 0, seed=seed), q, k, vv, vl, go_v, go_l)
        yard = _fwd_bwd(lambda *a: _torch_tf32(*a, bias, cmin, cmax, masks, p), q, k, vv, vl, go_v, go_l)
    with tf32(False):
        model = _fwd_bwd(lambda *a: _tf32_model(*a, bias, cmin, cmax, masks, p), q, k, vv, vl, go_v, go_l)
    want = _fwd_bwd(lambda *a: _restate(*a, bias, cmin, cmax, masks, p), *(t.double() for t in (q, k, vv, vl)),
                    go_v, go_l)
    for name, g, y, m, w in zip(NAMES, got, yard, model, want):
        e, ey = _err(g, w), max(_err(y, w), _err(m, w))
        assert e <= 2 * ey + 1e-4, (name, e, _err(y, w), _err(m, w))


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_tf32_within_torch_tf32_error(case):
    *shape, cmin, cmax, bias_kind, big = case
    q, k, vv, vl, bias = _inputs(*shape, bias_kind, big)
    _check_tf32(q, k, vv, vl, bias, cmin, cmax)


def test_tf32_dropout_within_torch_tf32_error():
    q, k, vv, vl, bias = _inputs(2, 4, 1000, 40, 128, "partial")
    _check_tf32(q, k, vv, vl, bias, True, True, seed=_seed(1234), p=0.1)


@pytest.mark.parametrize("fwd_mode", [True, False])
def test_backward_keeps_the_forward_mode(fwd_mode):
    q, k, vv, vl, bias = _inputs(2, 4, 700, 40, 256, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)

    def run(bwd_mode):
        leaves = [t.detach().clone().requires_grad_(True) for t in (q, k, vv, vl)]
        with tf32(fwd_mode):
            o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True, seed=_seed(5))
        with tf32(bwd_mode):
            return torch.autograd.grad((o_v, o_l), leaves, (go_v, go_l))

    same, flipped = run(fwd_mode), run(not fwd_mode)
    assert all(torch.equal(a, b) for a, b in zip(same, flipped))


def test_tf32_runs_are_bit_identical():
    q, k, vv, vl, bias = _inputs(2, 8, 5000, 256, 256, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    run = lambda: _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=_seed(99)),
                           q, k, vv, vl, go_v, go_l)
    with tf32():
        a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_tf32_training_step_repeats_under_manual_seed():
    from tests.test_gpu_vlfuse import _train_step
    with tf32():
        a, b = _train_step(3), _train_step(3)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_tf32_core_runs_under_deterministic_algorithms():
    q, k, vv, vl, bias = _inputs(1, 8, 700, 40, 256, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    torch.use_deterministic_algorithms(True)
    try:
        with tf32():
            a = _fwd_bwd(lambda *x: vf.vl_attention(*x, bias, True, True, 0.1, True, seed=_seed(3)), q, k, vv, vl,
                         go_v, go_l)        # raises if anything on the path alerts
    finally:
        torch.use_deterministic_algorithms(False)
    with tf32():
        b = _fwd_bwd(lambda *x: vf.vl_attention(*x, bias, True, True, 0.1, True, seed=_seed(3)), q, k, vv, vl,
                     go_v, go_l)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_tf32_cuda_graph_replay_equals_eager_and_redraws_the_seed():
    q, k, vv, vl, bias = _inputs(1, 8, 700, 40, 256, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, vv, vl)]

    def step():
        seed = vf.draw_seed("cuda")
        o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True, seed=seed)
        grads = torch.autograd.grad((o_v, o_l), leaves, (go_v, go_l))
        return [seed, o_v, o_l, *grads]

    with tf32():
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


@pytest.mark.parametrize("T,stable,mode,want", [
    (17, False, True, TC | SHARED), (256, False, True, TC | SHARED), (17, False, False, SIMT | SHARED),
    (256, False, False, SIMT | SHARED), (257, False, True, set()), (17, True, True, set())])
def test_profiler_shows_which_kernels_run(T, stable, mode, want):
    q, k, vv, vl, _ = _inputs(1, 8, 300, T, 256, None)
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]

    def fn():
        o_v, o_l = vf.vl_attention(*leaves, None, True, True, 0.0, False, stable)
        (o_v.sum() + o_l.sum()).backward()

    with tf32(mode):
        fn()
        for _ in range(4):      # a window that misses records is profiled again; the path is fixed by the inputs
            names, launched = _vlf_kernels(fn)
            if want <= names:
                break
            time.sleep(0.5)
    assert launched == (3 * 9 if want else 0), launched
    assert names == want, names


def test_tf32_peak_memory_stays_below_one_logits_copy():
    B, H, S, T, D = 2, 8, 22323, 256, 256
    q, k, vv, vl, bias = _inputs(B, H, S, T, D, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with tf32():
        o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True)
        torch.autograd.backward((o_v, o_l), (go_v, go_l))
    torch.cuda.synchronize()
    outputs = sum(t.numel() * 4 for t in (o_v, o_l, *(x.grad for x in leaves)))
    extra = torch.cuda.max_memory_allocated() - base - outputs
    assert extra < B * H * S * T * 4, extra / 2 ** 20


@pytest.mark.parametrize("name", sorted(vc.CASES))
def test_tf32_block_matches_reference_fixture(name):
    """BiAttentionBlock with the fused TF32 core, and with the torch composition under TF32, against the reference."""
    import tests.test_vlfuse_reference as ref
    want = dict(np.load(os.path.join(ref.GOLDEN, f"vlfuse_{name}.npz")))
    want.pop("state_dict_keys")
    with tf32():
        fused = vc.run(ref._block(), name, "cuda")
        orig = vf.fused_supported
        vf.fused_supported = lambda *a, **kw: False
        try:
            comp = vc.run(ref._block(), name, "cuda")
        finally:
            vf.fused_supported = orig
    for key, w in want.items():
        scale = max(np.abs(w).max(), 1e-30)
        e = np.abs(fused[key].astype(np.float64) - w).max() / scale
        ec = np.abs(comp[key].astype(np.float64) - w).max() / scale
        assert e <= 2 * ec + 2e-4, (name, key, e, ec)


# ---- the ways of allowing TF32, each in a fresh process --------------------------------------------------------------
SETTERS = {
    "allow_tf32": "torch.backends.cuda.matmul.allow_tf32 = True",
    "matmul_precision": "torch.set_float32_matmul_precision('high')",
    "cuda_fp32_precision": "torch.backends.cuda.matmul.fp32_precision = 'tf32'",
    "backends_fp32_precision": "torch.backends.fp32_precision = 'tf32'",
}

_ROUTE_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, sys.argv[1])
    exec(sys.argv[2])
    from torch.profiler import ProfilerActivity, profile
    from uninext_b200.modules import vl_fusion as vf
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, vv, vl = (torch.randn(1, n, 8, 256, device="cuda", generator=g).requires_grad_(True)
                    for n in (300, 17, 300, 17))
    for _ in range(4):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device="cuda").add_(1)
            for _ in range(3):
                o_v, o_l = vf.vl_attention(q, k, vv, vl)
                (o_v.sum() + o_l.sum()).backward()
            torch.cuda.synchronize()
        names = {e.name.split("<")[0].split("(")[0].split("::")[-1] for e in prof.events() if "vlf_" in e.name}
        if {"vlf_tc_fwd_rows", "vlf_tc_bwd_cols"} <= names:
            break
    print("KERNELS", " ".join(sorted(names)))
""")


def _subprocess(script, *args):
    proc = subprocess.run([sys.executable, "-c", script, ROOT, *args], capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]
    return proc.stdout


@pytest.mark.parametrize("setter", sorted(SETTERS))
def test_each_way_of_allowing_tf32_selects_the_tc_kernels(setter):
    out = _subprocess(_ROUTE_SCRIPT, SETTERS[setter])
    names = set(out.split("KERNELS", 1)[1].split())
    assert names == TC | SHARED, names


_GEMM_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, sys.argv[1])
    exec(sys.argv[2])
    from uninext_b200 import _cabi
    from uninext_b200.modules.ms_deform_attn import MSDeformAttn
    from uninext_b200.workloads import CONFIGS, encoder_reference_points, level_tensors
    cfg = CONFIGS["cfg1"]
    ss, lsi = level_tensors(cfg.shapes, "cuda")
    torch.manual_seed(0)
    mod = MSDeformAttn(256, 4, 8, 4).cuda()
    assert mod.gemm == "auto"
    n, s = 2, cfg.S
    src = torch.randn(n, s, 256, device="cuda", requires_grad=True)
    ref = encoder_reference_points(cfg.shapes, "cuda").view(1, s, 1, 2).expand(n, s, 4, 2).contiguous()
    mask = torch.zeros(n, s, dtype=torch.bool, device="cuda")
    mask[1, -200:] = True
    lib = _cabi.load()
    mod(src, ref, src, ss, lsi, mask).square().mean().backward()
    torch.cuda.synchronize()
    before = lib.msda_launch_count()
    out = mod(src, ref, src, ss, lsi, mask)
    out.square().mean().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(src.grad).all()
    print("LAUNCHES", lib.msda_launch_count() - before)
""")


def test_gemm_auto_under_the_new_api_matches_allow_tf32():
    new = _subprocess(_GEMM_SCRIPT, SETTERS["cuda_fp32_precision"]).split("LAUNCHES", 1)[1].split()[0]
    legacy = _subprocess(_GEMM_SCRIPT, SETTERS["allow_tf32"]).split("LAUNCHES", 1)[1].split()[0]
    assert new == legacy, (new, legacy)
