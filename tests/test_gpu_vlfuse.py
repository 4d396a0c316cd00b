"""GPU tests of the fused image-text attention (msda_vlfuse.cuh, uninext_b200/modules/vl_fusion.py): accuracy against an
fp64 restatement, dropout, determinism, CUDA-graph replay, which kernels run, and peak memory."""
import time

import numpy as np
import pytest
import torch

from uninext_b200 import _cabi
from uninext_b200.modules import vl_fusion as vf

pytestmark = pytest.mark.gpu

MASKED = float(np.float32(-9e15))    # fl32(x - 9e15) for any |x| < 2^28: the logit of a padded text token


def _inputs(B, H, S, T, D, bias_kind, big=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    q, k = r(B, S, H, D) * (3.0 / D ** 0.5), r(B, T, H, D)
    vv, vl = r(B, S, H, D), r(B, T, H, D)
    if big:           # exact +-50000 ties: q[..., 0] in {-400, 0, 400} against k[..., 0] in {0, 400}
        q[..., 0] = 400.0 * torch.randint(-1, 2, (B, S, H), device="cuda", generator=g).float()
        k[..., 0] = 400.0 * torch.randint(0, 2, (B, T, H), device="cuda", generator=g).float()
    mask = None
    if bias_kind is not None:
        mask = torch.ones(B, T, dtype=torch.int64, device="cuda")
        mask[0, T // 2 + 1:] = 0
        if bias_kind == "padded" and B > 1:
            mask[1] = 0
    return q, k, vv, vl, vf.text_bias(mask, T)


def _restate(q, k, vv, vl, bias, cmin, cmax, masks=None, p=0.0):
    """fp64 restatement: the logits in fp64; a padded token's logit is what fp32 makes of x - 9e15 (the gradient still
    passes, as through the reference's add); dropout applies the given keep-masks."""
    x = torch.einsum("bshd,bthd->bhst", q, k)
    xc = x
    if cmin:
        xc = xc.clamp(min=-50000)
    if cmax:
        xc = xc.clamp(max=50000)
    y = xc.transpose(2, 3)
    p_l = (y - y.max(dim=-1, keepdim=True)[0]).softmax(dim=-1)
    xm = xc
    if bias is not None:
        b = bias[:, None, None, :].double()
        xm = xc + torch.where(b < -1e15, MASKED - xc, b).detach()
    p_v = xm.softmax(dim=-1)
    if masks is not None:
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
        p_v, p_l = p_v * masks[0].double() * scale, p_l * masks[1].double() * scale
    return torch.einsum("bhst,bthd->bshd", p_v, vl), torch.einsum("bhts,bshd->bthd", p_l, vv)


def _fwd_bwd(fn, q, k, vv, vl, go_v, go_l):
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, k, vv, vl)]
    o_v, o_l = fn(*leaves)
    grads = torch.autograd.grad((o_v, o_l), leaves, (go_v.to(o_v.dtype), go_l.to(o_l.dtype)))
    return [o_v.detach(), o_l.detach(), *grads]


def _check(q, k, vv, vl, bias, cmin, cmax, seed=None, p=0.0, tol=1e-4):
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    got = _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, cmin, cmax, p, p > 0, seed=seed), q, k, vv, vl, go_v, go_l)
    masks = None
    if p > 0:
        B, S, H, _ = q.shape
        masks = vf.dropout_masks(seed, B, H, S, k.shape[1], p)
    want = _fwd_bwd(lambda *a: _restate(*a, bias, cmin, cmax, masks, p), *(t.double() for t in (q, k, vv, vl)),
                    go_v, go_l)
    for name, g, w in zip(("O_v", "O_l", "dQ", "dK", "dVv", "dVl"), got, want):
        err = ((g.double() - w).abs().max() / w.abs().max().clamp_min(1e-30)).item()
        assert err < tol, (name, err)


CASES = [  # B, H, S, T, D, clamp_min, clamp_max, text mask, large logits
    (2, 8, 2125, 17, 256, True, True, "partial", False),       # cfg1 S, UNINEXT heads
    (2, 8, 22323, 256, 256, True, True, "partial", False),     # cfg2 S, MAX_QUERY_LEN
    (1, 4, 2125, 1, 128, True, True, None, False),             # T = 1
    (2, 2, 1, 256, 256, True, True, "padded", False),          # S = 1, one element fully padded
    (2, 4, 1000, 17, 128, True, True, "padded", False),        # S not a multiple of any tile
    (1, 8, 333, 256, 128, False, False, None, False),          # both clamps off
    (2, 2, 517, 33, 256, True, False, "partial", False),       # one clamp each way
    (1, 2, 517, 40, 256, False, True, None, False),
    (2, 4, 1500, 256, 256, True, True, "partial", True),       # logits past +-50000 on both sides
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_fused_matches_fp64_restatement(case):
    *shape, cmin, cmax, bias_kind, big = case
    q, k, vv, vl, bias = _inputs(*shape, bias_kind, big)
    _check(q, k, vv, vl, bias, cmin, cmax)


def _seed(value):
    return torch.tensor([value], dtype=torch.int64, device="cuda")


def test_dropout_matches_restatement_with_exported_masks():
    q, k, vv, vl, bias = _inputs(2, 4, 1000, 40, 128, "partial")
    _check(q, k, vv, vl, bias, True, True, seed=_seed(1234), p=0.1)


def test_dropout_masks_statistics_and_reproducibility():
    B, H, S, T, p = 2, 8, 2125, 256, 0.1
    mv, ml = vf.dropout_masks(_seed(7), B, H, S, T, p)
    n = mv.numel()
    for m in (mv, ml):
        kept = m.sum().item()
        sd = (n * p * (1 - p)) ** 0.5
        assert abs(kept - n * (1 - p)) < 6 * sd, kept / n
    assert (mv != ml.transpose(2, 3)).float().mean().item() > 0.1
    mv2, ml2 = vf.dropout_masks(_seed(7), B, H, S, T, p)
    assert torch.equal(mv, mv2) and torch.equal(ml, ml2)
    mv3, _ = vf.dropout_masks(_seed(8), B, H, S, T, p)
    assert not torch.equal(mv, mv3)


def _train_step(seed):
    torch.manual_seed(seed)
    block = vf.BiAttentionBlock(256, 768, 2048, 8, dropout=0.1, init_values=1.0 / 6).cuda().train()
    v = torch.randn(2, 2125, 256, device="cuda", requires_grad=True)
    l = torch.randn(2, 17, 768, device="cuda", requires_grad=True)
    mask = torch.ones(2, 17, dtype=torch.int64, device="cuda")
    mask[1, 9:] = 0
    out_v, out_l = block(v, l, mask)
    (out_v.square().sum() + out_l.square().sum()).backward()
    return [out_v, out_l, v.grad, l.grad] + [p.grad for p in block.parameters()]


def test_manual_seed_reproduces_training_step_bit_for_bit():
    a, b = _train_step(3), _train_step(3)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    c = _train_step(4)
    assert not torch.equal(a[0], c[0])


def test_two_runs_with_dropout_are_bit_identical():
    q, k, vv, vl, bias = _inputs(2, 8, 5000, 256, 256, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    run = lambda: _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=_seed(99)),
                           q, k, vv, vl, go_v, go_l)
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_cuda_graph_replay_equals_eager_and_redraws_the_seed():
    q, k, vv, vl, bias = _inputs(1, 8, 700, 40, 256, "partial")
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
        eager = [seed] + _fwd_bwd(lambda *a: vf.vl_attention(*a, bias, True, True, 0.1, True, seed=seed),
                                  q, k, vv, vl, go_v, go_l)
        assert all(torch.equal(x, y) for x, y in zip(static[1:], eager[1:]))
    assert seeds[0] != seeds[1]


def _vlf_kernels(fn, calls=3):
    """Short names of the vlf_* kernels `calls` runs of `fn` launched, and how many kernels they launched through the
    library.  The profiler can lose the first kernel records of its window, so a small kernel opens it and `fn` runs
    several times inside it: the kernels a call runs are fixed by its inputs, so each run launches the same set."""
    from torch.profiler import ProfilerActivity, profile
    lib = _cabi.load()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        before = lib.msda_launch_count()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
        launched = lib.msda_launch_count() - before
    return {e.name.split("<")[0].split("(")[0].split("::")[-1] for e in prof.events() if "vlf_" in e.name}, launched


@pytest.mark.parametrize("T,stable,fused", [(17, False, True), (256, False, True), (257, False, False),
                                            (17, True, False)])
def test_profiler_shows_which_path_runs(T, stable, fused):
    q, k, vv, vl, _ = _inputs(1, 8, 300, T, 256, None)
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]

    def fn():
        o_v, o_l = vf.vl_attention(*leaves, None, True, True, 0.0, False, stable)
        (o_v.sum() + o_l.sum()).backward()

    fn()
    want = {"vlf_fwd_rows", "vlf_colstats", "vlf_fwd_cols", "vlf_reduce", "vlf_bwd_delta", "vlf_bwd_rows", "vlf_bwd_cols"}
    for _ in range(4):      # a window that misses records is profiled again; the path is fixed by the inputs
        names, launched = _vlf_kernels(fn)
        if not fused or want <= names:
            break
        time.sleep(0.5)
    # 4 forward + 5 backward launches per fused call (msda_vlfuse_forward_f32 / _backward_f32), none on the fallback
    assert launched == (3 * 9 if fused else 0), launched
    assert (want <= names) if fused else not names, names


def test_peak_memory_stays_below_one_logits_copy():
    B, H, S, T, D = 2, 8, 22323, 256, 256
    q, k, vv, vl, bias = _inputs(B, H, S, T, D, "partial")
    go_v, go_l = torch.randn_like(q), torch.randn_like(k)
    leaves = [t.requires_grad_(True) for t in (q, k, vv, vl)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    o_v, o_l = vf.vl_attention(*leaves, bias, True, True, 0.1, True)
    torch.autograd.backward((o_v, o_l), (go_v, go_l))
    torch.cuda.synchronize()
    outputs = sum(t.numel() * 4 for t in (o_v, o_l, *(x.grad for x in leaves)))
    extra = torch.cuda.max_memory_allocated() - base - outputs
    logits_copy = B * H * S * T * 4
    assert extra < logits_copy, (extra / 2 ** 20, logits_copy / 2 ** 20)
