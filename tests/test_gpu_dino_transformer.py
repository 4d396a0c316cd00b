"""GPU tests of the encoder's input preparation and DINO's whole transformer (uninext_b200/modules/dino_transformer.py on
the kernels of msda_flatten.cuh and the rest of the library): against the reference's stored results; flatten_levels
bit for bit against the reference's torch chain at the sizes UNINEXT runs; the launch count; determinism; CUDA-graph
replay and no host synchronisation of the whole transformer."""
import math

import pytest
import torch

from tests import dino_case as dc
from tests.test_dino_transformer_host import build_model, compare_with_golden, run_case
from uninext_b200.modules.dino_transformer import flatten_levels
from uninext_b200.workloads import CONFIGS

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


@pytest.mark.parametrize("name", list(dc.CASES))
def test_matches_reference_golden(name, no_tf32):
    out, leaves, params, g = run_case(name, DEV)
    torch.cuda.synchronize()
    compare_with_golden(out, leaves, params, g, 2e-4)


# ---- flatten_levels against the reference's chain --------------------------------------------------------------------
def pyramid(cfg, c, seed=0):
    """N = 2 at the config's pyramid, image 1 padded to 75 % x 66 % of each level; -> (srcs, masks, pos, level_embed)."""
    g = torch.Generator().manual_seed(seed)
    shapes = CONFIGS[cfg].shapes
    srcs = [torch.randn(2, c, h, w, generator=g).to(DEV) for h, w in shapes]
    pos = [torch.randn(2, c, h, w, generator=g).to(DEV) for h, w in shapes]
    masks = []
    for h, w in shapes:
        m = torch.zeros(2, h, w, dtype=torch.bool)
        m[1, math.ceil(0.66 * h):, :] = True
        m[1, :, math.ceil(0.75 * w):] = True
        masks.append(m.to(DEV))
    return srcs, masks, pos, torch.randn(len(shapes), c, generator=g).to(DEV)


def reference_chain(srcs, masks, pos_embeds, level_embed):
    """deformable_transformer_dino.py:181-201 as the reference writes it."""
    src_flatten, mask_flatten, lvl_pos_embed_flatten, spatial_shapes = [], [], [], []
    for lvl, (src, mask, pos_embed) in enumerate(zip(srcs, masks, pos_embeds)):
        bs, c, h, w = src.shape
        spatial_shapes.append((h, w))
        src_flatten.append(src.flatten(2).transpose(1, 2))
        mask_flatten.append(mask.flatten(1))
        lvl_pos_embed_flatten.append(pos_embed.flatten(2).transpose(1, 2) + level_embed[lvl].view(1, 1, -1))
    src_flatten, mask_flatten = torch.cat(src_flatten, 1), torch.cat(mask_flatten, 1)
    lvl_pos_embed_flatten = torch.cat(lvl_pos_embed_flatten, 1)
    spatial_shapes = torch.as_tensor(spatial_shapes, dtype=torch.long, device=src_flatten.device)
    level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))

    def get_valid_ratio(mask):
        _, H, W = mask.shape
        valid_H, valid_W = torch.sum(~mask[:, :, 0], 1), torch.sum(~mask[:, 0, :], 1)
        return torch.stack([valid_W.float() / W, valid_H.float() / H], -1)

    valid_ratios = torch.stack([get_valid_ratio(m) for m in masks], 1)
    return src_flatten, mask_flatten, lvl_pos_embed_flatten, spatial_shapes, level_start_index, valid_ratios


def _leaves(srcs, pos, le):
    return [s.clone().requires_grad_(True) for s in srcs], [p.clone().requires_grad_(True) for p in pos], \
        le.clone().requires_grad_(True)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
@pytest.mark.parametrize("c", [256, 4 * 63])
def test_flatten_levels_is_the_reference_chain_bit_for_bit(cfg, c):
    srcs, masks, pos, le = pyramid(cfg, c)
    outs = {}
    for arm, fn in (("kernel", flatten_levels), ("reference", reference_chain)):
        s, p, e = _leaves(srcs, pos, le)
        out = fn(s, masks, p, e)
        g = torch.Generator(device=DEV).manual_seed(1)
        cot_src = torch.randn(out[0].shape, device=DEV, generator=g)
        cot_pos = torch.randn(out[2].shape, device=DEV, generator=g)
        torch.autograd.backward((out[0], out[2]), (cot_src, cot_pos))
        outs[arm] = (out, [t.grad for t in s], [t.grad for t in p], e.grad, cot_pos)
    (ko, ks, kp, ke, cot), (ro, rs, rp, re, _) = outs["kernel"], outs["reference"]
    for i, (a, b) in enumerate(zip(ko, ro)):
        assert a.dtype == b.dtype and torch.equal(a, b), i
    for a, b in zip(ks + kp, rs + rp):
        assert torch.equal(a, b)
    # grad_level_embed against the fp64 sum over images and each level's positions
    starts = [0]
    for h, w in CONFIGS[cfg].shapes:
        starts.append(starts[-1] + h * w)
    want = torch.stack([cot[:, a:b].double().sum((0, 1)) for a, b in zip(starts[:-1], starts[1:])])
    assert (ke.double() - want).abs().max().item() <= 1e-6 * want.abs().max().item()


def test_flatten_levels_grad_level_embed_is_deterministic():
    srcs, masks, pos, le = pyramid("cfg2", 256)
    grads = []
    with torch.no_grad():
        cot = torch.randn(2, CONFIGS["cfg2"].S, 256, device=DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(3):
            s, p, e = _leaves(srcs, pos, le)
            out = flatten_levels(s, masks, p, e)
            out[2].backward(cot)
            grads.append(e.grad)
    finally:
        torch.use_deterministic_algorithms(prev)
    for g in grads[1:]:
        assert torch.equal(g, grads[0])


def test_launch_count_of_the_input_preparation():
    """Forward: the flattening kernel and msda_valid_counts.  Backward with every gradient: the transpose and the
    reduction; without level_embed's: the transpose alone."""
    from uninext_b200 import _cabi
    lib = _cabi.load()
    srcs, masks, pos, le = pyramid("cfg2", 256)
    for want_le, bwd in ((True, 2), (False, 1)):
        s, p, e = _leaves(srcs, pos, le)
        e.requires_grad_(want_le)
        flatten_levels(s, masks, p, e)                                    # warm-up: level tables built
        before = lib.msda_launch_count()
        out = flatten_levels(s, masks, p, e)
        mid = lib.msda_launch_count()
        torch.autograd.backward((out[0], out[2]), (torch.ones_like(out[0]), torch.ones_like(out[2])))
        torch.cuda.synchronize()
        assert (mid - before, lib.msda_launch_count() - mid) == (2, bwd)


def test_flatten_levels_writes_only_the_wanted_gradients():
    srcs, masks, pos, le = pyramid("cfg3", 256)
    s = [t.clone().requires_grad_(True) for t in srcs]
    out = flatten_levels(s, masks, pos, le)
    (out[0].sum() + out[2].sum()).backward()
    assert all(torch.equal(t.grad, torch.ones_like(t)) for t in s)


# ---- the whole transformer: CUDA graph and host synchronisation ------------------------------------------------------
def _step(model, name, x, seed):
    params = [p for p in model.parameters() if p.requires_grad]
    with torch.no_grad():
        cot = {k: v.to(DEV) for k, v in dc.cotangents(dc.run(model, name, x, DEV)[0], seed).items()}

    def fn():
        out, leaves = dc.run(model, name, x, DEV)
        keys = [k for k, v in out.items() if v.requires_grad]
        ins = leaves["srcs"] + leaves["pos_embeds"] + [leaves["hidden"]]
        grads = torch.autograd.grad([out[k] for k in keys], ins + params, [cot[k] for k in keys],
                                    allow_unused=True)
        return [out[k].detach() for k in sorted(out)] + [g for g in grads if g is not None]
    return fn


def test_whole_transformer_graph_replay_equals_eager(no_tf32):
    from uninext_b200.graphs import GraphedStep
    name = "dn"
    model, _, seed, _ = build_model(name, DEV)
    x = {k: (v.to(DEV) if torch.is_tensor(v) else [t.to(DEV) for t in v]) for k, v in dc.inputs(name, seed).items()}
    fn = _step(model, name, x, seed)
    eager = fn()
    step = GraphedStep(fn)
    got = step.replay()
    torch.cuda.synchronize()
    assert len(got) == len(eager)
    for a, b in zip(got, eager):
        fin = torch.isfinite(b)
        assert torch.equal(fin, torch.isfinite(a))
        assert (a[fin] - b[fin]).abs().max().item() <= 1e-5 * max(b[fin].abs().max().item(), 1e-30)


def test_whole_transformer_does_not_synchronise_after_warm_up():
    name = "production"
    model, _, seed, _ = build_model(name, DEV)
    model.train()
    x = {k: (v.to(DEV) if torch.is_tensor(v) else [t.to(DEV) for t in v]) for k, v in dc.inputs(name, seed).items()}
    fn = _step(model, name, x, seed)
    fn()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
