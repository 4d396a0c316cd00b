"""GPU tests of the two-stage query selection (uninext_b200/modules/two_stage.py on the kernels of msda_twostage.cuh):
against the reference's stored results, against an fp64 restatement with a stable sort at the sizes UNINEXT runs,
exact tie order, determinism, CUDA-graph replay and the launch count."""
import math

import pytest
import torch

from tests import two_stage_case as tc
from tests.test_two_stage_host import compare_with_golden, run_case
from uninext_b200.modules.deformable_transformer import MLP, gen_encoder_output_proposals
from uninext_b200.modules.two_stage import Still_Classifier, VL_Align, two_stage_select
from uninext_b200.workloads import CONFIGS

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name", list(tc.CASES))
def test_matches_reference_golden(name):
    out, g_mem, grads = run_case(name, DEV)
    torch.cuda.synchronize()
    close = compare_with_golden(name, out, g_mem, grads, 2e-4)
    assert close <= 0.02 * tc.N * tc.K, close                  # neighbours within 1e-5 of the scale are rare


# ---- user sizes against an fp64 restatement --------------------------------------------------------------------------
def user_problem(cfg, head, seed=0, box_layers=1):
    """N = 2 at the config's pyramid, image 1 padded to 75 % x 66 %; random modules of the given head (VL_Align at its
    default scale, with the clamp on: no logit comes near it).  bbox_embed has one layer unless asked otherwise: among
    the 2 x 256 ReLUs of the reference's three-layer MLP over 44646 rows, some input lies within rounding of 0, takes the
    other branch in fp64 than in fp32 and changes that row's gradient by O(1) -- a property of the MLP, not of the path
    under test (the three-layer MLP is compared with the reference's results on the test pyramid)."""
    c = CONFIGS[cfg]
    masks = []
    for b in range(2):
        lv = []
        for h, w in c.shapes:
            m = torch.zeros(h, w, dtype=torch.bool)
            if b == 1:
                m[math.ceil(0.66 * h):, :] = True
                m[:, math.ceil(0.75 * w):] = True
            lv.append(m.flatten())
        masks.append(torch.cat(lv))
    return make_problem(c.shapes, torch.stack(masks), head, seed, box_layers)


def make_problem(shapes, mask, head, seed=0, box_layers=1):
    """user_problem's modules and inputs at any pyramid: mask [N, S] bool; -> (shapes, mods, x)."""
    n, s = mask.shape
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mods = {"enc_output": torch.nn.Linear(256, 256), "enc_output_norm": torch.nn.LayerNorm(256),
            "class_embed": Still_Classifier(256) if head == "still" else VL_Align(256, 768, 0.0, clamp_dot_product=True),
            "bbox_embed": MLP(256, 256, 4, box_layers)}
    with torch.no_grad():
        mods["enc_output_norm"].weight.normal_(1.0, 0.1)
        mods["enc_output_norm"].bias.normal_(0.0, 0.1)
    for m in mods.values():
        m.to(DEV)
    x = {"memory": torch.randn(n, s, 256, generator=g).to(DEV), "mask": mask.to(DEV),
         "lang_feat_pool": torch.randn(n, 768, generator=g).to(DEV)}
    return shapes, mods, x


def run_fused(shapes, mods, x, k, cot=None):
    memory = x["memory"].clone().requires_grad_(True)
    for m in mods.values():
        m.zero_grad(set_to_none=True)
    out = two_stage_select(memory, x["mask"], shapes, mods["enc_output"], mods["enc_output_norm"], mods["class_embed"],
                           mods["bbox_embed"], k, x["lang_feat_pool"])
    if cot is None:
        return out
    tc.backward(out, cot)
    return out, memory.grad, {f"{p}.{n}": t.grad for p, m in mods.items() for n, t in m.named_parameters()}


def restated_fp64(shapes, mods, x, idx, cot):
    """The reference's chain in fp64, gathering at the given indices; -> (class, coord, ref, order, memory grad, grads)."""
    import copy
    m64 = {k: copy.deepcopy(m).double() for k, m in mods.items()}
    memory = x["memory"].double().requires_grad_(True)
    prop, keep = gen_encoder_output_proposals(x["mask"].cpu(), shapes)
    prop, keep = prop.to(DEV).double(), keep.to(DEV)
    om = m64["enc_output_norm"](m64["enc_output"](memory.masked_fill(~keep, 0.0)))
    cls = m64["class_embed"](om, x["lang_feat_pool"].double().unsqueeze(1))
    coord = m64["bbox_embed"](om) + prop
    order = torch.sort(cls[..., 0], dim=1, descending=True, stable=True)[1]
    ref = torch.gather(coord, 1, idx.unsqueeze(-1).repeat(1, 1, 4)).sigmoid()
    torch.autograd.backward((cls, coord, ref), (cot["g_class"].double(), cot["g_coord"].double(), cot["g_ref"].double()))
    grads = {f"{p}.{n}": t.grad for p, m in m64.items() for n, t in m.named_parameters()}
    return cls.detach(), coord.detach(), ref.detach(), order, memory.grad, grads


def rel(a, b):
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("cfg,k,head", [("cfg2", 300, "still"), ("cfg2", 900, "vl"), ("cfg3", 900, "still"),
                                        ("cfg2", "S", "vl")])
def test_user_sizes_against_fp64(cfg, k, head):
    shapes, mods, x = user_problem(cfg, head)
    s = x["memory"].shape[1]
    check_against_fp64(shapes, mods, x, s if k == "S" else k)


def check_against_fp64(shapes, mods, x, k):
    """Run the kernels forward and backward on random cotangents and assert they match restated_fp64: values and
    gradients within 2e-4 of scale, the fp64 stable order, the top-k set.  -> (outputs, memory grad, grads, cot)."""
    n, s = x["memory"].shape[:2]
    g = torch.Generator().manual_seed(7)
    cot = {"g_class": torch.randn(n, s, 1, generator=g).to(DEV), "g_coord": torch.randn(n, s, 4, generator=g).to(DEV),
           "g_ref": torch.randn(n, k, 4, generator=g).to(DEV)}
    (cls, coord, ref, idx), g_mem, grads = run_fused(shapes, mods, x, k, cot)
    w_cls, w_coord, w_ref, order, w_mem, w_grads = restated_fp64(shapes, mods, x, idx, cot)
    assert idx.shape == (n, k) and idx.dtype == torch.int64
    assert rel(cls, w_cls) < 2e-4
    inf = torch.isinf(w_coord)
    assert torch.equal(torch.isinf(coord), inf) and rel(coord[~inf], w_coord[~inf]) < 2e-4
    assert (ref.double() - w_ref).abs().max().item() < 2e-4
    assert rel(g_mem, w_mem) < 2e-4
    for key, v in w_grads.items():
        assert rel(grads[key], v) < 2e-4, key
    # The fp64 stable order wherever neighbouring ranks are further apart than twice the fp32 logits' largest error
    # (closer ones may swap), and exact ties (the dropped rows) by ascending row.
    thr = 2 * (cls.double() - w_cls).abs().max().item()
    for b in range(n):
        lg = w_cls[b, order[b, :k], 0]
        gap = torch.cat((lg[:-1] - lg[1:], lg.new_tensor([math.inf])))
        prev = torch.cat((lg.new_tensor([math.inf]), gap[:-1]))
        clear = ((gap > thr) | (gap == 0)) & ((prev > thr) | (prev == 0))
        assert torch.equal(idx[b][clear], order[b, :k][clear]), b
        if k < s:                               # the selected set is the top k
            assert w_cls[b, idx[b], 0].min() >= w_cls[b, order[b, k:], 0].max() - thr
    return (cls, coord, ref, idx), g_mem, grads, cot


def test_exact_ties_invalid_rows_and_nan():
    """gamma = 0: every row's om is beta, every logit is equal: the order is ascending row.  A NaN logit ranks first.
    Selected rows with +inf proposals give reference points 1 and a zero gradient."""
    shapes, mods, x = user_problem("cfg2", "still", seed=3)
    n, s = x["memory"].shape[:2]
    with torch.no_grad():
        mods["enc_output_norm"].weight.zero_()
    k = 2000
    cls, coord, ref, idx = run_fused(shapes, mods, x, k)
    assert (cls == cls[0, 0]).all()
    want = torch.arange(k, device=DEV).expand(n, k)
    assert torch.equal(idx, want)
    assert torch.allclose(ref, torch.gather(coord, 1, want.unsqueeze(-1).repeat(1, 1, 4)).sigmoid(), rtol=0, atol=1e-6)
    inf = torch.isinf(coord[1, :k]).all(-1)
    assert inf.any() and (ref[1][inf] == 1).all()
    # the gradient of the selected invalid rows: the selection adds exactly zero to what coord_unact brings
    memory = x["memory"].clone().requires_grad_(True)
    box_grad = {}
    def keep_grad(module, inputs, output):
        output.register_hook(lambda g: box_grad.update(g=g))

    h = mods["bbox_embed"].layers[-1].register_forward_hook(keep_grad)
    try:
        out = two_stage_select(memory, x["mask"], shapes, mods["enc_output"], mods["enc_output_norm"],
                               mods["class_embed"], mods["bbox_embed"], k)
        torch.autograd.backward(out[2], torch.ones_like(out[2]))
    finally:
        h.remove()
    gb = box_grad["g"][1, :k]
    assert (gb[inf] == 0).all() and (gb[~inf] > 0).all()
    # NaN ranks above everything, the other rows keep their order
    r = 50 * shapes[0][1] + 50                              # a row with a valid proposal: its memory reaches the head
    with torch.no_grad():
        x["memory"][0, r] = float("nan")
        mods["enc_output_norm"].weight.fill_(1.0)
        mods["enc_output"].weight.zero_()                   # every other logit stays equal
    cls, coord, ref, idx = run_fused(shapes, mods, x, 50)
    assert torch.isnan(cls[0, r, 0]) and idx[0, 0].item() == r
    assert torch.equal(idx[0, 1:], torch.arange(49, device=DEV))


def test_deterministic_algorithms_and_bitwise_repeat(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    shapes, mods, x = user_problem("cfg2", "vl")
    n, s = x["memory"].shape[:2]
    cot = {"g_class": torch.randn(n, s, 1, device=DEV), "g_coord": torch.randn(n, s, 4, device=DEV),
           "g_ref": torch.randn(n, 900, 4, device=DEV)}

    def flat():
        out, g_mem, grads = run_fused(shapes, mods, x, 900, cot)
        return [t.detach().clone() for t in (*out, g_mem, *grads.values())]

    torch.use_deterministic_algorithms(True)
    try:
        a = flat()                                          # raises if anything on the path alerts
        b = flat()
    finally:
        torch.use_deterministic_algorithms(False)
    c = flat()
    assert all(torch.equal(u, v) for u, v in zip(a, b)) and all(torch.equal(u, v) for u, v in zip(a, c))


def test_cuda_graph_replay_equals_eager():
    shapes, mods, x = user_problem("cfg2", "still")
    n, s = x["memory"].shape[:2]
    cot = {"g_class": torch.randn(n, s, 1, device=DEV), "g_coord": torch.randn(n, s, 4, device=DEV),
           "g_ref": torch.randn(n, 300, 4, device=DEV)}
    memory = x["memory"].clone().requires_grad_(True)
    leaves = [memory] + [p for m in mods.values() for p in m.parameters()]

    def step():
        out = two_stage_select(memory, x["mask"], shapes, mods["enc_output"], mods["enc_output_norm"],
                               mods["class_embed"], mods["bbox_embed"], 300)
        grads = torch.autograd.grad(out[:3], leaves, (cot["g_class"], cot["g_coord"], cot["g_ref"]))
        return [*out, *grads]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    with torch.no_grad():
        memory.copy_(torch.randn_like(memory))
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    assert all(torch.equal(u, v) for u, v in zip(static, eager))


def test_kernels_ran_and_other_inputs_raise():
    from uninext_b200 import _cabi
    lib = _cabi.load()
    shapes, mods, x = user_problem("cfg2", "still")
    out = run_fused(shapes, mods, x, 300)                   # warm: level tables cached
    before = lib.msda_launch_count()
    out = run_fused(shapes, mods, x, 300)
    after_fwd = lib.msda_launch_count()
    torch.autograd.backward(out[:3], [torch.ones_like(t) for t in out[:3]])
    torch.cuda.synchronize()
    after_bwd = lib.msda_launch_count()
    assert after_fwd - before == 4          # valid counts, proposals, head forward, select forward
    assert after_bwd - after_fwd == 3       # select backward, head backward, its fixed-order reduction
    with pytest.raises(ValueError, match="fp32"):
        two_stage_select(x["memory"].double(), x["mask"], shapes, mods["enc_output"], mods["enc_output_norm"],
                         mods["class_embed"], mods["bbox_embed"], 300)
    with pytest.raises(ValueError, match="width"):
        m128 = torch.nn.Linear(128, 128).to(DEV)
        two_stage_select(x["memory"][..., :128].contiguous(), x["mask"], shapes, m128, torch.nn.LayerNorm(128).to(DEV),
                         mods["class_embed"], mods["bbox_embed"], 300)
    with pytest.raises(RuntimeError, match="out of range"):
        run_fused(shapes, mods, x, x["memory"].shape[1] + 1)
