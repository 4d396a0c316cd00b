"""GPU tests (-m gpu): this repo's mirrors of the reference's classes (``MSDeformAttn``, encoder / decoder layers of both
transformer files, the DINO decoder layer with its ``attn_masks``, ``DeformableReidHead``, the DINO decoder loop) and
geometry kernels on the sm_90a kernels, against the results of the REFERENCE's own classes and functions stored in
tests/golden/reference/*.npz (tests/refgolden.py): forward + input gradients + every parameter gradient, 2e-4 of scale
(fp32).  The reference classes initialise their parameters exactly like this repo's under the same seed, so both sides
run with the same weights.
"""
import os
import types
import warnings

import pytest
import torch

from tests import refgolden

pytestmark = pytest.mark.gpu

DEV = "cpu" if refgolden.RECORDING else "cuda"
if torch.cuda.is_available() or refgolden.RECORDING:
    from uninext_b200.modules import MSDeformAttn
    from uninext_b200.modules.deformable_layers import (DeformableTransformerDecoderLayer,
                                                        DeformableTransformerEncoderLayer)
    from uninext_b200.modules.deformable_transformer import (MLP, DeformableReidHead, DeformableTransformerDecoder,
                                                             get_reference_points, valid_ratios_from_masks)
    from uninext_b200.workloads import level_tensors

TOL = 2e-4
SHAPES = [(20, 28), (10, 14), (5, 7), (3, 4)]


def _classes(which):
    """The classes a test builds: the reference's (recording) or this repo's."""
    if refgolden.RECORDING:
        from tests import stage_reference
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = stage_reference.import_reference()
        t, dino = ref[2 + which], ref[3]
        return types.SimpleNamespace(MSDeformAttn=ref[1].MSDeformAttn, Enc=t.DeformableTransformerEncoderLayer,
                                     Dec=t.DeformableTransformerDecoderLayer, Reid=dino.DeformableReidHead,
                                     DecDino=dino.DeformableTransformerDecoderLayer,
                                     Decoder=dino.DeformableTransformerDecoder, MLP=dino.MLP, dino=dino)
    return types.SimpleNamespace(MSDeformAttn=MSDeformAttn, Enc=DeformableTransformerEncoderLayer,
                                 Dec=DeformableTransformerDecoderLayer, Reid=DeformableReidHead,
                                 DecDino=DeformableTransformerDecoderLayer, Decoder=DeformableTransformerDecoder, MLP=MLP)


def _rel(got, want):
    return ((got.detach().double() - want.detach().double()).abs().max() /
            want.detach().double().abs().max().clamp_min(1e-30)).item()


def _compare(group, build, run, inputs, which=0, tol=TOL):
    """build(classes) -> module; run(module, *leaf inputs) -> output.  Runs this repo's module and compares output, input
    grads and parameter grads with the reference's stored ones (recording: runs the reference's module and stores them)."""
    mod = build(_classes(which)).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in inputs]
    if not refgolden.RECORDING:
        from uninext_b200 import _cabi
        lib = _cabi.load()
        before = lib.msda_launch_count()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = run(mod, *leaves)
        go = torch.randn(out.shape, generator=torch.Generator().manual_seed(99)).to(out.device)
        out.backward(go)
    grads = {f"in{i}": l.grad for i, l in enumerate(leaves)}
    grads.update({"p:" + k: p.grad for k, p in mod.named_parameters()})
    if refgolden.RECORDING:
        refgolden.put(group, "out", out)
        for k, g in grads.items():
            assert g is not None, k
            refgolden.put(group, k, g)
        refgolden.flush(group)
        return
    assert lib.msda_launch_count() > before, "no kernel of libmsda_b200.so ran"
    want = refgolden.load(group)
    assert refgolden.rel(out, want, "out", group) < tol
    names = {k for k in want if k.startswith("p:") and not k.endswith((".scale", ".shape", ".index"))}
    assert names == {k for k in grads if k.startswith("p:")}
    for k, g in grads.items():
        assert g is not None, k
        assert refgolden.rel(g, want, k, group) < 5 * tol, k


def _pyramid_inputs(n, gen, c=256, masked=True):
    ss, lsi = level_tensors(SHAPES, DEV)
    s = sum(h * w for h, w in SHAPES)
    masks = []
    for h, w in SHAPES:
        m = torch.zeros(n, h, w, dtype=torch.bool)
        if masked:
            for b in range(n):
                m[b, int(h * (0.7 + 0.3 * b / max(1, n - 1))):, :] = True
                m[b, :, int(w * (0.6 + 0.4 * b / max(1, n - 1))):] = True
        masks.append(m.to(DEV))
    flat = torch.cat([m.flatten(1) for m in masks], 1)
    src = torch.randn(n, s, c, generator=gen).to(DEV)
    pos = torch.randn(n, s, c, generator=gen).to(DEV)
    return ss, lsi, masks, flat, src, pos


@pytest.mark.parametrize("which", [0, 1])          # 0: deformable_transformer.py, 1: deformable_transformer_dino.py
def test_reference_module_and_encoder_layer_on_dropin(which):
    g = torch.Generator().manual_seed(40 + which)
    n = 2
    ss, lsi, masks, flat, src, pos = _pyramid_inputs(n, g)
    vr = valid_ratios_from_masks(masks)
    refpts = get_reference_points(SHAPES, vr)
    # (a9) the module
    def build_attn(c):
        torch.manual_seed(1)
        m = c.MSDeformAttn(256, 4, 8, 4)
        with torch.no_grad():                     # the reference zero-initialises these two; make the test see them
            m.sampling_offsets.weight.normal_(0, 0.02)
            m.attention_weights.weight.normal_(0, 0.05)
        return m
    _compare(f"msdeformattn_{which}", build_attn, lambda m, q, x: m(q, refpts, x, ss, lsi, flat), [src + pos, src], which)

    # (a10) the encoder layer
    def build_layer(c):
        torch.manual_seed(2)
        m = c.Enc(256, 512, 0.0, "relu", 4, 8, 4)
        with torch.no_grad():
            m.self_attn.sampling_offsets.weight.normal_(0, 0.02)
            m.self_attn.attention_weights.weight.normal_(0, 0.05)
        return m
    _compare(f"encoder_layer_{which}", build_layer, lambda m, x: m(x, pos, refpts, ss, lsi, flat), [src], which)


def _decoder_inputs(n, q, gen):
    tgt = torch.randn(n, q, 256, generator=gen).to(DEV)
    qpos = torch.randn(n, q, 256, generator=gen).to(DEV)
    boxes = torch.cat((torch.rand(n, q, 2, generator=gen), 0.05 + 0.3 * torch.rand(n, q, 2, generator=gen)), -1).to(DEV)
    return tgt, qpos, boxes


@pytest.mark.parametrize("which", [0, 1])
def test_reference_decoder_layer_on_dropin(which):
    g = torch.Generator().manual_seed(50 + which)
    n, q = 2, 37
    ss, lsi, masks, flat, src, _ = _pyramid_inputs(n, g)
    vr = valid_ratios_from_masks(masks)
    tgt, qpos, boxes = _decoder_inputs(n, q, g)
    ref_in = boxes[:, :, None] * torch.cat((vr, vr), -1)[:, None]                      # _dino.py:451-452

    def build(c):
        torch.manual_seed(3)
        m = c.Dec(256, 512, 0.0, "relu", 4, 8, 4)
        with torch.no_grad():
            m.cross_attn.sampling_offsets.weight.normal_(0, 0.02)
            m.cross_attn.attention_weights.weight.normal_(0, 0.05)
        return m
    if which == 0:
        run = lambda m, t, x: m(t, qpos, ref_in, x, ss, lsi, flat)
    else:
        # DINO: denoising groups must not attend to each other (float mask, -inf where blocked; _dino.py:408-412)
        am = torch.zeros(q, q, device=DEV)
        am[:12, 12:] = float("-inf"); am[12:, :12] = float("-inf")
        run = lambda m, t, x: m(t, qpos, ref_in, x, ss, lsi, flat, am)
    _compare(f"decoder_layer_{which}", build, run, [tgt, src], which)


def test_reference_reid_head_on_dropin():
    g = torch.Generator().manual_seed(60)
    n, q = 2, 19
    ss, lsi, masks, flat, src, _ = _pyramid_inputs(n, g)
    vr = valid_ratios_from_masks(masks)
    tgt, _, boxes = _decoder_inputs(n, q, g)

    def build(c):
        torch.manual_seed(4)
        m = c.Reid(256, c.DecDino(256, 512, 0.0, "relu", 4, 8, 4), 2)
        with torch.no_grad():
            for layer in m.layers:
                layer.cross_attn.sampling_offsets.weight.normal_(0, 0.02)
                layer.cross_attn.attention_weights.weight.normal_(0, 0.05)
        return m
    _compare("reid_head", build, lambda m, t, x: m(t, boxes, x, ss, lsi, vr, None, flat, None), [tgt, src], 1)


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("refine", [True, False])
def test_reference_decoder_loop_on_dropin(refine, batched):
    """The whole DINO decoder loop (sine embedding -> ref_point_head -> layer -> box refinement, look_forward_twice),
    reference class on the drop-in against this repo's decoder, which projects the memory for all layers in ONE batched
    GEMM (SURVEY.md section 8 f-2)."""
    from uninext_b200.modules.ms_deform_attn import use_batched_value_proj
    was = use_batched_value_proj()
    use_batched_value_proj(batched)
    g = torch.Generator().manual_seed(80)
    n, q, nl = 2, 23, 3
    ss, lsi, masks, flat, src, _ = _pyramid_inputs(n, g)
    vr = valid_ratios_from_masks(masks)
    tgt, _, boxes = _decoder_inputs(n, q, g)

    def build(c):
        torch.manual_seed(6)
        m = c.Decoder(256, c.DecDino(256, 512, 0.0, "relu", 4, 8, 4), nl, return_intermediate=True, look_forward_twice=refine)
        if refine:      # the detector attaches the box heads to the decoder (iterative refinement), as the reference does
            m.bbox_embed = torch.nn.ModuleList(c.MLP(256, 256, 4, 3) for _ in range(nl))
        with torch.no_grad():
            for layer in m.layers:
                layer.cross_attn.sampling_offsets.weight.normal_(0, 0.02)
                layer.cross_attn.attention_weights.weight.normal_(0, 0.05)
        return m

    def run(m, t, x):
        hs, refs = m(t, boxes, x, ss, lsi, vr, None, flat, None)
        return torch.cat((hs.flatten(), refs.flatten()))
    try:
        _compare(f"decoder_loop_{int(refine)}", build, run, [tgt, src], 1)    # batched or not: the same reference result
    finally:
        use_batched_value_proj(was)


def test_batched_value_proj_equals_per_layer_projection():
    from uninext_b200.modules.ms_deform_attn import batched_value_proj
    g = torch.Generator().manual_seed(81)
    ss, lsi, masks, flat, src, _ = _pyramid_inputs(2, g)
    torch.manual_seed(7)
    mods = [MSDeformAttn(256, 4, 8, 4).to(DEV) for _ in range(3)]
    x = src.clone().requires_grad_(True)
    vals = batched_value_proj(mods, x, flat)
    want = [m.value_proj(src).masked_fill(flat[..., None], 0.0) for m in mods]
    for a, b in zip(vals, want):
        assert _rel(a, b) < 1e-5
    sum((v * (i + 1)).sum() for i, v in enumerate(vals)).backward()
    gw = [m.value_proj.weight.grad.clone() for m in mods]
    gx = x.grad.clone()
    for m in mods:
        m.zero_grad()
    x2 = src.clone().requires_grad_(True)
    sum((m.value_proj(x2).masked_fill(flat[..., None], 0.0) * (i + 1)).sum() for i, m in enumerate(mods)).backward()
    assert _rel(gx, x2.grad) < 1e-4
    for a, m in zip(gw, mods):
        assert _rel(a, m.value_proj.weight.grad) < 1e-4


def test_layers_run_fp32_under_autocast_like_reference():
    """custom_fwd(cast_inputs=float32) on the reference layers (deformable_transformer.py:351,398): under autocast the
    whole layer, FFN included, computes in fp32 -- ours must give the fp32 result too."""
    g = torch.Generator().manual_seed(70)
    ss, lsi, masks, flat, src, pos = _pyramid_inputs(1, g, masked=False)
    refpts = get_reference_points(SHAPES, valid_ratios_from_masks(masks))
    torch.manual_seed(5)
    layer = DeformableTransformerEncoderLayer(256, 512, 0.0, "relu", 4, 8, 4).to(DEV)
    want = layer(src, pos, refpts, ss, lsi, None)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        got = layer(src.bfloat16(), pos, refpts, ss, lsi, None)
    assert got.dtype == torch.float32
    assert _rel(got, layer(src.bfloat16().float(), pos, refpts, ss, lsi, None)) < 1e-5
    assert _rel(got, want) < 2e-2            # only the bf16 rounding of the input separates them


def test_geometry_kernels_match_reference_functions():
    """f-3 on the GPU: reference points, two-stage proposals and the sine position embedding as single kernels against the
    stored results of the reference's own functions (deformable_transformer_dino.py:132-171,289-301,612-646)."""
    from uninext_b200.modules.deformable_transformer import gen_encoder_output_proposals, get_sine_pos_embed
    g = torch.Generator().manual_seed(90)
    n = 3
    ss, lsi, masks, flat, src, _ = _pyramid_inputs(n, g)

    class Holder(torch.nn.Module):          # the reference method reads self.enc_output / self.enc_output_norm
        def __init__(self):
            super().__init__()
            self.enc_output = torch.nn.Linear(256, 256)
            self.enc_output_norm = torch.nn.LayerNorm(256)
    torch.manual_seed(91)
    h = Holder().to(DEV)
    pos = torch.rand(2, 19, 4, generator=g).to(DEV)
    go = torch.randn(2, 19, 512, generator=g).to(DEV)
    if refgolden.RECORDING:
        dino = _classes(1).dino
        holder = dino.DeformableTransformerVLDINO.__new__(dino.DeformableTransformerVLDINO)
        vr = torch.stack([dino.DeformableTransformerVLDINO.get_valid_ratio(holder, m) for m in masks], 1)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            refpts = dino.DeformableTransformerEncoderVL.get_reference_points(ss, vr, device=DEV)
            mem, prop = dino.DeformableTransformerVLDINO.gen_encoder_output_proposals(h, src, flat, ss)
        b = pos.clone().requires_grad_(True)
        y = dino.get_sine_pos_embed(b)
        y.backward(go)
        for k, t in (("vr", vr), ("refpts", refpts), ("mem", mem), ("prop", prop.masked_fill(torch.isinf(prop), 0.0)),
                     ("prop_inf", torch.isinf(prop).double()), ("sine", y), ("sine_grad", b.grad),
                     ("sine_64_20", dino.get_sine_pos_embed(pos[..., :2], 64, 20, False))):
            refgolden.put("geometry", k, t)
        refgolden.flush("geometry")
        return
    from uninext_b200 import _cabi
    want = refgolden.load("geometry")
    want_vr = torch.from_numpy(want["vr"]).reshape(tuple(want["vr.shape"])).float().to(DEV)
    lib = _cabi.load()
    n0 = lib.msda_launch_count()
    got = get_reference_points(ss, want_vr)
    assert lib.msda_launch_count() - n0 == 1
    close = lambda t, k, rtol, atol: torch.allclose(torch.from_numpy(refgolden.sample(t, want, k, "geometry")),
                                                    torch.from_numpy(want[k]), rtol=rtol, atol=atol)
    assert tuple(got.shape) == tuple(want["refpts.shape"]) and close(got, "refpts", 1e-6, 1e-7)

    n0 = lib.msda_launch_count()
    prop, keep = gen_encoder_output_proposals(flat, ss)
    assert lib.msda_launch_count() - n0 == 2
    inf = torch.isinf(prop)
    assert tuple(prop.shape) == tuple(want["prop.shape"])
    assert (refgolden.sample(inf.double(), want, "prop_inf", "geometry") == want["prop_inf"]).all()
    assert close(prop.masked_fill(inf, 0.0), "prop", 1e-5, 1e-5)
    got_mem = h.enc_output_norm(h.enc_output(src.masked_fill(~keep, 0.0)))
    assert close(got_mem, "mem", 1e-4, 1e-5)

    a = pos.clone().requires_grad_(True)
    ya = get_sine_pos_embed(a)
    assert tuple(ya.shape) == tuple(want["sine.shape"]) and close(ya, "sine", 0, 2e-5)
    ya.backward(go)
    assert refgolden.rel(a.grad, want, "sine_grad", "geometry") < 1e-4
    assert close(get_sine_pos_embed(pos[..., :2], 64, 20, False), "sine_64_20", 0, 2e-5)
