"""CPU tests: the host-side mirrors of the reference's helpers around the op (reference points, proposals, sine position
embedding, MLP, layer signatures) against stored results of the REFERENCE functions themselves
(deformable_transformer_dino.py; tests/golden/reference/mirrors.npz, tests/refgolden.py)."""
import inspect

import numpy as np
import torch

from tests import refgolden

GROUP = "mirrors"
SHAPES = [(12, 20), (6, 10), (3, 5), (2, 3)]


def _masks(n, shapes, gen):
    """Padding masks the way the reference pads a batch: valid region top-left, padded right / bottom."""
    out = []
    fr = torch.rand(n, 2, generator=gen) * 0.5 + 0.5
    for h, w in shapes:
        m = torch.ones(n, h, w, dtype=torch.bool)
        for b in range(n):
            vh, vw = max(1, int(round(h * fr[b, 0].item()))), max(1, int(round(w * fr[b, 1].item())))
            m[b, :vh, :vw] = False
        out.append(m)
    return out


def _sine_inputs():
    g = torch.Generator().manual_seed(0)
    pos = torch.rand(2, 7, 4, generator=g)
    x = torch.randn(3, 5, 512, generator=g)
    return pos, x


def _proposal_inputs():
    g = torch.Generator().manual_seed(3)
    masks = _masks(2, SHAPES, g)
    flat = torch.cat([m.flatten(1) for m in masks], 1)
    memory = torch.randn(2, flat.shape[1], 16, generator=g)

    class Holder(torch.nn.Module):          # the reference method reads self.enc_output / self.enc_output_norm
        def __init__(self):
            super().__init__()
            self.enc_output = torch.nn.Linear(16, 16)
            self.enc_output_norm = torch.nn.LayerNorm(16)
    torch.manual_seed(4)
    return flat, memory, Holder()


def _signature(f):
    """Positional parameter names after self (keyword-only extras are this repo's extensions)."""
    return [n for n, p in inspect.signature(f).parameters.items() if p.kind != p.KEYWORD_ONLY][1:]


def record():
    """Store the reference's results (tests/golden/make_reference_golden.py)."""
    from tests import stage_reference
    dino = stage_reference.import_reference()[3]
    put = lambda k, t: refgolden.put(GROUP, k, t)
    pos, x = _sine_inputs()
    for xy in (True, False):
        put(f"sine_{int(xy)}", dino.get_sine_pos_embed(pos, exchange_xy=xy))
    put("sine_64_20", dino.get_sine_pos_embed(pos[..., :2], 64, 20))
    torch.manual_seed(1)
    put("mlp", dino.MLP(512, 256, 256, 2)(x))
    masks = _masks(3, SHAPES, torch.Generator().manual_seed(2))
    holder = dino.DeformableTransformerVLDINO.__new__(dino.DeformableTransformerVLDINO)     # get_valid_ratio uses no state
    vr = torch.stack([dino.DeformableTransformerVLDINO.get_valid_ratio(holder, m) for m in masks], 1)
    put("valid_ratios", vr)
    put("reference_points", dino.DeformableTransformerEncoderVL.get_reference_points(torch.as_tensor(SHAPES), vr, device="cpu"))
    flat, memory, h = _proposal_inputs()
    mem, prop = dino.DeformableTransformerVLDINO.gen_encoder_output_proposals(h, memory, flat, torch.as_tensor(SHAPES))
    put("proposal_memory", mem)
    put("proposals", prop.masked_fill(torch.isinf(prop), 0.0))
    put("proposals_inf", torch.isinf(prop).double())
    for name, cls in (("enc", dino.DeformableTransformerEncoderLayer), ("dec", dino.DeformableTransformerDecoderLayer),
                      ("reid", dino.DeformableReidHead)):
        refgolden.put_raw(GROUP, f"signature_{name}", np.array(_signature(cls.forward)))
    head = dino.DeformableReidHead(256, dino.DeformableTransformerDecoderLayer(256, 512, 0.0, "relu", 4, 8, 4), 2)
    sd = head.state_dict()
    refgolden.put_raw(GROUP, "reid_keys", np.array(sorted(sd)))
    refgolden.put_raw(GROUP, "reid_shapes", np.array([",".join(map(str, sd[k].shape)) for k in sorted(sd)]))
    refgolden.flush(GROUP)


def _close(got, want, key, rtol, atol):
    assert tuple(got.shape) == tuple(want[key + ".shape"]), key
    return np.allclose(refgolden.sample(got, want, key, GROUP), want[key], rtol=rtol, atol=atol)


def test_sine_pos_embed_and_mlp():
    from uninext_b200.modules.deformable_transformer import MLP, get_sine_pos_embed
    want = refgolden.load(GROUP)
    pos, x = _sine_inputs()
    for xy in (True, False):
        assert _close(get_sine_pos_embed(pos, exchange_xy=xy), want, f"sine_{int(xy)}", 0, 1e-6)
    assert _close(get_sine_pos_embed(pos[..., :2], 64, 20), want, "sine_64_20", 1e-5, 1e-6)
    torch.manual_seed(1)                     # the reference MLP initialises exactly like this one under the same seed
    got = MLP(512, 256, 256, 2)(x)
    assert tuple(got.shape) == tuple(want["mlp.shape"])
    assert np.array_equal(refgolden.sample(got, want, "mlp", GROUP), want["mlp"])


def test_reference_points_and_valid_ratios():
    from uninext_b200.modules.deformable_transformer import get_reference_points, valid_ratios_from_masks
    want = refgolden.load(GROUP)
    masks = _masks(3, SHAPES, torch.Generator().manual_seed(2))
    vr = valid_ratios_from_masks(masks)
    assert tuple(vr.shape) == tuple(want["valid_ratios.shape"])
    assert np.array_equal(refgolden.sample(vr, want, "valid_ratios", GROUP), want["valid_ratios"])
    ss = torch.as_tensor(SHAPES)
    assert _close(get_reference_points(ss, vr), want, "reference_points", 1e-6, 1e-7)
    assert _close(get_reference_points(SHAPES, vr), want, "reference_points", 1e-6, 1e-7)     # cached grid, list input


def test_encoder_output_proposals():
    from uninext_b200.modules.deformable_transformer import gen_encoder_output_proposals
    want = refgolden.load(GROUP)
    flat, memory, h = _proposal_inputs()
    prop, keep = gen_encoder_output_proposals(flat, SHAPES)
    inf = torch.isinf(prop)
    assert tuple(prop.shape) == tuple(want["proposals.shape"])
    assert np.array_equal(refgolden.sample(inf.double(), want, "proposals_inf", GROUP), want["proposals_inf"])
    assert _close(prop.masked_fill(inf, 0.0), want, "proposals", 1e-5, 1e-6)
    got_mem = h.enc_output_norm(h.enc_output(memory.masked_fill(~keep, 0.0)))
    assert _close(got_mem, want, "proposal_memory", 1e-5, 1e-6)


def test_layer_signatures_match_reference():
    from uninext_b200.modules.deformable_layers import (DeformableTransformerDecoderLayer,
                                                        DeformableTransformerEncoderLayer)
    from uninext_b200.modules.deformable_transformer import DeformableReidHead
    want = refgolden.load(GROUP)
    # positional signature = the reference's; keyword-only extras (projected_value) are this repo's extensions
    assert _signature(DeformableTransformerEncoderLayer.forward) == list(want["signature_enc"])
    assert _signature(DeformableTransformerDecoderLayer.forward) == list(want["signature_dec"])
    assert _signature(DeformableReidHead.forward) == list(want["signature_reid"])
    ours = DeformableReidHead(256, DeformableTransformerDecoderLayer(256, 512, 0.0, "relu", 4, 8, 4), 2)
    sd = ours.state_dict()
    assert sorted(sd) == list(want["reid_keys"])
    assert [",".join(map(str, sd[k].shape)) for k in sorted(sd)] == list(want["reid_shapes"])
