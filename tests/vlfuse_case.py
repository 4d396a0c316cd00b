"""The early-fusion block cases pinned to the reference (tests/golden/reference/vlfuse_*.npz): weights, inputs and the
output gradients come from numpy's PCG64 with fixed seeds, so the recorder and the tests build them identically.

UNINEXT dims (v 256, l 768, embed 2048, 8 heads), S = 2125 (the cfg1 pyramid), T = 17, B = 2.  Stored: every 17th image
token of the visual output and its input gradient, the whole text output and gradient, the small parameter gradients in
full and each weight gradient's product with a fixed [in, 4] matrix (a sketch that keeps the fixture small)."""
import numpy as np
import torch

V_DIM, L_DIM, EMBED, HEADS = 256, 768, 2048, 8
B, S, T = 2, 2125, 17
ROW_STRIDE = 17
CASES = {
    "partial": dict(seed=11, lengths=(17, 9), qk_gain=1.0),     # second element padded after 9 tokens
    "padded": dict(seed=12, lengths=(12, 0), qk_gain=1.0),      # second element fully padded
    "clamped": dict(seed=13, lengths=(17, 14), qk_offset=3000.0),   # logits of heads 0-3 past +50000, 4-5 past -50000
}
WEIGHTS = ("v_proj", "l_proj", "values_v_proj", "values_l_proj", "out_v_proj", "out_l_proj")


def build(name):
    """(state_dict, v, l, mask, grad_v_out, grad_l_out) as CPU fp32 tensors."""
    c = CASES[name]
    rng = np.random.default_rng(c["seed"])
    f = lambda *shape, s=1.0: torch.from_numpy((rng.standard_normal(shape) * s).astype(np.float32))
    sd = {}
    for w, (o, i) in zip(WEIGHTS, ((EMBED, V_DIM), (EMBED, L_DIM), (EMBED, V_DIM), (EMBED, L_DIM), (V_DIM, EMBED),
                                   (L_DIM, EMBED))):
        sd[f"attn.{w}.weight"] = f(o, i, s=(2.0 / (o + i)) ** 0.5)
        sd[f"attn.{w}.bias"] = f(o, s=0.02)
    # A large first channel per head in q and +-k shifts whole heads past a clamp: every logit of the head is clamped to
    # the same value, so the result does not hinge on the last bits of logits near 50000.
    off = c.get("qk_offset", 0.0)
    head0 = torch.arange(HEADS) * (EMBED // HEADS)
    sd["attn.v_proj.bias"][head0[:6]] += off
    sd["attn.l_proj.bias"][head0[:4]] += off
    sd["attn.l_proj.bias"][head0[4:6]] -= off
    for side, d in (("v", V_DIM), ("l", L_DIM)):
        sd[f"layer_norm_{side}.weight"] = 1.0 + f(d, s=0.1)
        sd[f"layer_norm_{side}.bias"] = f(d, s=0.1)
        sd[f"gamma_{side}"] = 0.5 + f(d, s=0.1)
    v, l = f(B, S, V_DIM), f(B, T, L_DIM)
    mask = torch.zeros(B, T, dtype=torch.int64)
    for b, n in enumerate(c["lengths"]):
        mask[b, :n] = 1
    return sd, v, l, mask, f(B, S, V_DIM), f(B, T, L_DIM)


def sketch_matrix(n_in):
    return torch.from_numpy(np.random.default_rng(1000 + n_in).standard_normal((n_in, 4)).astype(np.float32))


def record(out_v, out_l, grad_v, grad_l, param_grads):
    """What the fixture stores, as float32 numpy arrays (sketches formed in float64), from the block's results (any device)."""
    c = lambda t: t.detach().double().cpu()
    rec = {"out_v": c(out_v)[:, ::ROW_STRIDE], "out_l": c(out_l), "grad_v": c(grad_v)[:, ::ROW_STRIDE],
           "grad_l": c(grad_l)}
    for k, g in param_grads.items():
        g = c(g)
        rec["grad." + k] = g @ sketch_matrix(g.shape[1]).double() if g.dim() == 2 else g
    return {k: v.float().numpy() for k, v in rec.items()}


def run(block, name, device):
    """Forward + backward of `block` (eval mode) on the case; returns ``record(...)``."""
    sd, v, l, mask, gv, gl = build(name)
    block.load_state_dict(sd)
    block.to(device).eval()
    v, l = v.to(device).requires_grad_(True), l.to(device).requires_grad_(True)
    out_v, out_l = block(v, l, mask.to(device))
    ((out_v * gv.to(device)).sum() + (out_l * gl.to(device)).sum()).backward()
    return record(out_v, out_l, v.grad, l.grad, {k: p.grad for k, p in block.named_parameters()})
