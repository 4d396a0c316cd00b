"""CPU test: ``op_dtype`` of the early-fusion modules (BiMultiHeadAttention, BiAttentionBlock, VLFuse).  On CPU tensors
``op_dtype=torch.bfloat16`` runs the attention core as the torch composition in bf16."""
import pytest
import torch

from uninext_b200.modules import vl_fusion as vf


def _inputs():
    g = torch.Generator().manual_seed(0)
    v, l = torch.randn(2, 300, 256, generator=g), torch.randn(2, 17, 768, generator=g)
    mask = torch.ones(2, 17, dtype=torch.int64)
    mask[1, 9:] = 0
    return v, l, mask


def test_bf16_attention_stays_within_bf16_tolerance_of_fp32():
    torch.manual_seed(0)
    a = vf.BiMultiHeadAttention(256, 768, 2048, 8).eval()
    b = vf.BiMultiHeadAttention(256, 768, 2048, 8, op_dtype=torch.bfloat16).eval()
    b.load_state_dict(a.state_dict())
    v, l, mask = _inputs()
    want, got = a(v, l, mask), b(v, l, mask)
    for w, g in zip(want, got):
        assert g.dtype == torch.float32
        assert ((g - w).abs().max() / w.abs().max()).item() < 1e-2


def test_bf16_block_stays_within_bf16_tolerance_of_fp32_with_gradients():
    """Outputs, input gradients and parameter gradients within 1e-2 of scale; the l_proj bias gradient, a sum of dK over
    the text tokens whose vision-softmax part cancels exactly, within 3e-2 of its own (small) scale."""
    torch.manual_seed(0)
    a = vf.BiAttentionBlock(256, 768, 2048, 8, init_values=1.0).eval()
    b = vf.BiAttentionBlock(256, 768, 2048, 8, init_values=1.0, op_dtype=torch.bfloat16).eval()
    b.load_state_dict(a.state_dict())
    v, l, mask = _inputs()
    results = []
    for blk in (a, b):
        vv, ll = v.clone().requires_grad_(True), l.clone().requires_grad_(True)
        out_v, out_l = blk(vv, ll, mask)
        (out_v.square().mean() + out_l.square().mean()).backward()
        results.append({"out_v": out_v, "out_l": out_l, "grad_v": vv.grad, "grad_l": ll.grad,
                        **{"grad." + n: p.grad for n, p in blk.named_parameters()}})
    for key, w in results[0].items():
        g = results[1][key]
        assert g.dtype == torch.float32
        err = ((g - w).abs().max() / w.abs().max()).item()
        assert err < (3e-2 if key == "grad.attn.l_proj.bias" else 1e-2), (key, err)


@pytest.mark.parametrize("cls,args", [(vf.BiMultiHeadAttention, (256, 768, 2048, 8)),
                                      (vf.BiAttentionBlock, (256, 768, 2048, 8)), (vf.VLFuse, ())])
def test_state_dict_keys_do_not_depend_on_op_dtype(cls, args):
    a, b = cls(*args), cls(*args, op_dtype=torch.bfloat16)
    assert list(a.state_dict()) == list(b.state_dict())
    assert all(p.dtype == torch.float32 for p in b.parameters())


@pytest.mark.parametrize("op_dtype", [torch.float16, torch.float32, "bf16"])
@pytest.mark.parametrize("cls,args", [(vf.BiMultiHeadAttention, (256, 768, 2048, 8)),
                                      (vf.BiAttentionBlock, (256, 768, 2048, 8)), (vf.VLFuse, ())])
def test_other_op_dtypes_are_refused(cls, args, op_dtype):
    with pytest.raises(ValueError, match="op_dtype"):
        cls(*args, op_dtype=op_dtype)


def test_vlfuse_passes_op_dtype_down():
    m = vf.VLFuse(op_dtype=torch.bfloat16)
    assert m.b_attn.op_dtype == m.b_attn.attn.op_dtype == torch.bfloat16
    assert vf.VLFuse().b_attn.attn.op_dtype is None
