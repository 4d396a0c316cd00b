"""How the package calls the C ABI (uninext_b200/_cabi.py: ``call``, ``workspace``, ``entry``).

CPU, with a fake library and fake ``torch.cuda.device`` / ``torch.cuda.current_stream``: tensors arrive as their data
pointers and None as NULL, the stream of the given device is the last argument and that device's context is entered
around the call, a non-zero code raises RuntimeError naming the entry point, a size query returns what the library
wrote, and a missing optional entry point raises MSDALibraryError.  No module but _cabi.py writes the plumbing itself.

GPU, with two devices: every kind of call on cuda:1 tensors, made while cuda:0 is current, equals the same call on
cuda:0 (skipped on a machine with one GPU)."""
import ctypes
import os
import types

import pytest
import torch

from uninext_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREAMS = {"cuda:0": 0x5000, "cuda:1": 0x5100}
E_BADARG = -1


class _FakeLib:
    """Entry points that record their arguments and which devices were entered when they ran."""

    def __init__(self, entered):
        self.entered, self.calls, self.code = entered, [], 0
        self.missing = {"msda_twostage_select_forward_f32", "msda_twostage_select_workspace"}

    def msda_strerror(self, code):
        return b"invalid argument"

    def msda_colsum_f32(self, *args):
        self.calls.append((args, list(self.entered)))
        return self.code

    def msda_vlfuse_workspace(self, *args):
        self.calls.append((args, list(self.entered)))
        args[-1]._obj.value = 12345
        return self.code


@pytest.fixture
def fake(monkeypatch):
    entered = []

    class Device:
        def __init__(self, device):
            self.device = str(device)

        def __enter__(self):
            entered.append(self.device)

        def __exit__(self, *exc):
            entered.pop()

    monkeypatch.setattr(torch.cuda, "device", Device)
    monkeypatch.setattr(torch.cuda, "current_stream",
                        lambda device=None: types.SimpleNamespace(cuda_stream=STREAMS[str(device)]))
    lib = _FakeLib(entered)
    monkeypatch.setattr(_cabi, "_lib", lib)
    monkeypatch.setattr(_cabi, "_entries", {})
    return lib


def test_tensors_go_as_pointers_none_as_null_and_the_rest_unchanged(fake):
    x, y = torch.ones(4, 8), torch.zeros(3)
    scale = ctypes.c_float(0.5)
    _cabi.call("msda_colsum_f32", x, 4, None, 2.5, scale, y, x.data_ptr() + 16, device=torch.device("cuda:1"))
    (args, _), = fake.calls
    assert args[:-1] == (x.data_ptr(), 4, None, 2.5, scale, y.data_ptr(), x.data_ptr() + 16)
    assert args[4] is scale


@pytest.mark.parametrize("device", ["cuda:0", "cuda:1"])
def test_runs_in_the_device_context_on_its_stream(fake, device):
    _cabi.call("msda_colsum_f32", torch.ones(2), device=torch.device(device))
    (args, entered), = fake.calls
    assert args[-1] == STREAMS[device]
    assert entered == [device]
    assert fake.entered == []


def test_nonzero_code_raises_naming_the_entry_point(fake):
    fake.code = E_BADARG
    with pytest.raises(RuntimeError, match="msda_colsum_f32 failed with code -1: invalid argument"):
        _cabi.call("msda_colsum_f32", torch.ones(2), device=torch.device("cuda:0"))
    assert fake.entered == []


def test_workspace_returns_what_the_library_wrote(fake):
    assert _cabi.workspace("msda_vlfuse_workspace", 1, 2, 3, 4, 128) == 12345
    (args, entered), = fake.calls
    assert args[:-1] == (1, 2, 3, 4, 128) and entered == []
    fake.code = E_BADARG
    with pytest.raises(RuntimeError, match="msda_vlfuse_workspace failed with code -1: invalid argument"):
        _cabi.workspace("msda_vlfuse_workspace", 1, 2, 3, 4, 128)


def test_missing_optional_entry_point_raises(fake):
    with pytest.raises(_cabi.MSDALibraryError, match="msda_twostage_select_forward_f32"):
        _cabi.call("msda_twostage_select_forward_f32", torch.ones(2), device=torch.device("cuda:0"))
    with pytest.raises(_cabi.MSDALibraryError, match="msda_twostage_select_workspace"):
        _cabi.workspace("msda_twostage_select_workspace", 1, 2, 3)
    assert fake.calls == []


def test_no_module_but_cabi_writes_the_call_plumbing():
    offenders = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "uninext_b200")):
        for f in files:
            path = os.path.join(dirpath, f)
            if not f.endswith(".py") or path == os.path.join(ROOT, "uninext_b200", "_cabi.py"):
                continue
            text = open(path).read()
            offenders += [f"{os.path.relpath(path, ROOT)}: {s}" for s in ("cuda_stream", "_cabi.check(", "ctypes.byref")
                          if s in text]
    assert not offenders, offenders


# ---- GPU: a call on the second device, made while the first is current, equals the call on the first -----------------
def _cpu(*ts):
    return [t.detach().cpu() for t in ts]


def _vl_attention(dev):
    from uninext_b200.modules.vl_fusion import dropout_masks, vl_attention
    g = torch.Generator().manual_seed(0)
    q, k, vv, vl = (torch.randn(1, n, 2, 128, generator=g).to(dev).requires_grad_(True) for n in (64, 16, 64, 16))
    seed = torch.tensor([1234], dtype=torch.int64, device=dev)
    o_v, o_l = vl_attention(q, k, vv, vl, dropout_p=0.1, training=True, seed=seed)
    (o_v.square().sum() + o_l.sum()).backward()
    return _cpu(o_v, o_l, q.grad, k.grad, vv.grad, vl.grad, *dropout_masks(seed, 1, 2, 64, 16, 0.1))


def _two_stage_select(dev):
    from uninext_b200.modules.deformable_transformer import MLP
    from uninext_b200.modules.two_stage import Still_Classifier, two_stage_select
    torch.manual_seed(0)
    shapes = ((8, 8), (4, 4))
    mods = [m.to(dev) for m in (torch.nn.Linear(256, 256), torch.nn.LayerNorm(256), Still_Classifier(256),
                                MLP(256, 256, 4, 1))]
    memory = torch.randn(2, 80, 256).to(dev).requires_grad_(True)
    mask = torch.zeros(2, 80, dtype=torch.bool, device=dev)
    cls, coord, ref, idx = two_stage_select(memory, mask, shapes, *mods, 10)
    (cls.sum() + coord.square().sum() + ref.sum()).backward()
    return _cpu(cls, coord, ref, idx, memory.grad, mods[0].weight.grad)


def _flatten_levels(dev):
    from uninext_b200.modules.dino_transformer import flatten_levels
    g = torch.Generator().manual_seed(0)
    shapes = ((9, 7), (4, 5))
    srcs = [torch.randn(2, 8, h, w, generator=g).to(dev).requires_grad_(True) for h, w in shapes]
    pos = [torch.randn(2, 8, h, w, generator=g).to(dev).requires_grad_(True) for h, w in shapes]
    masks = [(torch.rand(2, h, w, generator=g) > 0.7).to(dev) for h, w in shapes]
    level_embed = torch.randn(2, 8, generator=g).to(dev).requires_grad_(True)
    src_flat, mask_flat, pos_flat, _, _, ratios = flatten_levels(srcs, masks, pos, level_embed)
    (src_flat.square().sum() + pos_flat.sum()).backward()
    return _cpu(src_flat, mask_flat, pos_flat, ratios, *[s.grad for s in srcs], *[p.grad for p in pos], level_embed.grad)


def _condinst(dev):
    from uninext_b200.modules.dynamic_mask_head import dynamic_mask_with_coords
    g = torch.Generator().manual_seed(0)
    feats = torch.randn(2, 8, 12, 10, generator=g).to(dev).requires_grad_(True)
    refs = (torch.rand(1, 5, 2, generator=g) * 80).to(dev).requires_grad_(True)
    params = (0.3 * torch.randn(1, 5, 169, generator=g)).to(dev).requires_grad_(True)
    logits = dynamic_mask_with_coords(feats, refs, params, [3, 2], 8)
    logits.square().sum().backward()
    return _cpu(logits, feats.grad, refs.grad, params.grad)


def _ms_deform_attn(dev):
    from uninext_b200.dropin.MultiScaleDeformableAttention import ms_deform_attn_backward, ms_deform_attn_forward
    from uninext_b200.workloads import CONFIGS, make_inputs
    inp = {k: v.to(dev) for k, v in make_inputs(CONFIGS["cfg1"], "dec", "cpu", seed=0).items()}
    args = (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
            inp["attention_weights"])
    out = ms_deform_attn_forward(*args, 64)
    return _cpu(out, *ms_deform_attn_backward(*args, inp["grad_output"], 64, deterministic=True))


CALLS = {"vl_attention": _vl_attention, "two_stage_select": _two_stage_select, "flatten_levels": _flatten_levels,
         "condinst": _condinst, "ms_deform_attn": _ms_deform_attn}


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
@pytest.mark.parametrize("name", list(CALLS))
def test_second_device_while_first_is_current_equals_first(name):
    with torch.cuda.device(0):
        want = CALLS[name]("cuda:0")
        got = CALLS[name]("cuda:1")
        assert torch.cuda.current_device() == 0
    for w, g in zip(want, got, strict=True):
        scale = w.abs().max().item() if w.is_floating_point() and w.numel() else 1.0
        torch.testing.assert_close(g, w, rtol=1e-5, atol=1e-5 * scale, equal_nan=True)
