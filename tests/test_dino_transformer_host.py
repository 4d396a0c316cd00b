"""CPU tests of the encoder's input preparation and DINO's whole transformer (uninext_b200/modules/dino_transformer.py,
include/msda_flatten.h): the header, the ctypes table and the library's exports agree; every entry point's argument
checks; the kernels compile without spills; a library without the entry points fails loudly; the CPU path equals the
reference's stored results; the state_dict keys are the reference's."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests import dino_case as dc
from tests import refgolden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "msda_flatten.h")
BADARG = -1
BASE = 0x7F0000000000                           # fake, 1 MiB-spaced device addresses
BIG_WS = 1 << 40


def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): len([a for a in m.group(2).split(",") if a.strip()])
            for m in re.finditer(r"\bint\s+(msda_\w+)\s*\(([^;{]*)\)\s*;", text)}


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    build.build()
    return _cabi.flatten()


def test_header_ctypes_table_and_exports_agree(lib):
    from uninext_b200 import _cabi
    decl = _declared()
    assert set(decl) == set(_cabi.FLATTEN_SIGNATURES) and len(decl) == 3
    assert not set(decl) & (set(_cabi.SIGNATURES) | set(_cabi.TWOSTAGE_SIGNATURES))
    for name, nargs in decl.items():
        assert len(_cabi.FLATTEN_SIGNATURES[name][1]) == nargs, name
        assert getattr(lib, name).argtypes == _cabi.FLATTEN_SIGNATURES[name][1], name
    assert lib.msda_abi_version() == 11


def test_library_without_the_entry_points_records_them_as_missing(tmp_path):
    """A library that exports msda_b200.h but not msda_flatten.h loads for the rest of the package, load() records its
    entry points as missing, and asking for them raises MSDALibraryError."""
    from uninext_b200 import _cabi
    src = tmp_path / "stub.c"
    body = ["int msda_abi_version(void) { return %d; }" % _cabi.ABI_VERSION]
    body += [f"int {n}(void) {{ return 0; }}" for n in _cabi.SIGNATURES if n != "msda_abi_version"]
    src.write_text("\n".join(body) + "\n")
    so = tmp_path / "libstub.so"
    try:
        subprocess.run(["gcc", "-shared", "-fPIC", "-o", str(so), str(src)], check=True, capture_output=True)
    except (OSError, subprocess.CalledProcessError) as exc:
        pytest.skip(f"no C compiler: {exc}")
    stub = _cabi.load(str(so))
    assert stub.missing == set(_cabi.TWOSTAGE_SIGNATURES) | set(_cabi.FLATTEN_SIGNATURES)
    with pytest.raises(_cabi.MSDALibraryError, match="msda_flatten_"):
        _cabi.flatten(str(so))
    for name in _cabi.FLATTEN_SIGNATURES:
        with pytest.raises(_cabi.MSDALibraryError, match=name):
            _cabi.entry(name, str(so))


# ---- argument checks (fake addresses: skipped where a GPU would run the kernels on them) -----------------------------
cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="calls with fake device addresses")
SHAPES = [(13, 21), (7, 11), (4, 6)]


def _p(i):
    return BASE + (i << 20)


def _arr(ctype, values):
    return (ctype * len(values))(*values)


def _fwd_args(shapes=SHAPES, N=2, C=256, null=None):
    """Pointers 0 .. 3L + 3 in order: src[l], pos[l], mask[l], level_embed, src_flat, pos_flat, mask_flat."""
    L = len(shapes)
    p = [None if i == null else _p(i) for i in range(3 * L + 4)]
    return [_arr(ctypes.c_void_p, p[:L]), _arr(ctypes.c_void_p, p[L:2 * L]), _arr(ctypes.c_void_p, p[2 * L:3 * L]),
            _arr(ctypes.c_int, [h for h, _ in shapes]), _arr(ctypes.c_int, [w for _, w in shapes]), L, N, C,
            *p[3 * L:], None]


def _bwd_args(shapes=SHAPES, N=2, C=256, null=None):
    """Pointers 0 .. 2L + 3 in order: grad_src_flat, grad_pos_flat, grad_src[l], grad_pos[l], grad_level_embed, workspace."""
    L = len(shapes)
    p = [None if i == null else _p(i) for i in range(2 * L + 4)]
    return [p[0], p[1], _arr(ctypes.c_int, [h for h, _ in shapes]), _arr(ctypes.c_int, [w for _, w in shapes]), L, N, C,
            _arr(ctypes.c_void_p, p[2:2 + L]), _arr(ctypes.c_void_p, p[2 + L:2 + 2 * L]), p[2 + 2 * L], p[3 + 2 * L],
            BIG_WS, None]


@cpu_only
def test_valid_calls_get_past_the_checks_and_each_null_is_badarg(lib):
    assert lib.msda_flatten_levels_forward_f32(*_fwd_args()) not in (BADARG, -2)
    assert lib.msda_flatten_levels_backward_f32(*_bwd_args()) not in (BADARG, -2)
    for i in range(3 * len(SHAPES) + 4):
        assert lib.msda_flatten_levels_forward_f32(*_fwd_args(null=i)) == BADARG, i
    for i in range(2 * len(SHAPES) + 4):
        got = lib.msda_flatten_levels_backward_f32(*_bwd_args(null=i))
        if i == 2 + 2 * len(SHAPES):
            assert got not in (BADARG, -2), "grad_level_embed may be NULL"
        else:
            assert got == BADARG, i
    for k in (0, 1):                                                    # a NULL array
        args = _fwd_args()
        args[k] = None
        assert lib.msda_flatten_levels_forward_f32(*args) == BADARG, k


@cpu_only
def test_optional_backward_outputs(lib):
    """grad_src, grad_pos and grad_level_embed may each be NULL; their inputs are then not required."""
    args = _bwd_args()
    args[7] = None                                                      # no grad_src: grad_src_flat unread
    args[0] = None
    assert lib.msda_flatten_levels_backward_f32(*args) not in (BADARG, -2)
    args = _bwd_args()
    args[8], args[9] = None, None                                       # grad_src only: grad_pos_flat, workspace unread
    args[1], args[10] = None, None
    assert lib.msda_flatten_levels_backward_f32(*args) not in (BADARG, -2)
    args = _bwd_args()
    args[8] = None                                                      # grad_level_embed alone still reads grad_pos_flat
    args[1] = None
    assert lib.msda_flatten_levels_backward_f32(*args) == BADARG
    args = _bwd_args()
    args[0], args[1], args[7], args[8], args[9] = None, None, None, None, None
    assert lib.msda_flatten_levels_backward_f32(*args) == 0             # nothing wanted: no launch


@cpu_only
def test_limits(lib):
    bad = [dict(N=0), dict(N=65536), dict(C=0), dict(C=258), dict(C=1028), dict(C=-4), dict(shapes=[]),
           dict(shapes=[(2, 2)] * 9), dict(shapes=[(0, 5)]), dict(shapes=[(5, -1)])]
    for kw in bad:
        assert lib.msda_flatten_levels_forward_f32(*_fwd_args(**kw)) == BADARG, kw
        assert lib.msda_flatten_levels_backward_f32(*_bwd_args(**kw)) == BADARG, kw
    for kw in (dict(N=65535, C=4), dict(C=1024), dict(C=252), dict(shapes=[(1, 1)] * 8)):
        assert lib.msda_flatten_levels_forward_f32(*_fwd_args(**kw)) not in (BADARG, -2), kw
    for i in (3 * len(SHAPES) + k for k in range(3)):                   # level_embed, src_flat, pos_flat misaligned
        args = _fwd_args()
        args[8 + i - 3 * len(SHAPES)] += 4
        assert lib.msda_flatten_levels_forward_f32(*args) == BADARG, i
    args = _fwd_args()
    args[11] += 1                                                       # mask_flat: bytes, any address
    assert lib.msda_flatten_levels_forward_f32(*args) not in (BADARG, -2)
    for k in (0, 1):                                                    # grad_src_flat, grad_pos_flat misaligned
        args = _bwd_args()
        args[k] += 4
        assert lib.msda_flatten_levels_backward_f32(*args) == BADARG, k
    args = _bwd_args()
    args[11] = 2 * 13 * 256 * 4 - 1                                     # too small a workspace
    assert lib.msda_flatten_levels_backward_f32(*args) == BADARG
    args[11] = 2 * 13 * 256 * 4
    assert lib.msda_flatten_levels_backward_f32(*args) not in (BADARG, -2)


def test_workspace_queries(lib):
    b = ctypes.c_int64(-7)
    h, w = _arr(ctypes.c_int, [s[0] for s in SHAPES]), _arr(ctypes.c_int, [s[1] for s in SHAPES])
    assert lib.msda_flatten_levels_workspace(h, w, 3, 2, 256, ctypes.byref(b)) == 0
    assert b.value == 2 * (9 + 3 + 1) * 256 * 4                         # 32-position tiles: 273, 77, 24 positions
    assert lib.msda_flatten_levels_workspace(h, w, 3, 2, 252, ctypes.byref(b)) == 0 and b.value == 2 * 13 * 252 * 4 // 256 * 256 + 256
    assert lib.msda_flatten_levels_workspace(h, w, 3, 2, 254, ctypes.byref(b)) == BADARG
    assert lib.msda_flatten_levels_workspace(h, w, 3, 2, 256, None) == BADARG
    assert lib.msda_flatten_levels_workspace(None, w, 3, 2, 256, ctypes.byref(b)) == BADARG


def test_kernels_are_built_without_spills():
    from uninext_b200 import build as b
    log = os.path.join(b.LIB_DIR, "build.log")
    if not os.path.exists(log):
        pytest.skip("library not built: no build.log")
    text = open(log).read()
    reports = re.findall(r"Function properties for (\S*flatten_levels_\w+?)E\S*\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    names = {re.search(r"flatten_levels_\w+", n).group(0) for n, *_ in reports}
    assert {"flatten_levels_fwd", "flatten_levels_bwd", "flatten_levels_reduce"} <= names, names
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"


# ---- the whole transformer against the reference's stored results ----------------------------------------------------
class _CpuOp:
    """The op's two entry points on CPU tensors, from the oracle's torch restatement of the reference's CPU function."""

    @staticmethod
    def ms_deform_attn_forward(value, shapes, lsi, loc, attn, im2col_step):
        from oracle.msda_oracle import core_pytorch_port
        with torch.no_grad():
            return core_pytorch_port(value, shapes, loc, attn)

    @staticmethod
    def ms_deform_attn_backward(value, shapes, lsi, loc, attn, grad_output, im2col_step):
        from oracle.msda_oracle import core_pytorch_port
        with torch.enable_grad():
            v, lo, at = (t.detach().clone().requires_grad_(True) for t in (value, loc, attn))
            return list(torch.autograd.grad(core_pytorch_port(v, shapes, lo, at), (v, lo, at), grad_output))


def build_model(name, device="cpu"):
    from uninext_b200.modules.deformable_transformer import MLP
    from uninext_b200.modules.dino_transformer import DeformableTransformerVLDINO
    from uninext_b200.modules.two_stage import Still_Classifier
    kw, flags = dc.config(name)
    model = dc.attach_heads(DeformableTransformerVLDINO(**kw, **flags), Still_Classifier, MLP).eval()
    g = refgolden.load(f"dino_transformer_{name}")
    seed = int(g["seed"][0])
    params = dc.parameters(model, seed)
    return model.to(device), params, seed, g


def run_case(name, device="cpu"):
    """-> (outputs, input leaves, parameters, golden) after forward + backward of the case."""
    model, params, seed, g = build_model(name, device)
    params = dict(model.named_parameters())
    x = dc.inputs(name, seed)
    out, leaves = dc.run(model, name, x, device)
    dc.backward(out, dc.cotangents(out, seed))
    return out, leaves, params, g


def compare_with_golden(out, leaves, params, g, tol):
    for k, v in out.items():
        if k == "memory":
            assert refgolden.rel(v, g, "out.memory", None) <= tol
            continue
        want = torch.from_numpy(g["out." + k]).double()
        got = v.detach().double().cpu()
        assert got.shape == want.shape, k
        assert torch.equal(torch.isinf(got), torch.isinf(want)), k
        fin = torch.isfinite(want)
        err = (got[fin] - want[fin]).abs().max().item() / max(want[fin].abs().max().item(), 1e-30)
        assert err <= tol, (k, err)
    for k in ("srcs", "pos_embeds"):
        for lvl, t in enumerate(leaves[k]):
            assert refgolden.rel(t.grad, g, f"grad.{k}.{lvl}", None) <= tol, (k, lvl)
    for k in ("hidden", "dn_label", "dn_bbox"):
        if k in leaves:
            assert refgolden.rel(leaves[k].grad, g, f"grad.{k}", None) <= tol, k
    names = g["param_names"].tolist()
    assert sorted(k for k, p in params.items() if p.grad is not None) == sorted(names)
    for k in names:
        assert refgolden.rel(params[k].grad, g, "grad." + k, None) <= tol, k


@pytest.mark.parametrize("name", list(dc.CASES))
def test_cpu_path_equals_reference(name, monkeypatch):
    from uninext_b200.functions import ms_deform_attn_func
    monkeypatch.setattr(ms_deform_attn_func, "MSDA", _CpuOp)
    g = refgolden.load(f"dino_transformer_{name}")
    x = dc.inputs(name, int(g["seed"][0]))
    for k in ("srcs", "pos_embeds"):
        for lvl, t in enumerate(x[k]):
            assert np.array_equal(refgolden.sample(t, g, f"in.{k}.{lvl}", None), g[f"in.{k}.{lvl}"]), (k, lvl)
    out, leaves, params, g = run_case(name)
    compare_with_golden(out, leaves, params, g, 1e-4)


@pytest.mark.parametrize("name", list(dc.CASES))
def test_state_dict_keys_are_the_reference_ones(name):
    model, _, _, g = build_model(name)
    assert list(model.state_dict().keys()) == g["state_dict_keys"].tolist()
    model.load_state_dict(model.state_dict(), strict=True)


def test_unsupported_configurations_raise():
    from uninext_b200.modules.dino_transformer import DeformableTransformerVLDINO
    kw, flags = dc.config("production")
    for over in (dict(two_stage=False), dict(use_checkpoint=True)):
        with pytest.raises(ValueError):
            DeformableTransformerVLDINO(**{**kw, **over}, **flags)
    with pytest.raises(ValueError, match="BERT"):
        DeformableTransformerVLDINO(**kw, **flags, use_additional_bert=True)


def test_cpu_flatten_levels_is_the_reference_chain():
    """The CPU path against the reference's statements (deformable_transformer_dino.py:181-201), written out here."""
    from uninext_b200.modules.dino_transformer import flatten_levels
    g = torch.Generator().manual_seed(0)
    shapes = [(13, 21), (7, 11), (4, 6)]
    srcs = [torch.randn(2, 12, h, w, generator=g) for h, w in shapes]
    pos = [torch.randn(2, 12, h, w, generator=g) for h, w in shapes]
    masks = [torch.zeros(2, h, w, dtype=torch.bool) for h, w in shapes]
    for m in masks:
        m[1, :, m.shape[2] * 2 // 3:] = True
    le = torch.randn(3, 12, generator=g)
    src_f, mask_f, pos_f, ss, lsi, vr = flatten_levels(srcs, masks, pos, le)
    assert torch.equal(src_f, torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1))
    assert torch.equal(pos_f, torch.cat([p.flatten(2).transpose(1, 2) + le[i].view(1, 1, -1) for i, p in enumerate(pos)], 1))
    assert torch.equal(mask_f, torch.cat([m.flatten(1) for m in masks], 1))
    assert ss.tolist() == [list(s) for s in shapes] and lsi.tolist() == [0, 273, 350]
    want = torch.stack([torch.stack(((~m[:, 0, :]).sum(1).float() / m.shape[2], (~m[:, :, 0]).sum(1).float() / m.shape[1]),
                                    -1) for m in masks], 1)
    assert torch.equal(vr, want)
