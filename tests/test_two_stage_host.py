"""CPU tests of the two-stage query selection (uninext_b200/modules/two_stage.py, include/msda_twostage.h):
the header, the ctypes table and the library's exports agree; every entry point's argument checks; the kernels compile
without spills; a library without the entry points fails loudly; the CPU path equals the reference's stored results."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests import refgolden
from tests import two_stage_case as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "msda_twostage.h")
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
    return _cabi.twostage()


def test_header_ctypes_table_and_exports_agree(lib):
    from uninext_b200 import _cabi
    decl = _declared()
    assert set(decl) == set(_cabi.TWOSTAGE_SIGNATURES) and len(decl) == 6
    assert not set(decl) & set(_cabi.SIGNATURES)
    for name, nargs in decl.items():
        assert len(_cabi.TWOSTAGE_SIGNATURES[name][1]) == nargs, name
        assert getattr(lib, name).argtypes == _cabi.TWOSTAGE_SIGNATURES[name][1], name
    assert lib.msda_abi_version() == 11


def test_library_without_the_entry_points_records_them_as_missing(tmp_path):
    """A library that exports msda_b200.h but not msda_twostage.h loads for the rest of the package, load() records its
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
    with pytest.raises(_cabi.MSDALibraryError, match="msda_twostage_"):
        _cabi.twostage(str(so))
    for name in _cabi.TWOSTAGE_SIGNATURES:
        with pytest.raises(_cabi.MSDALibraryError, match=name):
            _cabi.entry(name, str(so))


# ---- argument checks (fake addresses: skipped where a GPU would run the kernels on them) -----------------------------
def _p(i):
    return BASE + (i << 20)


def _calls():
    """name -> (pointer count, call(ptrs, **sizes))."""
    f32 = ctypes.c_float
    return {
        "msda_twostage_head_forward_f32": (11, lambda p, N=2, S=747, C=256: (
            p[0], p[1], p[2], p[3], p[4], p[5], p[6], N, S, C, f32(1e-5), 1, p[7], p[8], p[9], p[10], None)),
        "msda_twostage_head_backward_f32": (18, lambda p, N=2, S=747, C=256: (
            *p[:11], N, S, C, 1, *p[11:17], p[17], BIG_WS, None)),
        "msda_twostage_select_forward_f32": (7, lambda p, N=2, S=747, k=300: (
            p[0], p[1], p[2], N, S, k, p[3], p[4], p[5], p[6], BIG_WS, None)),
        "msda_twostage_select_backward_f32": (4, lambda p, N=2, S=747, k=300: (p[0], p[1], p[2], N, S, k, p[3], None)),
    }


NO_WS = {"msda_twostage_select_forward_f32": 6}     # the sort workspace is only read when k > 2048


def _call(lib, name, null=None, **sizes):
    n, make = _calls()[name]
    ptrs = [None if i == null else _p(i) for i in range(n)]
    return getattr(lib, name)(*make(ptrs, **sizes))


cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="calls with fake device addresses")


@cpu_only
@pytest.mark.parametrize("name", sorted(_calls()))
def test_valid_call_gets_past_the_checks_and_each_null_is_badarg(lib, name):
    assert _call(lib, name) not in (BADARG, -2)
    for i in range(_calls()[name][0]):
        got = _call(lib, name, null=i)
        if NO_WS.get(name) == i:
            assert got != BADARG, f"{name}: workspace may be NULL at k <= 2048"
        else:
            assert got == BADARG, f"{name}: pointer {i} NULL"


@cpu_only
def test_limits(lib):
    for name in ("msda_twostage_select_forward_f32", "msda_twostage_select_backward_f32"):
        for k in (0, -1, 748):                                      # k <= 0, k > S
            assert _call(lib, name, k=k) == BADARG, (name, k)
        assert _call(lib, name, k=747) not in (BADARG, -2)          # k = S
        for over in ({"N": 0}, {"N": 65536}, {"S": 0}):
            assert _call(lib, name, **over) == BADARG, (name, over)
    ws = _calls()["msda_twostage_select_forward_f32"][1]
    p = [_p(i) for i in range(7)]
    args = list(ws(p, S=5000, k=4000))
    assert lib.msda_twostage_select_forward_f32(*args) not in (BADARG, -2)
    args[-2] = 2 * 4096 * 8 - 1                                     # too small a sort workspace at k > 2048
    assert lib.msda_twostage_select_forward_f32(*args) == BADARG
    args[-2], args[-3] = BIG_WS, None                               # ... or none
    assert lib.msda_twostage_select_forward_f32(*args) == BADARG
    for name in ("msda_twostage_head_forward_f32", "msda_twostage_head_backward_f32"):
        for c in (128, 255, 257, 512):                              # width != 256
            assert _call(lib, name, C=c) == BADARG, (name, c)
        for over in ({"N": 0}, {"S": 0}, {"S": -3}):
            assert _call(lib, name, **over) == BADARG, (name, over)
    a = [_p(i) for i in range(18)]
    a[4] += 4                                                       # a misaligned float4 operand (beta)
    assert lib.msda_twostage_head_backward_f32(*_calls()["msda_twostage_head_backward_f32"][1](a)) == BADARG
    args = list(_calls()["msda_twostage_head_backward_f32"][1]([_p(i) for i in range(18)]))
    args[-2] = 100                                                  # too small a workspace
    assert lib.msda_twostage_head_backward_f32(*args) == BADARG


def test_workspace_queries(lib):
    b = ctypes.c_int64(-7)
    assert lib.msda_twostage_head_workspace(2, 747, 256, ctypes.byref(b)) == 0
    assert b.value == (2 * 12 * (4 * 256 + 4) * 4 + 255) // 256 * 256    # 12 tiles of 64 rows per image, 256-aligned
    assert lib.msda_twostage_head_workspace(2, 747, 128, ctypes.byref(b)) == BADARG
    assert lib.msda_twostage_head_workspace(2, 747, 256, None) == BADARG
    assert lib.msda_twostage_select_workspace(2, 747, 300, ctypes.byref(b)) == 0 and b.value == 0
    assert lib.msda_twostage_select_workspace(2, 22323, 22323, ctypes.byref(b)) == 0 and b.value == 2 * 32768 * 8
    assert lib.msda_twostage_select_workspace(2, 747, 748, ctypes.byref(b)) == BADARG
    assert lib.msda_twostage_select_workspace(2, 747, 0, ctypes.byref(b)) == BADARG


def test_kernels_are_built_without_spills():
    from uninext_b200 import build as b
    log = os.path.join(b.LIB_DIR, "build.log")
    if not os.path.exists(log):
        pytest.skip("library not built: no build.log")
    text = open(log).read()
    reports = re.findall(r"Function properties for (\S*twostage_\w+?)E\S*\s*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    names = {re.search(r"twostage_\w+", n).group(0) for n, *_ in reports}
    assert {"twostage_head_fwd", "twostage_head_bwd", "twostage_head_reduce", "twostage_select_fwd",
            "twostage_select_bwd"} <= names, names
    for name, stack, st, ld in reports:
        assert int(st) == 0 and int(ld) == 0, f"{name}: {st} bytes spill stores, {ld} bytes spill loads"


# ---- the CPU path against the reference's stored results -------------------------------------------------------------
def make_modules(name, device="cpu"):
    from uninext_b200.modules.deformable_transformer import MLP
    from uninext_b200.modules.two_stage import Still_Classifier, VL_Align
    head, clamp, log_scale = tc.CASES[name]
    modules = {"enc_output": torch.nn.Linear(tc.C, tc.C), "enc_output_norm": torch.nn.LayerNorm(tc.C),
               "class_embed": Still_Classifier(tc.C) if head == "still" else VL_Align(tc.C, tc.LANG, log_scale,
                                                                                     clamp_dot_product=clamp),
               "bbox_embed": MLP(tc.C, tc.C, 4, 3)}
    for m in modules.values():
        m.to(device)
    return modules, tc.load_modules(name, modules)


def run_case(name, device="cpu"):
    """-> (outputs, memory.grad, {param name: grad}) of two_stage_select on the case."""
    from uninext_b200.modules.two_stage import two_stage_select
    modules, params = make_modules(name, device)
    x = tc.inputs(name)
    memory = x["memory"].to(device).requires_grad_(True)
    out = two_stage_select(memory, x["mask"].to(device), tc.SHAPES, modules["enc_output"], modules["enc_output_norm"],
                           modules["class_embed"], modules["bbox_embed"], tc.K, x["lang_feat_pool"].to(device))
    tc.backward(out, x)
    return out, memory.grad, {k: p.grad for k, p in params.items()}


def check_inputs_are_the_recorded_ones(name, g):
    x = tc.inputs(name)
    for k, v in list(x.items()) + [("state." + k, v) for k, v in tc.state(name).items()]:
        key = k if k.startswith("state.") else "in." + k
        assert np.array_equal(refgolden.sample(v, g, key, None), g[key]), key


def compare_with_golden(name, out, g_mem, grads, tol):
    """Outputs and gradients within tol of the reference's scale; indices equal wherever the reference's consecutive
    ranks are more than 1e-5 of the logit scale apart.  -> the number of ranks within 1e-5 of the next that is not an
    exact tie, counted once per neighbouring pair (exact ties -- the dropped rows -- are in torch.topk's unspecified order in
    the reference)."""
    g = refgolden.load(f"two_stage_{name}")
    cls, coord, ref, idx = (t.detach().cpu() for t in out)
    want_cls = torch.from_numpy(g["out.enc_outputs_class"])
    scale = want_cls.abs().max().item()
    assert (cls - want_cls).abs().max().item() <= tol * scale
    want_coord = torch.from_numpy(g["out.enc_outputs_coord_unact"])
    assert torch.equal(torch.isinf(coord), torch.isinf(want_coord))
    fin = torch.isfinite(want_coord)
    assert (coord[fin] - want_coord[fin]).abs().max().item() <= tol * want_coord[fin].abs().max().item()
    assert refgolden.rel(g_mem, g, "grad.memory", None) <= tol
    assert sorted(grads) == sorted(g["param_names"].tolist())
    for k, v in grads.items():
        assert refgolden.rel(v, g, "grad." + k, None) <= tol, k
    # indices: the reference's order is torch.topk's; compare where its neighbouring logits are clearly apart
    want_idx = torch.from_numpy(g["out.topk_proposals"])
    close = 0
    for b in range(want_idx.shape[0]):
        lg = want_cls[b, want_idx[b], 0]
        gap = torch.cat((lg[:-1] - lg[1:], torch.tensor([float("inf")])))    # to the next rank
        prev = torch.cat((torch.tensor([float("inf")]), gap[:-1]))
        clear = (gap > 1e-5 * scale) & (prev > 1e-5 * scale)
        assert torch.equal(idx[b][clear], want_idx[b][clear]), b
        want_ref = torch.from_numpy(g["out.reference_points"])[b]
        assert (ref[b][clear] - want_ref[clear]).abs().max().item() <= tol
        # elsewhere: the reference points of the rows this path picked, from the reference's coord_unact
        assert (ref[b] - want_coord[b, idx[b]].sigmoid()).abs().max().item() <= tol
        # ranks among near-ties hold the same set of rows' logits
        assert torch.allclose(want_cls[b, idx[b], 0], lg, rtol=0, atol=1e-5 * scale + tol * scale)
        close += int(((gap > 0) & (gap <= 1e-5 * scale)).sum())
    return close


@pytest.mark.parametrize("name", list(tc.CASES))
def test_cpu_path_equals_reference(name):
    check_inputs_are_the_recorded_ones(name, refgolden.load(f"two_stage_{name}"))
    out, g_mem, grads = run_case(name)
    assert out[3].dtype == torch.int64 and out[3].shape == (tc.N, tc.K) and out[2].shape == (tc.N, tc.K, 4)
    compare_with_golden(name, out, g_mem, grads, 1e-5)


def test_cpu_path_rejects_k_above_s():
    from uninext_b200.modules.two_stage import two_stage_select
    modules, _ = make_modules("still")
    x = tc.inputs("still")
    with pytest.raises(RuntimeError, match="out of range"):
        two_stage_select(x["memory"], x["mask"], tc.SHAPES, modules["enc_output"], modules["enc_output_norm"],
                         modules["class_embed"], modules["bbox_embed"], tc.S + 1)
