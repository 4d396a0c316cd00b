"""GPU tests of the deterministic backward (msda_backward_det_*, include/msda_b200.h; DESIGN.md section 3.10).

grad_value must equal the C oracle's bit for bit: the oracle adds the same contributions, rounded the same way, in the
same order.  grad_sampling_loc / grad_attn_weight must equal the default backward's bit for bit.  No tolerance is used.
"""
import ctypes
import os
import subprocess
import sys
import textwrap
import warnings

import numpy as np
import pytest
import torch

from oracle import msda_oracle
from tests.conftest import ROOT, golden_names, load_golden

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA
    from uninext_b200.functions import MSDeformAttnFunction, MSDeformAttnFunctionBF16
    from uninext_b200.workloads import CONFIGS, OpConfig, level_tensors, make_inputs

DEV = "cuda"


def _np(t):
    return t.detach().cpu().numpy()


def _args(inp):
    return (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
            inp["attention_weights"])


def _oracle_gv(inp, dtype=np.float32):
    """grad_value of the C oracle in `dtype` (bf16 inputs are widened exactly)."""
    a = [_np(t.float() if t.dtype == torch.bfloat16 else t) for t in _args(inp)]
    a[0], a[3], a[4] = a[0].astype(dtype), a[3].astype(dtype), a[4].astype(dtype)
    go = _np(inp["grad_output"].float() if inp["grad_output"].dtype == torch.bfloat16 else inp["grad_output"])
    gv, _, _ = msda_oracle.backward(go.astype(dtype), *a)
    return gv


def _golden_inputs(name, dtype):
    c = load_golden(name)
    aux = torch.float64 if dtype == torch.float64 else torch.float32
    t = lambda k, dt: torch.from_numpy(c[k]).to(DEV, dt).contiguous()
    return dict(value=t("value", dtype), spatial_shapes=t("spatial_shapes", torch.int64),
                level_start_index=t("level_start_index", torch.int64), sampling_locations=t("sampling_locations", aux),
                attention_weights=t("attention_weights", aux), grad_output=t("grad_output", dtype))


def _det(inp, **kw):
    return MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64, deterministic=True, **kw)


def _default(inp, **kw):
    return MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64, deterministic=False, **kw)


def _small(D, dtype=torch.float32, seed=0, kind="enc"):
    cfg = OpConfig(f"d{D}", 64, 96, 2, 37, heads=2, head_dim=D)
    return make_inputs(cfg, kind, DEV, dtype=dtype, seed=seed, wild_fraction=0.05)


def _one_pixel_case(lq=300):
    """Every tap of the 1x1 level lands on its one pixel (corner 0, weight 1): the longest possible segments."""
    shapes = [(8, 8), (1, 1)]
    ss, lsi = level_tensors(shapes, DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    n, m, d, p = 1, 2, 32, 4
    s = 65
    loc = torch.rand(n, lq, m, 2, p, 2, generator=g, device=DEV)
    loc[:, :, :, 1] = 0.5
    attn = torch.softmax(torch.randn(n, lq, m, 2 * p, generator=g, device=DEV), -1).view(n, lq, m, 2, p)
    return dict(value=torch.randn(n, s, m, d, generator=g, device=DEV), spatial_shapes=ss, level_start_index=lsi,
                sampling_locations=loc.contiguous(), attention_weights=attn.contiguous(),
                grad_output=torch.randn(n, lq, m * d, generator=g, device=DEV))


# ---- 1. bit-identical to the oracle ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", golden_names())
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_golden_grad_value_equals_oracle(name, dtype):
    inp = _golden_inputs(name, dtype)
    gv, _, _ = _det(inp)
    want = _oracle_gv(inp, np.float64 if dtype == torch.float64 else np.float32)
    assert np.array_equal(_np(gv), want)


@pytest.mark.parametrize("kind", ["enc", "dec"])
def test_cfg1_grad_value_equals_oracle(kind):
    inp = make_inputs(CONFIGS["cfg1"], kind, DEV, seed=3, wild_fraction=0.02)
    gv, _, _ = _det(inp)
    assert np.array_equal(_np(gv), _oracle_gv(inp))


def test_cfg2_encoder_grad_value_equals_oracle():
    inp = make_inputs(CONFIGS["cfg2"], "enc", DEV, seed=10)
    gv, _, _ = _det(inp)
    assert np.array_equal(_np(gv), _oracle_gv(inp))


# ---- 2. bf16: the fp32 accumulator follows the contract, the bf16 result is its rounding -------------------------------
@pytest.mark.parametrize("D", [32, 64, 48])
def test_bf16_accumulator_equals_oracle(D):
    inp = _small(D, torch.bfloat16, seed=D)
    acc, gl32, ga32 = _det(inp, grad_value_dtype=torch.float32)
    assert acc.dtype == torch.float32
    assert np.array_equal(_np(acc), _oracle_gv(inp))
    gv, gl, ga = _det(inp)
    assert gv.dtype == torch.bfloat16 and torch.equal(gv, acc.to(torch.bfloat16))
    assert torch.equal(gl, gl32) and torch.equal(ga, ga32)


# ---- 3. grad_loc / grad_attn are the default route's, bit for bit ---------------------------------------------------
@pytest.mark.parametrize("case", ["cfg2_enc_region", "cfg2_dec_split", "d30_generic", "fp64", "bf16_cfg2_dec"])
def test_loc_attn_equal_default_path(case):
    if case == "cfg2_enc_region":
        inp = make_inputs(CONFIGS["cfg2"], "enc", DEV, seed=1)
    elif case == "cfg2_dec_split":
        inp = make_inputs(CONFIGS["cfg2"], "dec", DEV, seed=2)
    elif case == "d30_generic":
        inp = _small(30, seed=4)
        assert _cabi.load().msda_uses_fast_path(4, 30, 4, 4) == 0
    elif case == "fp64":
        inp = _small(32, torch.float64, seed=6)
    else:
        inp = make_inputs(CONFIGS["cfg2"], "dec", DEV, dtype=torch.bfloat16, seed=7)
    _, gl_d, ga_d = _det(inp)
    _, gl, ga = _default(inp)
    assert torch.equal(gl_d, gl) and torch.equal(ga_d, ga)


# ---- 4. chunking changes no bit ------------------------------------------------------------------------------------
def _call_det_f32(inp, chunk_queries):
    v = inp["value"]
    n, s, m, d = v.shape
    dims = (n, s, m, d, inp["spatial_shapes"].shape[0], inp["sampling_locations"].shape[1],
            inp["sampling_locations"].shape[4])
    nbytes = _cabi.workspace("msda_backward_det_workspace", 4, *dims, chunk_queries)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gv = torch.full_like(v, float("nan"))                 # the callee zero-fills
    gl = torch.empty_like(inp["sampling_locations"])
    ga = torch.empty_like(inp["attention_weights"])
    _cabi.call("msda_backward_det_f32", inp["grad_output"], *_args(inp), *dims, gv, gl, ga, ws, ws.numel(),
               device=v.device)
    return gv, gl, ga, dims


@pytest.mark.parametrize("case", ["cfg1_enc", "one_pixel"])
def test_small_chunks_equal_one_pass(case):
    inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=8) if case == "cfg1_enc" else _one_pixel_case()
    gv7, gl7, ga7, dims = _call_det_f32(inp, 7)
    gv, gl, ga, _ = _call_det_f32(inp, dims[5])
    assert torch.equal(gv7, gv) and torch.equal(gl7, gl) and torch.equal(ga7, ga)
    assert np.array_equal(_np(gv), _oracle_gv(inp))


def test_workspace_errors():
    lib = _cabi.load()
    inp = _small(32)
    v = inp["value"]
    n, s, m, d = v.shape
    dims = (n, s, m, d, 4, inp["sampling_locations"].shape[1], 4)
    one = ctypes.c_int64(0)
    assert lib.msda_backward_det_workspace(4, *dims, 1, ctypes.byref(one)) == 0 and one.value > 0
    assert lib.msda_backward_det_workspace(4, *dims, 0, ctypes.byref(one)) == -1                 # MSDA_E_BADARG
    ws = torch.empty(one.value - 1, dtype=torch.uint8, device=DEV)                                  # one query does not fit
    gv, gl, ga = torch.empty_like(v), torch.empty_like(inp["sampling_locations"]), torch.empty_like(inp["attention_weights"])
    code = lib.msda_backward_det_f32(inp["grad_output"].data_ptr(), *(t.data_ptr() for t in _args(inp)), *dims,
                                     gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), ws.data_ptr(), ws.numel(), None)
    assert code == -1
    big = ctypes.c_int64(0)
    assert lib.msda_backward_det_workspace(4, 1, 1 << 29, 9, 32, 4, 10, 4, 1, ctypes.byref(big)) == -2   # M*S + 1 > 2^32


# ---- 5. CUDA graph ---------------------------------------------------------------------------------------------------
def test_cuda_graph_replay_equals_eager():
    inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=9)
    eager = _det(inp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _det(inp)                                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _det(inp)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(captured, eager):
            assert torch.equal(a, b)


# ---- 6. torch.use_deterministic_algorithms ---------------------------------------------------------------------------
class _DeterministicFlag:
    def __init__(self, warn_only=False):
        self.warn_only = warn_only

    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(True, warn_only=self.warn_only)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])


@pytest.mark.parametrize("fn", ["fp32", "bf16"])
def test_autograd_function_under_torch_flag_equals_oracle(fn):
    if fn == "fp32":
        inp = make_inputs(CONFIGS["cfg1"], "enc", DEV, seed=12, wild_fraction=0.02)
        value = inp["value"].clone().requires_grad_(True)
        func = MSDeformAttnFunction
    else:
        inp = _small(32, torch.bfloat16, seed=13)
        value = inp["value"].float().requires_grad_(True)      # fp32 value: MSDeformAttnFunctionBF16 returns the accumulator
        func = MSDeformAttnFunctionBF16
    with _DeterministicFlag():
        out = func.apply(value, inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
                         inp["attention_weights"], 64)
        out.backward(inp["grad_output"].to(out.dtype))
    assert np.array_equal(_np(value.grad), _oracle_gv(inp))


def test_fused_wrappers_take_stock_torch_under_flag():
    from uninext_b200.functions.fused import add_layer_norm, colsum
    lib = _cabi.load()
    norm = torch.nn.LayerNorm(256).to(DEV)
    a = torch.randn(1000, 256, device=DEV, requires_grad=True)
    b = torch.randn(1000, 256, device=DEV, requires_grad=True)
    x = torch.randn(1000, 256, device=DEV)
    before = lib.msda_launch_count()
    add_layer_norm(a, b, norm).sum().backward()
    colsum(x)
    torch.cuda.synchronize()
    assert lib.msda_launch_count() > before                    # premise: without the flag the library's kernels run
    with _DeterministicFlag():
        before = lib.msda_launch_count()
        y = add_layer_norm(a, b, norm)
        y.sum().backward()
        cs = colsum(x)
        torch.cuda.synchronize()
        assert lib.msda_launch_count() == before
    assert torch.equal(cs, x.sum(0))


def _condinst_case():
    from uninext_b200.modules.dynamic_mask_head import dynamic_mask_with_coords
    g = torch.Generator(device=DEV).manual_seed(14)
    feats = torch.randn(1, 8, 16, 20, generator=g, device=DEV, requires_grad=True)
    params = (0.1 * torch.randn(1, 3, 169, generator=g, device=DEV)).requires_grad_(True)
    refs = torch.rand(1, 3, 2, generator=g, device=DEV) * 64
    return dynamic_mask_with_coords(feats, refs, params, [3], 8, True, 4)


def test_condinst_backward_raises_under_flag_and_warns_under_warn_only():
    with _DeterministicFlag():
        logits = _condinst_case()
        with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
            logits.sum().backward()
    with _DeterministicFlag(warn_only=True):
        logits = _condinst_case()
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            logits.sum().backward()
        assert any("use_deterministic_algorithms" in str(w.message) for w in rec)


# ---- 7. whole layers, twice, bit for bit -----------------------------------------------------------------------------
_LAYER_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, sys.argv[1])
    torch.use_deterministic_algorithms(True)
    from uninext_b200.modules.deformable_layers import DeformableTransformerEncoderLayer
    from uninext_b200.modules.ms_deform_attn import MSDeformAttn
    from uninext_b200.workloads import CONFIGS, encoder_reference_points, level_tensors
    dev = "cuda"
    cfg = CONFIGS["cfg1"]
    ss, lsi = level_tensors(cfg.shapes, dev)
    torch.manual_seed(0)
    enc = DeformableTransformerEncoderLayer(d_ffn=512, dropout=0.0).to(dev)
    dec = MSDeformAttn(256, 4, 8, 4).to(dev)
    n, s, lq = 2, cfg.S, 100
    src = torch.randn(n, s, 256, device=dev)
    pos = torch.randn(n, s, 256, device=dev)
    ref = encoder_reference_points(cfg.shapes, dev).view(1, s, 1, 2).expand(n, s, 4, 2).contiguous()
    query = torch.randn(n, lq, 256, device=dev)
    boxes = torch.cat((torch.rand(n, lq, 1, 2, device=dev), 0.05 + 0.3 * torch.rand(n, lq, 1, 2, device=dev)), -1)
    boxes = boxes.expand(n, lq, 4, 4).contiguous()
    g_enc = torch.randn(n, s, 256, device=dev)
    g_dec = torch.randn(n, lq, 256, device=dev)

    def run():
        enc.zero_grad(set_to_none=True); dec.zero_grad(set_to_none=True)
        x = src.clone().requires_grad_(True); p = pos.clone().requires_grad_(True)
        q = query.clone().requires_grad_(True); f = src.clone().requires_grad_(True)
        y = enc(x, p, ref, ss, lsi)
        z = dec(q, boxes, f, ss, lsi)
        torch.autograd.backward((y, z), (g_enc, g_dec))
        res = [y, z, x.grad, p.grad, q.grad, f.grad]
        res += [t.grad for t in enc.parameters()] + [t.grad for t in dec.parameters()]
        return [t.detach().clone() for t in res]

    a, b = run(), run()
    bad = [i for i, (u, v) in enumerate(zip(a, b)) if u is None or not torch.equal(u, v)]
    print("DIFFER", bad)
    sys.exit(1 if bad else 0)
""")


def test_encoder_and_decoder_layers_are_bitwise_reproducible():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    proc = subprocess.run([sys.executable, "-c", _LAYER_SCRIPT, ROOT], env=env, capture_output=True, text=True,
                          timeout=600)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]
