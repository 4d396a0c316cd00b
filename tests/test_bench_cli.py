"""CPU tests of bench.py's command-line contract (no GPU): the --impl reference arm prints one JSON line with the
contract's keys, and the product arm refuses to run without CUDA instead of falling back."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True, env=e,
                          timeout=600)


def test_reference_arm_prints_contract_line():
    p = _run("--impl", "reference", "--config", "cfg1", "--steps", "2", "--warmup", "1")
    assert p.returncode == 0, p.stderr[-2000:]
    line = json.loads(p.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "msdeformattn_fwd_bwd_gsamples_per_s"
    for key in ("value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert key in line, key
    assert line["steps"] == 2 and line["value"] > 0 and line["e2e"]["h2d_bytes_per_step"] == 0
    cb = line["cpu_baseline"]
    sys.path.insert(0, ROOT)
    from oracle import refpy
    assert cb["kind"] == ("reference" if refpy.available() else "port")
    assert cb["value"] == line["value"] and cb["cores"] >= 1 and "sample" in cb
    assert line["config"]["workload"].startswith("cfg1")
    # same `config` object as the product arm prints (the driver compares the two lines)
    import bench
    from uninext_b200.workloads import CONFIGS
    assert line["config"] == json.loads(json.dumps(bench.step_config(CONFIGS["cfg1"], 1)))


def test_reference_file_and_port_agree():
    """The reference's own ms_deform_attn_core_pytorch and the port bench.py falls back to are the same function: the
    port's outputs and autograd gradients on a seeded case match the reference's, stored in
    tests/golden/reference/core_pytorch.npz (tests/refgolden.py)."""
    import numpy as np
    sys.path.insert(0, ROOT)
    from oracle.msda_oracle import core_pytorch_port
    from tests import refgolden
    from uninext_b200.workloads import CONFIGS, make_inputs
    c = make_inputs(CONFIGS["cfg1"], "dec", "cpu", seed=5, wild_fraction=0.1)
    if refgolden.RECORDING:
        from oracle import refpy
        assert refpy.stage()
        fn = refpy.core_pytorch()
    else:
        fn = core_pytorch_port
    v = c["value"].clone().requires_grad_(True)
    lo = c["sampling_locations"].clone().requires_grad_(True)
    at = c["attention_weights"].clone().requires_grad_(True)
    out = fn(v, c["spatial_shapes"], lo, at)
    out.backward(c["grad_output"])
    got = {"out": out, "grad_value": v.grad, "grad_loc": lo.grad, "grad_attn": at.grad}
    if refgolden.RECORDING:
        for k, t in got.items():
            refgolden.put("core_pytorch", k, t)
        refgolden.flush("core_pytorch")
        return
    want = refgolden.load("core_pytorch")
    for k, t in got.items():
        assert tuple(t.shape) == tuple(want[k + ".shape"]), k
        assert np.allclose(refgolden.sample(t, want, k, "core_pytorch"), want[k], rtol=1e-5, atol=1e-6), k


def test_reference_arm_non_zero_ranks_exit_quietly():
    p = _run("--impl", "reference", "--config", "cfg1", "--steps", "1", "--warmup", "1", "--gpus", "2",
             env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert p.returncode == 0 and p.stdout.strip() == ""


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU refusal")
def test_product_arm_refuses_without_cuda():
    p = _run("--steps", "1", "--warmup", "1")
    assert p.returncode != 0 and "no CPU fallback" in (p.stderr + p.stdout)


def test_algorithmic_bytes_formula():
    sys.path.insert(0, ROOT)
    from uninext_b200.workloads import CONFIGS, algorithmic_bytes
    c = CONFIGS["cfg2"]
    n, s, m, d, lq = c.batch, c.S, c.heads, c.head_dim, c.S
    taps = c.samples("enc")
    fwd = n * s * m * d * 4 + taps * 8 + taps * 4 + n * lq * m * d * 4
    assert algorithmic_bytes(c, "enc", 4, "fwd") == fwd == 28 * taps
    assert algorithmic_bytes(c, "enc", 4, "bwd") == fwd + 2 * n * s * m * d * 4 + taps * 12 == 56 * taps
    assert algorithmic_bytes(c, "enc", 4, "fwd+bwd") == 84 * taps
    assert algorithmic_bytes(c, "enc", 2, "fwd") == 20 * taps             # bf16 value / out, fp32 loc / attn


def test_dump_outputs_writes_float_arrays_and_seeded_samples(tmp_path):
    """--dump-outputs: every file is float32 / float64; small arrays whole, large ones as the same seeded sample each run."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    calls = [{"kind": "enc"}, {"kind": "dec"}]
    g = torch.Generator().manual_seed(0)
    big, small = torch.randn(300, 400, generator=g), torch.randn(7, 3, generator=g).double()
    results = [(big, small, small, small), (small, big, small, small)]
    for d in (tmp_path / "a", tmp_path / "b"):
        bench.dump_outputs(str(d), calls, results)
    files = sorted(p.name for p in (tmp_path / "a").iterdir())
    assert "enc0_out.npy" in files and "enc0_out_index.npy" in files and "enc0_grad_value.npy" in files
    assert "dec1_grad_value_index.npy" in files and "dec1_out_index.npy" not in files   # file stem: kind + index % 6
    for name in files:
        a, b = np.load(tmp_path / "a" / name), np.load(tmp_path / "b" / name)
        assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), name
    idx = np.load(tmp_path / "a" / "enc0_out_index.npy").astype(np.int64)
    assert len(idx) == 1 << 16 and np.array_equal(np.load(tmp_path / "a" / "enc0_out.npy"), big.reshape(-1)[idx].numpy())
    assert np.array_equal(np.load(tmp_path / "a" / "enc0_grad_value.npy"), small.reshape(-1).float().numpy())
