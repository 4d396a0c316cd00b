"""CPU tests of uninext_b200._precision.tf32_allowed and the GEMM routing that uses it, each in a fresh process: once
torch's newer ``fp32_precision`` API has been used, reading ``allow_tf32`` in that process raises."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, sys.argv[1])
    exec(sys.argv[2])
    from uninext_b200._precision import tf32_allowed
    from uninext_b200.functions.fused import resolve_gemm
    print("RESULT", tf32_allowed(), resolve_gemm("auto"), resolve_gemm("cublas"))
""")


def _run(setter, gemm_auto=None):
    env = dict(os.environ)
    env.pop("MSDA_GEMM_AUTO", None)
    if gemm_auto:
        env["MSDA_GEMM_AUTO"] = gemm_auto
    proc = subprocess.run([sys.executable, "-c", _SCRIPT, ROOT, setter], capture_output=True, text=True, env=env,
                          timeout=300)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]
    return proc.stdout.split("RESULT", 1)[1].split()


@pytest.mark.parametrize("setter,allowed", [
    ("", "False"),
    ("torch.set_float32_matmul_precision('highest')", "False"),
    ("torch.backends.cuda.matmul.allow_tf32 = True", "True"),
    ("torch.set_float32_matmul_precision('high')", "True"),
    ("torch.backends.cuda.matmul.fp32_precision = 'tf32'", "True"),
    ("torch.backends.fp32_precision = 'tf32'", "True"),
])
def test_tf32_allowed_follows_every_setter(setter, allowed):
    assert _run(setter)[0] == allowed


@pytest.mark.parametrize("gemm_auto", [None, "tcgen05"])
def test_resolve_gemm_under_the_new_api_matches_the_legacy_api(gemm_auto):
    legacy = _run("torch.backends.cuda.matmul.allow_tf32 = True", gemm_auto)
    new = _run("torch.backends.cuda.matmul.fp32_precision = 'tf32'", gemm_auto)
    assert new == legacy
    assert legacy[1] == ("tcgen05" if gemm_auto else "cublas")
    assert _run("", gemm_auto)[1] == "cublas"
