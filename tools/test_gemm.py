#!/usr/bin/env python
"""Bring-up check for msda_linear_tf32 (wgmma TF32 GEMM): compare with torch (TF32 tolerance), then time it vs cuBLAS."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200 import _cabi
lib = _cabi.load()

def linear_tf32(a, w, b):
    m, k = a.shape; n = w.shape[0]
    c = torch.empty((m, n), dtype=torch.float32, device=a.device)
    rc = lib.msda_linear_tf32(a.data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None, m, n, k, c.data_ptr(),
                              torch.cuda.current_stream().cuda_stream)
    assert rc == 0, (rc, lib.msda_strerror(rc))
    return c

torch.manual_seed(0)
ok = True
for (m, n, k) in [(128, 256, 256), (128, 64, 32), (300, 256, 256), (1000, 384, 256), (44646, 256, 256), (44646, 384, 256), (513, 512, 64), (77, 32, 96), (200, 448, 128)]:
    a = torch.randn(m, k, device="cuda"); w = torch.randn(n, k, device="cuda") * 0.1; b = torch.randn(n, device="cuda")
    c = linear_tf32(a, w, b)
    torch.cuda.synchronize()
    ref = a.double() @ w.double().t() + b.double()
    err = ((c.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"M={m} N={n} K={k}: rel err {err:.2e}", "OK" if err < 2e-3 else "FAIL")
    ok &= err < 2e-3
if not ok:
    sys.exit(1)
torch.backends.cuda.matmul.allow_tf32 = True
for (m, n, k) in [(44646, 256, 256), (44646, 384, 256)]:
    a = torch.randn(m, k, device="cuda"); w = torch.randn(n, k, device="cuda") * 0.1; b = torch.randn(n, device="cuda")
    for name, fn in (("wgmma-tf32", lambda: linear_tf32(a, w, b)), ("cublas-tf32", lambda: torch.addmm(b, a, w.t()))):
        for _ in range(5): fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20): fn()
        e1.record(); torch.cuda.synchronize()
        print(f"{name:12s} M={m} N={n}: {e0.elapsed_time(e1)/20*1e3:.1f} us")
