"""Every kernel instantiation of the op, run at the launch sizes and inputs that select it and compared with the oracle.

The router (uninext_b200/csrc/msda_cabi.cu) picks a kernel from the dtype, D, L*P, the input alignment, the knobs and the
launch size: launches of at most 56 pairs per SM run the SPLIT variants of the tiled kernels, larger ones the non-split
variants, with TMA-staged taps when L*P % 4 == 0 and plain loads otherwise.  ROUTES is a table of cases, each naming the
instantiations it must run, written out as the compiler names them.  Launch sizes are given in units of the split
threshold and resolved from the device's SM count.  For every row:
  - forward and backward through the drop-in against the fp64 C oracle, with border and out-of-map taps;
  - the C ABI once more into outputs pre-filled with NaN: every element is written, grad_value is zero where no tap lands;
  - torch.profiler: the named instantiations, and no other kernel of the five families, ran;
  - deterministic rows: grad_value equals the C oracle bit for bit, grad_loc / grad_attn equal the default route's.

test_every_instantiation_has_a_route runs without a GPU: it reads the instantiations from the built library and fails
when one has no row, or a row names one the library does not have.  The opt-in slab / tmem kernels are tested in
test_gpu_slab.py.

test_offsets_past_2_31_elements runs a value tensor of 2.2e9 elements, whose second batch element starts past 2^31
elements and ends past 2^33 bytes, against an fp64 reference over the rows its taps touch."""
import math
import os
import re
import subprocess
import time
import zlib

import numpy as np
import pytest
import torch

from oracle import msda_oracle
from tests.test_gpu_deterministic import _oracle_gv
from tests.test_gpu_parity import _gl_ok, _maxerr
from tests.test_gpu_region_bwd import _encoder_inputs
from uninext_b200 import build as _build
from uninext_b200.workloads import level_tensors

if torch.cuda.is_available():
    from uninext_b200 import _cabi
    from uninext_b200.dropin import MultiScaleDeformableAttention as MSDA

DEV = "cuda"
F32, BF16, F64 = "float32", "bfloat16", "float64"
TOL = {F32: 1e-4, BF16: 1e-2, F64: 1e-10}
FAMILY = re.compile(r"(msda_(?:fwd_tiled|bwd_tiled|bwd_region|fwd_generic|bwd_generic)<[^<>()]*>)")

# level tables: decoder-shaped calls (Lq independent of S) and encoder pyramids (odd S)
T2 = [(24, 36), (12, 18)]
T3 = [(20, 30), (10, 15), (5, 8)]
T4 = [(20, 30), (10, 15), (5, 8), (3, 4)]
T8 = [(12, 16), (10, 12), (8, 10), (6, 8), (5, 6), (4, 5), (3, 4), (2, 3)]
T9 = T8 + [(1, 1)]
ENC4 = [(33, 31), (17, 16), (9, 8), (5, 4)]
ENC3 = [(33, 31), (17, 16), (9, 8)]

VEC8 = (("F32_VEC8_FWD", 1), ("F32_VEC8_BWD", 1))
PACKED = (("BF16_PACKED_FWD", 1),)
FINE = (("BF16_FINE_ROWS", 500),)        # the 1023-row level accumulates in bf16, the coarser ones in fp32


def _row(rid, dtype, D, shapes, P, kind, N, M, size, kernels, knobs=(), align="aligned", det=False):
    """size = (f, k): about f x (56 x SM count) + k pairs.  Decoder rows take N and M as given and round Lq up (to an odd
    number when N*M > 1, so that no group count divides the pairs); encoder rows (Lq == S) round N up."""
    return dict(id=rid, dtype=dtype, D=D, shapes=shapes, P=P, kind=kind, N=N, M=M, size=size, kernels=kernels,
                knobs=knobs, align=align, det=det)


BIG, SMALL, TINY = (2.5, 0), (0.25, 0), (0.05, 0)

ROUTES = [
    # ---- default route, non-split: every (dtype, D, LP_MAX, TMA / LDG); odd M and pair counts; L*P < LP_MAX ----------
    _row("f32-d16-tma-enc", F32, 16, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, true, false, false, false>"]),
    _row("f32-d16-ldg", F32, 16, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, false, false, false, false>"]),
    _row("f32-d16-lp32", F32, 16, T8, 3, "dec", 3, 5, BIG,
         ["msda_fwd_tiled<float, 4, 16, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 16, 32, 2, false, false, false, false>"]),
    _row("f32-d32-tma", F32, 32, T2, 4, "dec", 3, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, true, false, false, false>"]),
    _row("f32-d32-ldg", F32, 32, T3, 3, "dec", 1, 5, BIG,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, false, false, false, false>"]),
    _row("f32-d32-lp32", F32, 32, T4, 5, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 32, 32, 2, false, false, false, false>"]),
    _row("f32-d64-tma-enc", F32, 64, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, true, false, false, false>"]),
    _row("f32-d64-ldg", F32, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, false, false, false>"]),
    _row("f32-d64-lp32", F32, 64, T8, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 64, 32, 2, false, false, false, false>"]),
    _row("f32-d32-region-enc", F32, 32, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>", "msda_bwd_region<8, 2>"]),
    _row("bf16-d32-tma-enc", BF16, 32, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, true, false, false, false>"]),
    _row("bf16-d32-ldg", BF16, 32, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, false, false, false>"]),
    _row("bf16-d32-lp32", BF16, 32, T8, 4, "dec", 1, 5, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 32, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 32, 2, false, false, false, false>"]),
    _row("bf16-d64-tma", BF16, 64, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, true, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, true, false, false, false>"]),
    _row("bf16-d64-ldg", BF16, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, false, false, false, false>"]),
    _row("bf16-d64-lp32", BF16, 64, T4, 5, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 32, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 32, 2, false, false, false, false>"]),
    # ---- the split boundary: exactly 56 x SM count pairs is split, one more is not --------------------------------------
    _row("f32-d32-split-at-threshold", F32, 32, T4, 4, "dec", 1, 1, (1, 0),
         ["msda_fwd_tiled<float, 4, 32, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, false, true, false, false>"]),
    _row("f32-d32-tma-past-threshold", F32, 32, T4, 4, "dec", 1, 1, (1, 1),
         ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, true, false, false, false>"]),
    # ---- default route, split ------------------------------------------------------------------------------------------
    _row("f32-d16-split", F32, 16, T2, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, false, true, false, false>"]),
    _row("f32-d16-lp32-split", F32, 16, T8, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 16, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 16, 32, 2, false, true, false, false>"]),
    _row("f32-d32-lp32-split", F32, 32, T4, 5, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 32, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 32, 32, 2, false, true, false, false>"]),
    _row("f32-d64-split", F32, 64, T3, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, true, false, false>"]),
    _row("f32-d64-lp32-split", F32, 64, T8, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 64, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 64, 32, 2, false, true, false, false>"]),
    _row("bf16-d32-split", BF16, 32, T2, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, true, false, false>"]),
    _row("bf16-d32-lp32-split", BF16, 32, T8, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 32, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 32, 2, false, true, false, false>"]),
    _row("bf16-d64-split", BF16, 64, T3, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, false, true, false, false>"]),
    _row("bf16-d64-lp32-split", BF16, 64, T4, 5, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 32, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 32, 2, false, true, false, false>"]),
    # ---- fp32 32-byte lanes (MSDA_KNOB_F32_VEC8_FWD / _BWD; the backward has them at D = 32 only) -----------------------
    _row("f32-vec8-d32-tma", F32, 32, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 8, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 8, 32, 16, 2, true, false, false, false>"], knobs=VEC8),
    _row("f32-vec8-d32-ldg", F32, 32, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 8, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 8, 32, 16, 2, false, false, false, false>"], knobs=VEC8),
    _row("f32-vec8-d32-split", F32, 32, T4, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 8, 32, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 8, 32, 16, 2, false, true, false, false>"], knobs=VEC8),
    _row("f32-vec8-d64-tma-enc", F32, 64, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<float, 8, 64, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, true, false, false, false>"], knobs=VEC8),
    _row("f32-vec8-d64-ldg", F32, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 8, 64, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, false, false, false>"], knobs=VEC8),
    _row("f32-vec8-d64-split", F32, 64, T2, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 8, 64, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, true, false, false>"], knobs=VEC8),
    # ---- bf16 forward with the packed corner blend (MSDA_KNOB_BF16_PACKED_FWD): non-split launches only ---------------
    _row("bf16-packed-d32-tma", BF16, 32, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, true, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, true, false, false, false>"], knobs=PACKED),
    _row("bf16-packed-d32-ldg", BF16, 32, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, false, false, false>"], knobs=PACKED),
    _row("bf16-packed-d32-lp32", BF16, 32, T8, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 32, 4, false, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 32, 2, false, false, false, false>"], knobs=PACKED),
    _row("bf16-packed-d64-tma-enc", BF16, 64, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, true, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, true, false, false, false>"], knobs=PACKED),
    _row("bf16-packed-d64-ldg", BF16, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, false, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, false, false, false, false>"], knobs=PACKED),
    _row("bf16-packed-d64-lp32", BF16, 64, T4, 5, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 32, 4, false, false, true>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 32, 2, false, false, false, false>"], knobs=PACKED),
    # ---- bf16 backward with the fine levels accumulated in bf16 (MSDA_KNOB_BF16_FINE_ROWS) -----------------------------
    _row("bf16-fine-rows-tma-enc", BF16, 32, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, true, false, true, false>"], knobs=FINE),
    _row("bf16-fine-rows-ldg-enc", BF16, 32, ENC3, 3, "enc", None, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, false, true, false>"], knobs=FINE),
    # ---- deterministic route: grad_loc / grad_attn from the NORED kernels, grad_value summed in a fixed order ----------
    _row("det-f32-d16-tma-enc", F32, 16, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, true, false, false, true>"], det=True),
    _row("det-f32-d16-ldg", F32, 16, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, false, false, false, true>"], det=True),
    _row("det-f32-d16-lp32", F32, 16, T8, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 16, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 16, 32, 2, false, false, false, true>"], det=True),
    _row("det-f32-d16-split", F32, 16, T2, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 16, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 16, 16, 2, false, true, false, true>"], det=True),
    _row("det-f32-d16-lp32-split", F32, 16, T8, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 16, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 16, 32, 2, false, true, false, true>"], det=True),
    _row("det-f32-d32-tma-enc", F32, 32, ENC4, 4, "enc", None, 3, BIG,        # default route: msda_bwd_region
         ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, true, false, false, true>"], det=True),
    _row("det-f32-d32-ldg", F32, 32, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, false, false, false, true>"], det=True),
    _row("det-f32-d32-lp32", F32, 32, T4, 5, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 32, 32, 2, false, false, false, true>"], det=True),
    _row("det-f32-d32-split", F32, 32, T4, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, false, true, false, true>"], det=True),
    _row("det-f32-d32-lp32-split", F32, 32, T4, 5, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 32, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 32, 32, 2, false, true, false, true>"], det=True),
    _row("det-f32-d64-tma", F32, 64, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, true, false, false, true>"], det=True),
    _row("det-f32-d64-ldg", F32, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, false, false, true>"], det=True),
    _row("det-f32-d64-lp32", F32, 64, T8, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 64, 32, 4, false, false, false>",
          "msda_bwd_tiled<float, 4, 64, 32, 2, false, false, false, true>"], det=True),
    _row("det-f32-d64-split", F32, 64, T3, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 64, 16, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 64, 16, 2, false, true, false, true>"], det=True),
    _row("det-f32-d64-lp32-split", F32, 64, T8, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<float, 4, 64, 32, 4, false, true, false>",
          "msda_bwd_tiled<float, 4, 64, 32, 2, false, true, false, true>"], det=True),
    _row("det-bf16-d32-tma-enc", BF16, 32, ENC4, 4, "enc", None, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, true, false, false, true>"], det=True),
    _row("det-bf16-d32-ldg", BF16, 32, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, false, false, true>"], det=True),
    _row("det-bf16-d32-lp32", BF16, 32, T8, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 32, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 32, 2, false, false, false, true>"], det=True),
    _row("det-bf16-d32-split", BF16, 32, T2, 4, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, true, false, true>"], det=True),
    _row("det-bf16-d32-lp32-split", BF16, 32, T8, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 32, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 32, 32, 2, false, true, false, true>"], det=True),
    _row("det-bf16-d64-tma", BF16, 64, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, true, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, true, false, false, true>"], det=True),
    _row("det-bf16-d64-ldg", BF16, 64, T3, 3, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, false, false, false, true>"], det=True),
    _row("det-bf16-d64-lp32", BF16, 64, T4, 5, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 32, 4, false, false, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 32, 2, false, false, false, true>"], det=True),
    _row("det-bf16-d64-split", BF16, 64, T3, 3, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 16, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 16, 2, false, true, false, true>"], det=True),
    _row("det-bf16-d64-lp32-split", BF16, 64, T4, 5, "dec", 1, 3, SMALL,
         ["msda_fwd_tiled<__nv_bfloat16, 8, 64, 32, 4, false, true, false>",
          "msda_bwd_tiled<__nv_bfloat16, 4, 64, 32, 2, false, true, false, true>"], det=True),
    # ---- alignment: views offset by one element run the generic kernels; a value that is 16-byte but not 32-byte
    #      aligned keeps the 16-byte-lane tiled kernels with the VEC8 knobs on ------------------------------------------
    _row("f32-offset-views", F32, 32, T4, 4, "dec", 1, 3, BIG,
         ["msda_fwd_generic<float, float>", "msda_bwd_generic<float, float, float, false>"], align="offset1"),
    _row("bf16-offset-views", BF16, 32, T4, 4, "dec", 1, 3, BIG,
         ["msda_fwd_generic<__nv_bfloat16, float>", "msda_bwd_generic<__nv_bfloat16, float, float, false>"],
         align="offset1"),
    _row("f32-vec8-value-16b-aligned", F32, 32, T2, 4, "dec", 1, 3, BIG,
         ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>",
          "msda_bwd_tiled<float, 4, 32, 16, 2, true, false, false, false>"], knobs=VEC8, align="value16"),
    # ---- generic kernels: fp64, odd D, L > 8, L*P > 32 -------------------------------------------------------------------
    _row("f64", F64, 32, T4, 4, "dec", 1, 3, TINY,
         ["msda_fwd_generic<double, double>", "msda_bwd_generic<double, double, double, false>"]),
    _row("det-f64", F64, 32, T4, 4, "dec", 1, 3, TINY,
         ["msda_fwd_generic<double, double>", "msda_bwd_generic<double, double, double, true>"], det=True),
    _row("f32-d24", F32, 24, T3, 3, "dec", 1, 3, TINY,
         ["msda_fwd_generic<float, float>", "msda_bwd_generic<float, float, float, false>"]),
    _row("det-f32-l9", F32, 32, T9, 2, "dec", 1, 3, TINY,
         ["msda_fwd_generic<float, float>", "msda_bwd_generic<float, float, float, true>"], det=True),
    _row("bf16-lp40", BF16, 32, T8, 5, "dec", 1, 3, TINY,
         ["msda_fwd_generic<__nv_bfloat16, float>", "msda_bwd_generic<__nv_bfloat16, float, float, false>"]),
    _row("det-bf16-d48", BF16, 48, T3, 3, "dec", 1, 3, TINY,
         ["msda_fwd_generic<__nv_bfloat16, float>", "msda_bwd_generic<__nv_bfloat16, float, float, true>"], det=True),
]


# ---- CPU: every instantiation in the library has a row -------------------------------------------------------------------
def _canonical(name):
    """A kernel name as the table writes it (demanglers may spell bools as (bool)0 / (bool)1)."""
    return re.sub(r"\s+", " ", name.replace("(bool)0", "false").replace("(bool)1", "true"))


def test_every_instantiation_has_a_route():
    lib = os.path.join(_build.LIB_DIR, "libmsda_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    syms = subprocess.run(["nm", "-C", lib], capture_output=True, text=True, check=True).stdout
    built = {_canonical(m.group(1)) for m in FAMILY.finditer(syms)}
    named = {k for r in ROUTES for k in r["kernels"]}
    assert built, "no msda_fwd_tiled / msda_bwd_tiled / msda_bwd_region / msda_*_generic symbol in " + lib
    assert not built - named, f"instantiations without a row in ROUTES: {sorted(built - named)}"
    assert not named - built, f"rows name instantiations the library does not have: {sorted(named - built)}"


# ---- GPU: the table ------------------------------------------------------------------------------------------------------
@pytest.fixture
def knobs():
    lib = _cabi.load()
    saved = [lib.msda_set_knob(k, -1000000) for k in range(10)]
    yield lib
    for k, v in enumerate(saved):
        lib.msda_set_knob(k, v)


def _split_threshold():
    return 56 * torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _decoder_inputs(shapes, N, Lq, M, D, P, dtype, seed, wild_fraction):
    """Decoder-shaped inputs (box queries, as workloads.make_inputs) for an arbitrary level table."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ss, lsi = level_tensors(shapes, DEV)
    L, S = len(shapes), sum(h * w for h, w in shapes)
    ctr = torch.rand(N, Lq, 1, 1, 1, 2, generator=g, device=DEV)
    box = 0.05 + 0.35 * torch.rand(N, Lq, 1, 1, 1, 2, generator=g, device=DEV)
    loc = ctr + torch.randn(N, Lq, M, L, P, 2, generator=g, device=DEV) / P * box * 0.5
    wild = torch.rand(loc.shape[:-1], generator=g, device=DEV) < wild_fraction
    loc = torch.where(wild[..., None], torch.rand(loc.shape, generator=g, device=DEV) * 2.0 - 0.5, loc)
    attn = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g, device=DEV), -1).view(N, Lq, M, L, P)
    aux = torch.float64 if dtype == torch.float64 else torch.float32
    return dict(value=torch.randn(N, S, M, D, generator=g, device=DEV).to(dtype), spatial_shapes=ss,
                level_start_index=lsi, sampling_locations=loc.to(aux).contiguous(),
                attention_weights=attn.to(aux).contiguous(),
                grad_output=torch.randn(N, Lq, M * D, generator=g, device=DEV).to(dtype))


def _inputs(row, thr):
    dtype = getattr(torch, row["dtype"])
    target = int(row["size"][0] * thr) + row["size"][1]
    M, seed = row["M"], zlib.crc32(row["id"].encode()) % 100000
    if row["kind"] == "enc":
        S = sum(h * w for h, w in row["shapes"])
        N = max(1, math.ceil(target / (S * M)))
        return _encoder_inputs(row["shapes"], N, M=M, D=row["D"], P=row["P"], seed=seed, wild_fraction=0.05,
                               dtype=dtype)
    N = row["N"]
    Lq = math.ceil(target / (N * M))
    if N * M > 1:
        Lq |= 1
    return _decoder_inputs(row["shapes"], N, Lq, M, row["D"], row["P"], dtype, seed, 0.05)


def _offset_copy(t, elems):
    """A contiguous view of a copy of t that starts `elems` elements into its allocation."""
    buf = torch.empty(t.numel() + elems, dtype=t.dtype, device=t.device)
    view = buf[elems:].view(t.shape)
    view.copy_(t)
    return view


def _aligned_as(row, inp):
    inp = dict(inp)
    if row["align"] == "offset1":
        for k in ("value", "sampling_locations", "attention_weights", "grad_output"):
            inp[k] = _offset_copy(inp[k], 1)
            assert inp[k].is_contiguous() and inp[k].data_ptr() % 16 != 0
    elif row["align"] == "value16":
        inp["value"] = _offset_copy(inp["value"], 4)
        assert inp["value"].data_ptr() % 32 == 16
    return inp


def _args(inp):
    return (inp["value"], inp["spatial_shapes"], inp["level_start_index"], inp["sampling_locations"],
            inp["attention_weights"])


def _dims(inp):
    n, s, m, d = inp["value"].shape
    return (n, s, m, d, inp["spatial_shapes"].shape[0], inp["sampling_locations"].shape[1],
            inp["sampling_locations"].shape[4])


def _run(row, inp):
    """Forward and backward through the drop-in; a deterministic bf16 row hands back the fp32 accumulator."""
    out = MSDA.ms_deform_attn_forward(*_args(inp), 64)
    kw = dict(deterministic=row["det"])
    if row["det"] and row["dtype"] == BF16:
        kw["grad_value_dtype"] = torch.float32
    gv, gl, ga = MSDA.ms_deform_attn_backward(*_args(inp), inp["grad_output"], 64, **kw)
    torch.cuda.synchronize()
    return out, gv, gl, ga


def _abi_into_nan(row, inp):
    """The C ABI called directly, into outputs pre-filled with NaN: (out, grad_value, grad_loc, grad_attn)."""
    lib = _cabi.load()
    v, ss, lsi, loc, at = _args(inp)
    go = inp["grad_output"]
    dims = _dims(inp)
    st = torch.cuda.current_stream().cuda_stream
    sfx = {F32: "f32", F64: "f64", BF16: "bf16"}[row["dtype"]]
    nan = float("nan")
    out = torch.full(go.shape, nan, dtype=go.dtype, device=DEV)
    code = getattr(lib, "msda_forward_" + sfx)(v.data_ptr(), ss.data_ptr(), lsi.data_ptr(), loc.data_ptr(), at.data_ptr(),
                                              *dims, out.data_ptr(), st)
    assert code == 0, lib.msda_strerror(code)
    gv, gl, ga = torch.full_like(v, nan), torch.full_like(loc, nan), torch.full_like(at, nan)
    grads = (gv.data_ptr(), gl.data_ptr(), ga.data_ptr())
    if row["dtype"] == BF16:           # fp32 accumulator (scratch of the coarse levels on the fine-rows route) + bf16 result
        acc = torch.full(v.shape, nan, dtype=torch.float32, device=DEV)
        grads = (acc.data_ptr(),) + grads
    tail = (st,)
    kind = "msda_backward_"
    if row["det"]:
        ws = MSDA._det_workspace(lib, v, dims)
        tail, kind = (ws.data_ptr(), ws.numel(), st), "msda_backward_det_"
    code = getattr(lib, kind + sfx)(go.data_ptr(), v.data_ptr(), ss.data_ptr(), lsi.data_ptr(), loc.data_ptr(),
                                    at.data_ptr(), *dims, *grads, *tail)
    torch.cuda.synchronize()
    assert code == 0, lib.msda_strerror(code)
    return out, gv, gl, ga


def _families(names):
    return {_canonical(m.group(1)) for n in names for m in FAMILY.finditer(n)}


def _profiled(fn, expected):
    """(fn's result, the kernels of the five families it ran, the names of every event recorded).  Now and then the
    profiler records a window's launches but delivers none of its kernel records, so a window whose kernels differ from
    `expected` is profiled again, up to four times: a call's route is fixed by its inputs and the knobs, so a wrong route
    fails every time."""
    for _ in range(4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=DEV).add_(1)          # the profiler can also lose the first kernels of its window
            torch.cuda.synchronize()
            res = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        ran = _families(names)
        if ran == expected:
            break
        time.sleep(0.5)
    return res, ran, names


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROUTES, ids=[r["id"] for r in ROUTES])
def test_route_vs_oracle(knobs, row):
    thr = _split_threshold()
    for name, value in row["knobs"]:
        knobs.msda_set_knob(getattr(_cabi, "KNOB_" + name), value)
    inp = _aligned_as(row, _inputs(row, thr))
    dims = _dims(inp)
    npairs = dims[0] * dims[5] * dims[2]

    (out, gv, gl, ga), ran, names = _profiled(lambda: _run(row, inp), set(row["kernels"]))
    assert ran == set(row["kernels"]), (row["id"], npairs, thr, sorted(ran), sorted(names))

    # against the fp64 oracle, and grad_loc strictly against the oracle in the kernels' compute type
    f64 = lambda t: t.detach().double().cpu().numpy()
    n = lambda t: t.detach().cpu().numpy()
    a = _args(inp)
    ss, lsi = n(a[1]), n(a[2])
    out_t = msda_oracle.forward(f64(a[0]), ss, lsi, f64(a[3]), f64(a[4]))
    gv_t, gl_t, ga_t = msda_oracle.backward(f64(inp["grad_output"]), f64(a[0]), ss, lsi, f64(a[3]), f64(a[4]))
    tol = TOL[row["dtype"]]
    assert _maxerr(f64(out), out_t) < tol
    assert _maxerr(f64(gv), gv_t) < tol
    assert _maxerr(f64(ga), ga_t) < tol
    assert _gl_ok(f64(gl), gl_t, 2 * tol)
    if row["dtype"] != F64:
        c = lambda t: t.detach().float().cpu().numpy()
        _, gl_c, _ = msda_oracle.backward(c(inp["grad_output"]), c(a[0]), ss, lsi, c(a[3]), c(a[4]))
        assert _maxerr(f64(gl), gl_c.astype(np.float64)) < 2 * tol

    # every output element written; grad_value zero where no tap lands
    o2, gv2, gl2, ga2 = _abi_into_nan(row, inp)
    for t in (o2, gv2, gl2, ga2):
        assert not t.isnan().any(), row["id"]
    assert torch.equal(o2, out) and torch.equal(gl2, gl) and torch.equal(ga2, ga)
    assert not gv2.double().cpu().numpy()[gv_t == 0].any()
    assert _maxerr(f64(gv2), gv_t) < tol

    if row["det"]:
        want = _oracle_gv(inp, np.float64 if row["dtype"] == F64 else np.float32)
        assert np.array_equal(n(gv), want)
        if row["dtype"] != BF16:
            assert torch.equal(gv2, gv)
        else:
            assert torch.equal(gv2, gv.to(torch.bfloat16))
        dgv, dgl, dga = MSDA.ms_deform_attn_backward(*a, inp["grad_output"], 64, deterministic=False)
        assert torch.equal(gl, dgl) and torch.equal(ga, dga)


# ---- offsets past 2^31 elements -------------------------------------------------------------------------------------------
def _touched_rows_reference(value, loc, attn, go, H, W):
    """fp64 forward and backward of a single-level call, over the rows its taps touch only: the four corners of every tap
    are gathered and their grad_value contributions index_add'ed into the touched (b, row, m) rows.  The pixel
    coordinates are the kernels' fp32 ones, as in the fp32 C oracle.
    -> out, grad_loc, grad_attn, touched row keys ((b * S + row) * M + m), grad_value of those rows."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    assert L == 1
    rows = value.view(-1, D)
    # the pixel coordinate as the kernels round it, fl(fl(y * H) - 0.5) in fp32: at 2048 pixels one fp32 ulp of it is
    # 2.4e-4 pixels, which moves a bilinear weight by more than the tolerance.  Everything after it is fp64.
    x, y = loc[..., 0].float(), loc[..., 1].float()                        # [N, Lq, M, 1, P]
    h_im, w_im = (y * H - 0.5).double(), (x * W - 0.5).double()
    inside = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
    h0, w0 = torch.floor(h_im), torch.floor(w_im)
    lh, lw = h_im - h0, w_im - w0
    hh, hw = 1 - lh, 1 - lw
    b = torch.arange(N, device=DEV).view(N, 1, 1, 1, 1)
    m = torch.arange(M, device=DEV).view(1, 1, M, 1, 1)
    a = attn.double()
    g = go.double().view(N, Lq, M, 1, 1, D)
    tg = g * a[..., None]                                                   # [N, Lq, M, 1, P, D]
    v, cw, keys = [], [], []
    for dy, dx, wk in ((0, 0, hh * hw), (0, 1, hh * lw), (1, 0, lh * hw), (1, 1, lh * lw)):
        hk, wk_ = (h0 + dy).long(), (w0 + dx).long()
        ok = inside & (hk >= 0) & (hk <= H - 1) & (wk_ >= 0) & (wk_ <= W - 1)
        key = torch.where(ok, (b * S + hk * W + wk_) * M + m, torch.zeros_like(hk))
        v.append(rows[key].double() * ok[..., None])
        cw.append(wk * ok)
        keys.append(torch.where(ok, key, torch.full_like(key, -1)))
    val = sum(c[..., None] * vk for c, vk in zip(cw, v))                    # [N, Lq, M, 1, P, D]
    out = (val * a[..., None]).sum((3, 4)).reshape(N, Lq, M * D)
    grad_attn = (g * val).sum(-1)
    gh = -hw[..., None] * v[0] - lw[..., None] * v[1] + hw[..., None] * v[2] + lw[..., None] * v[3]
    gw = -hh[..., None] * v[0] + hh[..., None] * v[1] - lh[..., None] * v[2] + lh[..., None] * v[3]
    grad_loc = torch.stack((W * (gw * tg).sum(-1), H * (gh * tg).sum(-1)), -1)
    key_all = torch.stack(keys, 0).view(-1)
    contrib = torch.stack([c[..., None] * tg for c in cw], 0).view(-1, D)
    live = key_all >= 0
    touched, inv = torch.unique(key_all[live], return_inverse=True)
    gv = torch.zeros(touched.numel(), D, dtype=torch.float64, device=DEV).index_add_(0, inv, contrib[live])
    return out, grad_loc, grad_attn, touched, gv



@pytest.mark.gpu
@pytest.mark.parametrize("dtype,lq,kernels", [
    (F32, 300, ["msda_fwd_tiled<float, 4, 32, 16, 4, false, true, false>",
                "msda_bwd_tiled<float, 4, 32, 16, 2, false, true, false, false>"]),
    (F32, 4096, ["msda_fwd_tiled<float, 4, 32, 16, 4, true, false, false>",
                 "msda_bwd_tiled<float, 4, 32, 16, 2, true, false, false, false>"]),
    (BF16, 300, ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, false, true, false>",
                 "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, false, true, false, false>"]),
    (BF16, 4096, ["msda_fwd_tiled<__nv_bfloat16, 8, 32, 16, 4, true, false, false>",
                  "msda_bwd_tiled<__nv_bfloat16, 4, 32, 16, 2, true, false, false, false>"]),
])
def test_offsets_past_2_31_elements(dtype, lq, kernels):
    """One 2048 x 2112 level, N = 2, M = 8, D = 32: value has 2.2e9 elements, and the rows of batch element 1 lie past
    2^31 elements (and, in fp32, past 2^33 bytes).  A quarter of batch element 1's queries sample the far corner of its
    map, the last rows of the tensor; 5 % of all taps land anywhere in or around the map."""
    free, _ = torch.cuda.mem_get_info()
    if free < 40 * 2 ** 30:
        pytest.skip(f"needs about 40 GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    H, W = 2048, 2112
    N, S, M, D, P = 2, H * W, 8, 32, 4
    dt = getattr(torch, dtype)
    g = torch.Generator(device=DEV).manual_seed(lq)
    value = torch.randn(N, S, M, D, generator=g, device=DEV, dtype=dt)
    ss, lsi = level_tensors([(H, W)], DEV)
    ctr = torch.rand(N, lq, 1, 1, 1, 2, generator=g, device=DEV)
    box = 0.05 + 0.35 * torch.rand(N, lq, 1, 1, 1, 2, generator=g, device=DEV)
    loc = ctr + torch.randn(N, lq, M, 1, P, 2, generator=g, device=DEV) / P * box * 0.5
    far = 1.0 - torch.rand(lq // 4, M, 1, P, 2, generator=g, device=DEV) * torch.tensor([3.0 / W, 3.0 / H], device=DEV)
    loc[1, :lq // 4] = far
    wild = torch.rand(loc.shape[:-1], generator=g, device=DEV) < 0.05
    loc = torch.where(wild[..., None], torch.rand(loc.shape, generator=g, device=DEV) * 2.0 - 0.5, loc).contiguous()
    attn = torch.softmax(torch.randn(N, lq, M, P, generator=g, device=DEV), -1).view(N, lq, M, 1, P).contiguous()
    go = torch.randn(N, lq, M * D, generator=g, device=DEV, dtype=dt)
    a = (value, ss, lsi, loc, attn)

    (out, (gv, gl, ga)), ran, names = _profiled(lambda: (MSDA.ms_deform_attn_forward(*a, 64),
                                                   MSDA.ms_deform_attn_backward(*a, go, 64, deterministic=False)),
                                         set(kernels))
    assert ran == set(kernels), (sorted(ran), sorted(names))

    out_t, gl_t, ga_t, touched, gv_t = _touched_rows_reference(value, loc, attn, go, H, W)
    assert int(touched.max()) * D >= 2 ** 31 and int(touched.min()) * D < 2 ** 31
    tol = TOL[dtype]
    n = lambda t: t.detach().double().cpu().numpy()
    assert _maxerr(n(out), n(out_t)) < tol
    assert _maxerr(n(ga), n(ga_t)) < tol
    assert _gl_ok(n(gl), n(gl_t), 2 * tol)
    rows = gv.view(-1, D)
    assert _maxerr(n(rows[touched]), n(gv_t)) < tol
    rows[touched] = 0
    assert not rows.any(), "grad_value has non-zero rows that no tap touches"
    del value, gv, rows, out, gl, ga
    torch.cuda.empty_cache()
