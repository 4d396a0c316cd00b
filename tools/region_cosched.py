#!/usr/bin/env python
"""Where the region backward's two kernels run: CTA placement of the grad_value pass and the tap pass on the bench's first
cfg2 encoder input (seed 1000).

    python tools/region_cosched.py [--runs 5] [--config cfg2] [--json FILE]

Compiles tools/region_cosched.cu -- msda_region.cuh with the placement hook (MSDA_REGION_COSCHED), launched as the library
launches it: zero-fill -> msda_region_grad_value_pass (PDL secondary of the fill) -> msda_bwd_region (PDL secondary of
the grad_value kernel), grids and padding from msda::region_grids -- with nvcc for sm_90a into a temporary directory.  Thread 0 of
each CTA records its %smid and %globaltimer at its start and when its work is done.  Prints, for the last of `runs`
back-to-back region backwards (the earlier ones warm up):
  - both grids, and the CTAs per SM of each kernel (min / max over SMs);
  - the span of each kernel (first CTA start to last CTA end) and their overlap;
  - the fraction of the tap CTAs' time during which grad_value CTAs are resident on the same SM (the tap CTAs' spans
    summed, against the time within them covered by at least one grad_value CTA of their SM);
and the GPU's name and power limit.  Read-only instrumentation: the hook changes no result."""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from uninext_b200 import build as libbuild  # noqa: E402
from uninext_b200.workloads import CONFIGS, make_inputs  # noqa: E402


def compile_driver(out_dir):
    so = os.path.join(out_dir, "libregion_cosched.so")
    cmd = [libbuild.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--shared",
           "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", libbuild.CSRC, "-I", libbuild.INCLUDE,
           "-o", so, os.path.join(ROOT, "tools", "region_cosched.cu")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise SystemExit("nvcc failed building the region_cosched driver")
    return so


def device_identity():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        pl, mhz = [x.strip() for x in q.stdout.strip().split(",")]
        return f"{name}, power limit {float(pl):.0f} W, max SM clock {float(mhz):.0f} MHz"
    except (OSError, ValueError, subprocess.SubprocessError):
        return f"{name}, power limit unknown"


def union_length(intervals):
    total, end = 0, None
    for s, e in sorted(intervals):
        if end is None or s > end:
            total += e - s
            end = e
        elif e > end:
            total += e - end
            end = e
    return total


def placement(gv_rec, tap_rec, sms):
    """Per-kernel CTAs per SM, kernel spans and the tap CTAs' co-residency with grad_value CTAs, from [grid x 3] records
    {smid, start ns, end ns}."""
    per_sm = {"grad_value": [0] * sms, "tap": [0] * sms}
    gv_on = [[] for _ in range(sms)]
    for smid, s, e in gv_rec:
        per_sm["grad_value"][smid] += 1
        gv_on[smid].append((s, e))
    covered = spans = 0
    for smid, s, e in tap_rec:
        per_sm["tap"][smid] += 1
        clipped = [(max(s, a), min(e, b)) for a, b in gv_on[smid] if a < e and b > s]
        covered += union_length(clipped)
        spans += e - s
    t0 = min(int(gv_rec[:, 1].min()), int(tap_rec[:, 1].min()))
    gv_span = (int(gv_rec[:, 1].min()) - t0, int(gv_rec[:, 2].max()) - t0)
    tap_span = (int(tap_rec[:, 1].min()) - t0, int(tap_rec[:, 2].max()) - t0)
    return {
        "ctas_per_sm": {k: {"min": min(v), "max": max(v)} for k, v in per_sm.items()},
        "grad_value_span_us": [x / 1e3 for x in gv_span],
        "tap_span_us": [x / 1e3 for x in tap_span],
        "kernel_overlap_us": max(0, min(gv_span[1], tap_span[1]) - max(gv_span[0], tap_span[0])) / 1e3,
        "tap_time_beside_grad_value": covered / spans if spans else 0.0,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("region_cosched.py needs a CUDA device")

    tmp = tempfile.mkdtemp(prefix="region_cosched_")
    try:
        lib = ctypes.CDLL(compile_driver(tmp))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)      # the loaded library stays mapped
    grids = (ctypes.c_int * 4)()
    if lib.region_cosched_grids(grids) != 0:
        raise SystemExit("region_cosched_grids failed")
    gv_grid, tap_grid, sms, gv_smem = grids[0], grids[1], grids[2], grids[3]
    run = lib.region_cosched_run
    run.restype = ctypes.c_int
    run.argtypes = [ctypes.c_void_p] * 9 + [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3

    inp = make_inputs(CONFIGS[args.config], "enc", "cuda", seed=1000)
    v, loc, attn, go = inp["value"], inp["sampling_locations"], inp["attention_weights"], inp["grad_output"]
    shapes, lsi = inp["spatial_shapes"], inp["level_start_index"]
    N, S, M, D = v.shape
    Lq, L, P = loc.shape[1], loc.shape[3], loc.shape[4]
    gv, gl, ga = torch.empty_like(v), torch.empty_like(loc), torch.empty_like(attn)
    gv_rec = torch.zeros(gv_grid * 3, dtype=torch.int64, device="cuda")
    tap_rec = torch.zeros(tap_grid * 3, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(args.runs):
        if run(stream, gv_rec.data_ptr(), tap_rec.data_ptr(), go.data_ptr(), v.data_ptr(), shapes.data_ptr(),
               lsi.data_ptr(), loc.data_ptr(), attn.data_ptr(), N, S, M, L, Lq, P, gv.data_ptr(), gl.data_ptr(),
               ga.data_ptr()) != 0:
            raise SystemExit("region_cosched_run failed")
    torch.cuda.synchronize()
    res = placement(gv_rec.view(gv_grid, 3).cpu().numpy(), tap_rec.view(tap_grid, 3).cpu().numpy(), sms)
    res.update(device=device_identity(), config=args.config, grids={"grad_value": gv_grid, "tap": tap_grid, "sms": sms},
               grad_value_dynamic_smem=gv_smem)

    print(f"device: {res['device']}")
    print(f"{args.config} encoder input (seed 1000): N={N} S={S} M={M} D={D} L={L} P={P}; last of {args.runs} runs")
    print(f"grids: grad_value {gv_grid} CTAs ({gv_smem} B dynamic shared memory), tap {tap_grid} CTAs, {sms} SMs")
    for k, c in res["ctas_per_sm"].items():
        print(f"  {k:10s} CTAs per SM: min {c['min']}, max {c['max']}")
    print(f"grad_value kernel span {res['grad_value_span_us'][0]:.1f}-{res['grad_value_span_us'][1]:.1f} us, "
          f"tap kernel span {res['tap_span_us'][0]:.1f}-{res['tap_span_us'][1]:.1f} us, "
          f"overlap {res['kernel_overlap_us']:.1f} us")
    print(f"tap CTAs' time with grad_value CTAs resident on their SM: {100 * res['tap_time_beside_grad_value']:.1f} %")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
