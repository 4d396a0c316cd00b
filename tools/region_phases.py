#!/usr/bin/env python
"""Per-kernel and per-phase time of the fp32 encoder backward (uninext_b200/csrc/msda_region.cuh) on the bench's first
cfg2 encoder input (seed 1000), for each halo of a sweep.

    python tools/region_phases.py [--halos 1,2,3,4,5,6] [--ctas 0] [--iters 30] [--config cfg2] [--csrc DIR]

Compiles tools/region_phases.cu -- the kernel header with the MSDA_REGION_PHASE_CLOCKS hook, msda_bwd_region<8, HALO>
(tap pass) and msda_region_grad_value_pass<8, HALO> for HALO in 1..6 -- with nvcc for sm_90a into a temporary
directory, and launches them as the library does, but one after the other without the PDL pairing.  Thread 0 of each
grad_value CTA sums clock64() spans taken after CTA barriers: tile geometry and count reset, phase A (tap geometry,
entries, direct reds), phase B (sort), phase C (row sums, one red per touched row).
Prints, per halo and grad_value occupancy (--ctas: comma-separated caps on its CTAs per SM, reached by padding its
dynamic shared memory; 0 = as the library launches it):
  - the tap kernel's and the grad_value kernel's times (CUDA events, median of `iters` launches; no zero-fill, no L2
    flush);
  - each grad_value span's share of its CTA's cycles, median over CTAs, and that share of the kernel time;
  - the knockout times of the grad_value kernel: no phase-A reds, no phase-C reds, neither (results wrong by
    construction: timing only);
and the GPU's name and power limit.  --csrc points the driver at another copy of the kernel headers with the same hook
and launch signature, for before / after tables."""
import argparse
import ctypes
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from uninext_b200 import build as libbuild  # noqa: E402
from uninext_b200.workloads import CONFIGS, make_inputs  # noqa: E402

SPANS = ("tile geometry", "phase A", "phase B", "phase C")
KNOCKOUTS = ((1, "no phase-A reds"), (2, "no phase-C reds"), (3, "no reds at all"))


def compile_driver(csrc, out_dir):
    so = os.path.join(out_dir, "libregion_phases.so")
    cmd = [libbuild.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--shared",
           "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I", csrc, "-I", libbuild.INCLUDE,
           "-o", so, os.path.join(ROOT, "tools", "region_phases.cu")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise SystemExit("nvcc failed building the region_phases driver")
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--halos", default="1,2,3,4,5,6")
    ap.add_argument("--ctas", default="0")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--csrc", default=libbuild.CSRC, help="directory holding msda_region.cuh and its includes")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("region_phases.py needs a CUDA device")
    halos = [int(h) for h in args.halos.split(",")]

    tmp = tempfile.mkdtemp(prefix="region_phases_")
    try:
        lib = ctypes.CDLL(compile_driver(os.path.abspath(args.csrc), tmp))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)      # the loaded library stays mapped
    nspans = lib.region_phases_spans()
    assert nspans == len(SPANS), (nspans, SPANS)
    fn = lib.region_phases_run
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 6 + \
        [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3

    inp = make_inputs(CONFIGS[args.config], "enc", "cuda", seed=1000)
    v, loc, attn, go = inp["value"], inp["sampling_locations"], inp["attention_weights"], inp["grad_output"]
    shapes, lsi = inp["spatial_shapes"], inp["level_start_index"]
    N, S, M, D = v.shape
    Lq, L, P = loc.shape[1], loc.shape[3], loc.shape[4]
    gv, gl, ga = torch.zeros_like(v), torch.zeros_like(loc), torch.zeros_like(attn)
    ptrs = [t.data_ptr() for t in (go, v, shapes, lsi, loc, attn)]
    dims = [N, S, M, L, Lq, P]
    outs = [t.data_ptr() for t in (gv, gl, ga)]

    def run(halo, which, ctas, knockout, clocks):
        if fn(halo, 1, ctas, 1, clocks.data_ptr(), knockout, *ptrs, *dims, *outs) < 0:
            raise SystemExit(f"driver setup failed (halo {halo})")
        xs = []
        for i in range(args.iters + 3):
            gv.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if fn(halo, which, ctas, 0, clocks.data_ptr(), knockout, *ptrs, *dims, *outs) < 0:
                raise SystemExit(f"launch failed (halo {halo})")
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                xs.append(e0.elapsed_time(e1))
        return statistics.median(xs)

    print(f"device: {device_identity()}")
    print(f"{args.config} encoder input (seed 1000): N={N} S={S} M={M} D={D} L={L} P={P}; msda_bwd_region<8, halo> and "
          f"msda_region_grad_value_pass<8, halo> with the phase-clock hook, median of {args.iters} launches; "
          f"csrc {os.path.relpath(os.path.abspath(args.csrc), ROOT)}")
    for halo in halos:
        for ctas in [int(c) for c in args.ctas.split(",")]:
            grid = fn(halo, 1, ctas, 1, 0, 0, *ptrs, *dims, *outs)
            clocks = torch.zeros(grid * nspans, dtype=torch.int64, device="cuda")
            tap_ms = run(halo, 0, ctas, 0, clocks)
            ms = run(halo, 1, ctas, 0, clocks)
            c = clocks.view(grid, nspans).double().cpu()
            c = c[c.sum(1) > 0]
            shares = c / c.sum(1, keepdim=True)
            med = [float(shares[:, k].median()) for k in range(nspans)]
            print(f"--- halo {halo}: tap kernel {tap_ms:.4f} ms; grad_value kernel {ms:.4f} ms ({grid} CTAs, "
                  f"{grid // torch.cuda.get_device_properties(0).multi_processor_count} per SM)")
            for k, name in enumerate(SPANS):
                print(f"  {name:17s} {100 * med[k]:5.1f} %  ~{med[k] * ms:.4f} ms")
            for bits, name in KNOCKOUTS:
                kms = run(halo, 1, ctas, bits, torch.zeros_like(clocks))
                print(f"  knockout, {name:15s} {kms:.4f} ms  ({kms - ms:+.4f} ms)")

if __name__ == "__main__":
    main()
