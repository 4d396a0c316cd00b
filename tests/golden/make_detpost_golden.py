"""Writes tests/golden/detpost/outputs.npz: postprocess_detections' outputs on the inputs of tests/test_gpu_detpost.py
(tests/test_gpu_trackpost.py: golden_cases), as the library computed them before its NMS code was shared with the video
trackers' detection selection.  Needs a GPU.

    python tests/golden/make_detpost_golden.py [--lib path/to/libmsda_b200.so] [--out tests/golden/detpost/outputs.npz]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="the library to take the outputs from (default: the built one)")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "detpost", "outputs.npz"))
    a = ap.parse_args()
    from uninext_b200 import _cabi
    if a.lib:
        _cabi.LIB_PATH = os.path.abspath(a.lib)
    from tests.test_gpu_trackpost import golden_cases
    arrays = {}
    for name, call in golden_cases():
        got = call()
        for field, t in zip(got._fields, got):
            arrays[f"{name}/{field}"] = t.cpu().numpy()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    np.savez_compressed(a.out, **arrays)
    print(f"{a.out}: {len(arrays)} arrays from {_cabi.LIB_PATH}")


if __name__ == "__main__":
    main()
