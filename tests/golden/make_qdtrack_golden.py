#!/usr/bin/env python
"""Regenerate tests/golden/qdtrack/*.npz: what the reference's own ``QuasiDenseEmbedTracker`` (models/tracker.py of a
reference checkout, with its real util/mmcv_utils.py, both loaded in place) returns and keeps on the CPU for the seeded
sequences of tests/qdtrack_case.py, one file per setting of ``qdtrack_case.SETTINGS``.  Per frame: the kept input rows
in the order returned, their ids, the returned indices; the live tracklets' id, last_frame, label and embed; the
backdrops' labels and embeds.  The tests do not need the reference.

    python tests/golden/make_qdtrack_golden.py
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refpy import REFERENCE  # noqa: E402
from tests import qdtrack_case as qc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "qdtrack")
PKG = os.path.join(REFERENCE, "projects", "UNINEXT", "uninext")


def load_reference_tracker():
    """models/tracker.py as module ``_qd_ref.models.tracker``, its ``..util.mmcv_utils`` the reference's file."""
    for name in ("_qd_ref", "_qd_ref.models", "_qd_ref.util"):
        mod = types.ModuleType(name)
        mod.__path__ = []
        sys.modules[name] = mod
    for name, rel in (("_qd_ref.util.mmcv_utils", "util/mmcv_utils.py"), ("_qd_ref.models.tracker", "models/tracker.py")):
        spec = importlib.util.spec_from_file_location(name, os.path.join(PKG, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
    return sys.modules["_qd_ref.models.tracker"].QuasiDenseEmbedTracker


def record(name, Tracker):
    seq = qc.golden_sequence(name)
    tracker = Tracker(**qc.SETTINGS[name])
    arrays = {"checksum": np.array(qc.checksum(seq)), "frames": np.array(len(seq))}
    for f, (boxes, scores, labels, embeds) in enumerate(seq):
        n = scores.shape[0]
        bboxes = torch.cat((boxes, scores[:, None]), 1)
        indices = [3 * r + 7 for r in range(n)]
        out_b, out_l, ids, out_idx = tracker.match(bboxes, labels, embeds, f, indices)
        rows = [int(torch.nonzero((bboxes == b).all(1))[0]) for b in out_b]
        arrays[f"{f}/rows"] = np.array(rows, np.int64)
        arrays[f"{f}/ids"] = ids.numpy().astype(np.int64)
        arrays[f"{f}/indices"] = np.array(out_idx, np.int64)
        tids = list(tracker.tracklets)
        arrays[f"{f}/track_ids"] = np.array(tids, np.int64)
        arrays[f"{f}/last_frame"] = np.array([tracker.tracklets[t]["last_frame"] for t in tids], np.int64)
        arrays[f"{f}/label"] = np.array([int(tracker.tracklets[t]["label"]) for t in tids], np.int64)
        arrays[f"{f}/embed"] = np.stack([tracker.tracklets[t]["embed"].numpy() for t in tids]) if tids else \
            np.zeros((0, embeds.shape[1]), np.float32)
        bl = [bd["labels"] for bd in tracker.backdrops]
        be = [bd["embeds"] for bd in tracker.backdrops]
        arrays[f"{f}/back_labels"] = torch.cat(bl).numpy().astype(np.int64) if bl else np.zeros(0, np.int64)
        arrays[f"{f}/back_embeds"] = torch.cat(be).numpy() if be else np.zeros((0, embeds.shape[1]), np.float32)
    return arrays


def main():
    Tracker = load_reference_tracker()
    os.makedirs(OUT, exist_ok=True)
    for name in qc.SETTINGS:
        path = os.path.join(OUT, f"{name}.npz")
        np.savez_compressed(path, **record(name, Tracker))
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
