#!/usr/bin/env python
"""Regenerate tests/golden/tracker/*.npz: what the reference's own ``IDOL_Tracker`` (models/tracker.py of a reference
checkout, loaded in place with a stub for its unused ``..util.mmcv_utils`` import) returns and keeps on the CPU for the
seeded sequences of tests/tracker_case.py, one file per (long_match, frame_weight, temporal_weight) setting.  Per frame:
the kept rows, their ids and indices; the live tracklets' id, last_frame, exist_frame, embed and rings.  The tests do
not need the reference.

    python tests/golden/make_tracker_golden.py
"""
import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refpy import REFERENCE  # noqa: E402
from tests import tracker_case as tc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "tracker")
SOURCE = os.path.join(REFERENCE, "projects", "UNINEXT", "uninext", "models", "tracker.py")


def load_reference_tracker():
    """models/tracker.py as module ``_idol_ref.models.tracker``; its ``from ..util.mmcv_utils import bbox_overlaps``
    (used only by QuasiDenseEmbedTracker) resolves to a stub."""
    for name in ("_idol_ref", "_idol_ref.models", "_idol_ref.util"):
        mod = types.ModuleType(name)
        mod.__path__ = []
        sys.modules[name] = mod
    stub = types.ModuleType("_idol_ref.util.mmcv_utils")
    stub.bbox_overlaps = None
    sys.modules[stub.__name__] = stub
    spec = importlib.util.spec_from_file_location("_idol_ref.models.tracker", SOURCE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.IDOL_Tracker


def state_arrays(tracker, L, D):
    ids = sorted(tracker.tracklets)
    n = len(ids)
    last, exist, lens = (np.zeros(n, np.int64) for _ in range(3))
    embed, ring_e, ring_s = np.zeros((n, D), np.float32), np.zeros((n, L, D), np.float32), np.zeros((n, L), np.float32)
    for c, k in enumerate(ids):
        v = tracker.tracklets[k]
        last[c], exist[c], lens[c] = v["last_frame"], v["exist_frame"], len(v["long_embed"])
        embed[c] = v["embed"].numpy()
        ring_e[c, :lens[c]] = torch.stack(v["long_embed"]).numpy()
        ring_s[c, :lens[c]] = torch.stack(v["long_score"]).numpy()
    return dict(track_ids=np.array(ids, np.int64), last_frame=last, exist_frame=exist, ring_len=lens, embed=embed,
                long_embed=ring_e, long_score=ring_s)


def record(flag_index, IDOL_Tracker):
    flags = tc.FLAG_SETS[flag_index]
    seq = tc.golden_sequence(flag_index)
    cfg = tc.settings(flags)
    tracker = IDOL_Tracker(**cfg)
    arrays = {"checksum": np.array(tc.checksum(seq)), "flags": np.array(flags)}
    for f, (scores, masks, embeds) in enumerate(seq):
        n = scores.shape[0]
        bboxes = torch.cat((torch.rand(n, 4, generator=torch.Generator().manual_seed(f)), scores[:, None]), 1)
        labels = torch.zeros(n, dtype=torch.long)
        indices = [3 * r + 7 for r in range(n)]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out_b, _, ids, out_idx = tracker.match(bboxes, labels, masks, embeds, f, indices)
        keep = [int(torch.nonzero((bboxes == b).all(1))[0]) for b in out_b]
        arrays[f"{f}/keep"] = np.array(keep, np.int64)
        arrays[f"{f}/ids"] = ids.numpy().astype(np.int64)
        arrays[f"{f}/indices"] = np.array(out_idx, np.int64)
        for k, v in state_arrays(tracker, cfg["memory_len"], embeds.shape[1]).items():
            arrays[f"{f}/{k}"] = v
    arrays["frames"] = np.array(len(seq))
    return arrays


def main():
    IDOL_Tracker = load_reference_tracker()
    os.makedirs(OUT, exist_ok=True)
    for i, flags in enumerate(tc.FLAG_SETS):
        name = "lm{}_fw{}_tw{}".format(*(int(x) for x in flags))
        path = os.path.join(OUT, f"{name}.npz")
        np.savez_compressed(path, **record(i, IDOL_Tracker))
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
