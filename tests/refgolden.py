"""Stored results of the reference's own Python classes and functions (tests/golden/reference/*.npz), so that the tests
comparing this repo with the reference need no reference checkout.  ``python tests/golden/make_reference_golden.py``
regenerates them where a checkout exists: it runs the reference classes on the CPU, on the reference's own CPU function
``ms_deform_attn_core_pytorch``, with the inputs and weights the tests build from fixed seeds.

Large tensors are stored as a sample of their elements -- the flat indices are stored next to the values -- together with
their max-abs scale, so that a comparison against a sample keeps the test's scale-relative tolerance.
"""
import os
import zlib

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
SAMPLE = 1024
RECORDING = os.environ.get("MSDA_RECORD_REFERENCE") == "1"      # set by make_reference_golden.py only
_pending = {}


def _index(key, n):
    """Recording: the elements to store (None = all of them)."""
    if n <= SAMPLE:
        return None
    g = torch.Generator().manual_seed(zlib.crc32(key.encode()))
    return torch.randperm(n, generator=g)[:SAMPLE].sort().values


def _stored(golden, key, n):
    """The flat indices stored for `key` (None = the whole tensor was stored)."""
    if key + ".index" not in golden:
        assert golden[key].size == n, (key, n)
        return None
    idx = torch.from_numpy(golden[key + ".index"])
    assert idx.numel() == golden[key].size and int(idx.max()) < n, key
    return idx


def _flat(t):
    return t.detach().reshape(-1).double().cpu()


def put(group, key, t):
    """Recording: remember tensor `t` (reference result) under group/key."""
    f = _flat(t)
    idx = _index(f"{group}/{key}", f.numel())
    _pending.setdefault(group, {})[key] = (f if idx is None else f[idx]).numpy()
    if idx is not None:
        _pending[group][key + ".index"] = idx.numpy().astype(np.int64)
    _pending[group][key + ".scale"] = np.array([f.abs().max().item() if f.numel() else 0.0])
    _pending[group][key + ".shape"] = np.array(tuple(t.shape), dtype=np.int64)


def put_raw(group, key, arr):
    """Recording: store a small array as it is (names, shapes)."""
    _pending.setdefault(group, {})[key] = np.asarray(arr)


def flush(group):
    d = _pending.pop(group, {})
    np.savez_compressed(os.path.join(GOLDEN, f"{group}.npz"), **d)


def load(group):
    with np.load(os.path.join(GOLDEN, f"{group}.npz")) as z:
        return {k: z[k] for k in z.files}


def rel(got, golden, key, group):
    """max |got - reference| over the stored elements / max |reference| over the whole tensor."""
    f = _flat(got)
    assert tuple(got.shape) == tuple(golden[key + ".shape"]), (key, tuple(got.shape))
    idx = _stored(golden, key, f.numel())
    g = f if idx is None else f[idx]
    return float(np.abs(g.numpy() - golden[key]).max(initial=0.0) / max(float(golden[key + ".scale"][0]), 1e-30))


def sample(got, golden, key, group):
    """The elements of `got` that were stored for `key` (float64 numpy), for exact / custom comparisons."""
    f = _flat(got)
    idx = _stored(golden, key, f.numel())
    return (f if idx is None else f[idx]).numpy()
