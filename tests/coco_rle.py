"""The COCO API's run-length encoding of a binary mask (maskApi.c: rleEncode, rleToString, rleFrString), restated in plain
Python for the tests; pycocotools itself is not needed.

    counts   scan the H x W mask column-major (k = X * H + Y); the run lengths, alternating and starting with a run of
             zeros (counts[0] = 0 when pixel 0 is set); they sum to H * W.
    string   x = counts[j] - counts[j - 2] for j > 2, else counts[j]; x as 5-bit groups, least significant first:
             c = x & 0x1f, x >>= 5 (arithmetic), continue while (c & 0x10 ? x != -1 : x != 0); 0x20 on every character
             but the value's last; + 48.

``counts_of`` / ``to_string`` / ``from_string`` follow those rules one value at a time; ``encode_np`` is the same
encoder vectorised with numpy, for masks with millions of runs."""
import numpy as np


def counts_of(mask):
    """mask [H, W] (nonzero = set) -> the COCO counts, a list of ints."""
    flat = (np.asarray(mask) != 0).T.reshape(-1)
    counts, run, prev = [], 0, False
    for bit in flat:
        if bit != prev:
            counts.append(run)
            run, prev = 0, bit
        run += 1
    counts.append(run)
    return counts


def to_string(counts):
    s = bytearray()
    for j, x in enumerate(counts):
        if j > 2:
            x -= counts[j - 2]
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            s.append(c + 48)
    return bytes(s)


def from_string(s):
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def counts_np(mask):
    """counts_of with numpy: the differences of 0, the boundaries (bit(k) != bit(k - 1), bit(-1) = 0) and H * W."""
    flat = (np.asarray(mask) != 0).T.reshape(-1).astype(np.int8)
    b = np.flatnonzero(np.diff(flat, prepend=np.int8(0)))
    return np.diff(np.concatenate(([0], b, [flat.size]))).astype(np.int64)


def string_np(counts):
    """to_string with numpy."""
    c = np.asarray(counts, dtype=np.int64)
    x = c.copy()
    x[3:] -= c[1:-2]
    chars = np.zeros((x.size, 7), np.uint8)
    keep = np.zeros((x.size, 7), bool)
    alive = np.ones(x.size, bool)
    for g in range(7):
        ch = x & 0x1f
        x = x >> 5
        more = np.where(ch & 0x10, x != -1, x != 0)
        chars[:, g] = (ch | np.where(more, 0x20, 0)) + 48
        keep[:, g] = alive
        alive &= more
    assert not alive.any(), "a count needs more than 7 characters"
    return chars[keep].tobytes()


def encode_np(mask):
    """What pycocotools.mask.encode returns for one [H, W] mask."""
    h, w = np.asarray(mask).shape
    return {"size": [h, w], "counts": string_np(counts_np(mask))}
