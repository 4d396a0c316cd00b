#!/usr/bin/env python
"""How often do backward row-adds hit the same grad_value row?  cfg2 encoder workload, CPU only (numpy):
per warp step of the tiled kernel (4 neighbouring queries x 1 tap x 4 corners) and per 8x8-patch tile of one head.
    python tools/row_duplicates.py [jitter_px ...]        # default: 2.0 = the bench workload (SURVEY.md 8d); e.g. 0 0.25 0.5 1 2
The Gaussian jitter on the module's ring offsets is the workload's only free parameter; it decides how much neighbouring
queries' taps overlap, i.e. what any combine-before-red scheme could save."""
import os
import sys

import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uninext_b200.workloads import CONFIGS, make_inputs
cfg = CONFIGS['cfg2']
import dataclasses
cfg1 = dataclasses.replace(cfg, batch=1)
JITTERS = [float(a) for a in sys.argv[1:]] or [2.0]
loc = None                                      # [S, M, L, P, 2], set per jitter below
shapes = cfg.shapes
S = cfg.S
starts = np.cumsum([0]+[h*w for h,w in shapes])
def rows_of(q_idx, m):
    """global row ids [len(q), L, P, 4] (-1 = outside)"""
    out = np.full((len(q_idx), 4, 4, 4), -1, dtype=np.int64)
    for l,(H,W) in enumerate(shapes):
        x = loc[q_idx, m, l, :, 0]*W - 0.5; y = loc[q_idx, m, l, :, 1]*H - 0.5
        x0 = np.floor(x).astype(int); y0 = np.floor(y).astype(int)
        inside = (y > -1) & (x > -1) & (y < H) & (x < W)
        for c,(dy,dx) in enumerate(((0,0),(0,1),(1,0),(1,1))):
            yy, xx = y0+dy, x0+dx
            ok = inside & (yy>=0)&(yy<H)&(xx>=0)&(xx<W)
            out[:, l, :, c] = np.where(ok, starts[l] + yy*W + xx, -1)
    return out
def measure():
    rng = np.random.default_rng(0)
    for ql,(H,W) in enumerate(shapes):
        tot_step = uniq_step = tot_tile = uniq_tile = 0
        for _ in range(40):
            py = rng.integers(0, max(1,H//8))*8; px = rng.integers(0, max(1,W//8))*8; m = rng.integers(0,8)
            ys, xs = np.meshgrid(np.arange(py, min(py+8,H)), np.arange(px, min(px+8,W)), indexing='ij')
            q = (starts[ql] + ys*W + xs)            # [8, 8]
            r = rows_of(q.reshape(-1), m).reshape(q.shape[0], q.shape[1], 4, 4, 4)      # [y, x, L, P, corner]
            # warp step: 4 neighbours in x, one (l,p), 4 corners
            for yy in range(r.shape[0]):
                for x4 in range(0, r.shape[1], 4):
                    blk = r[yy, x4:x4+4]          # [4, L, P, 4]
                    for l in range(4):
                        for p in range(4):
                            v = blk[:, l, p, :].reshape(-1); v = v[v>=0]
                            tot_step += len(v); uniq_step += len(np.unique(v))
            v = r.reshape(-1); v = v[v>=0]
            tot_tile += len(v); uniq_tile += len(np.unique(v))
        print(f"query level {ql} ({H}x{W}): unique/total row-adds per warp step (4 neighbours x 1 tap x 4 corners) {uniq_step/tot_step:.3f}; per 8x8-patch tile (64 pairs x 16 taps x 4 corners) {uniq_tile/tot_tile:.3f}")

    # the 16 corner rows of ONE (query, head, level): could a lane group combine its own taps in registers before issuing?
    tot = uniq = 0
    for _ in range(2000):
        q = rng.integers(0, S); m = rng.integers(0, 8)
        r = rows_of(np.array([q]), m)[0]                  # [L, P, corner]
        for l in range(4):
            v = r[l].reshape(-1); v = v[v >= 0]
            tot += len(v); uniq += len(np.unique(v))
    print(f"one (query, head, level), 4 taps x 4 corners: unique/total {uniq / tot:.3f}")


def region_estimate(loc0, settings=((8, 2), (8, 3), (8, 4), (8, 6), (12, 4), (16, 4))):
    """Region tiles of msda_bwd_region (msda_region.cuh), same geometry: tile = (head, R x R region of the finest level),
    query (x, y) of level l in region floor((x + 0.5) * Wref / W_l / R); window on level l = the region scaled to level l
    plus `halo` pixels.  Per (R, halo): tiles, max queries per tile, max in-window corner entries per tile, and the
    row-reds left (corners outside the window + touched window rows per tile) over today's one red per live corner.
    Ignores the kernel's capacities (stash, entry list, window rows): corners past them red directly."""
    H = np.array([h for h, _ in shapes]); W = np.array([w for _, w in shapes])
    Href, Wref = H.max(), W.max()
    ql = np.repeat(np.arange(len(shapes)), H * W)                     # level / pixel of every query
    qk = np.arange(S) - starts[ql]
    qy, qx = qk // W[ql], qk % W[ql]
    for R, halo in settings:
        nry, nrx = -(-Href // R), -(-Wref // R)
        ry = (2 * qy + 1) * Href // (2 * H[ql] * R)
        rx = (2 * qx + 1) * Wref // (2 * W[ql] * R)
        reg = ry * nrx + rx
        nq = np.bincount(reg, minlength=nry * nrx)
        total = outside = touched = 0
        max_entries = 0
        for m in range(loc0.shape[1]):
            keys, n_in = [], np.zeros(nry * nrx, dtype=np.int64)
            for l, (Hl, Wl) in enumerate(shapes):
                x = loc0[:, m, l, :, 0] * Wl - 0.5; y = loc0[:, m, l, :, 1] * Hl - 0.5      # [S, P]
                inside = (y > -1) & (x > -1) & (y < Hl) & (x < Wl)
                y0 = np.floor(y).astype(np.int64); x0 = np.floor(x).astype(np.int64)
                wy0 = np.maximum(0, ry * R * Hl // Href - halo)[:, None]
                wy1 = np.minimum(Hl, -(-(ry + 1) * R * Hl // Href) + halo)[:, None]
                wx0 = np.maximum(0, rx * R * Wl // Wref - halo)[:, None]
                wx1 = np.minimum(Wl, -(-(rx + 1) * R * Wl // Wref) + halo)[:, None]
                for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
                    yy, xx = y0 + dy, x0 + dx
                    live = inside & (yy >= 0) & (yy < Hl) & (xx >= 0) & (xx < Wl)
                    inw = live & (yy >= wy0) & (yy < wy1) & (xx >= wx0) & (xx < wx1)
                    total += live.sum(); outside += (live & ~inw).sum()
                    r = np.broadcast_to(reg[:, None], inw.shape)[inw]
                    n_in += np.bincount(r, minlength=nry * nrx)
                    keys.append(r * S + starts[l] + yy[inw] * Wl + xx[inw])
            touched += len(np.unique(np.concatenate(keys)))
            max_entries = max(max_entries, int(n_in.max()))
        print(f"R={R:2d} halo={halo}: tiles per batch element {nry * nrx} x M, max queries / tile {nq.max()}, "
              f"max in-window entries / tile {max_entries} ({max_entries * 8 / 1024:.0f} KB), "
              f"row-reds left / today {(outside + touched) / total:.3f} (outside-window {outside / total:.3f})")


for jit in JITTERS:
    loc = make_inputs(cfg1, 'enc', 'cpu', jitter_px=jit)['sampling_locations'][0].numpy()
    print(f"--- jitter {jit} px ---")
    measure()
    if jit == 2.0:         # the bench's first encoder input: make_inputs(cfg2, "enc", seed=1000), batch element 0
        print("region tiles, cfg2 seed 1000, batch element 0, all heads:")
        region_estimate(make_inputs(cfg, 'enc', 'cpu', seed=1000)['sampling_locations'][0].numpy())
