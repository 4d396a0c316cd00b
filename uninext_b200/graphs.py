"""CUDA-graph capture of a whole training / inference step around the op.

The deformable transformer step issues ~1000 kernels in eager mode, so host launch time matters (README.md: TF32 eager
against CUDA graph frames/s at cfg2).  The op and every caller kernel of this library are capture-safe: they launch on
the caller's current stream, never synchronise, never read ``spatial_shapes`` on the host (the level table stays on the
device; ``MSDeformAttn`` validates it once per distinct table, so warm-up iterations do the one host read before capture)
and allocate only through PyTorch's caching allocator, which CUDA graphs support via a private pool.

    step = GraphedStep(lambda: model(src, pos, shapes, ss, lsi).square().mean().backward())
    for _ in range(n):
        bucket.zero_()        # static buffers: gradients live in the same storage every replay
        step.replay()
        bucket.all_reduce_mean()          # collectives stay outside the graph

Static-shape, static-address contract (the usual CUDA-graph one): the callable must read its inputs from tensors that are
updated IN PLACE between replays and must not create new parameters / change shapes.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch


class GraphedStep:
    def __init__(self, fn: Callable[[], object], warmup: int = 3, device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("GraphedStep needs a CUDA device")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.fn = fn
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):                     # warm-up off the capture: lazy inits, the level-table check, cuBLAS plans
            for _ in range(max(1, warmup)):
                fn()
        torch.cuda.current_stream(self.device).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.result = fn()

    def replay(self):
        self.graph.replay()
        return self.result
