"""Capture the training step in a CUDA graph (DESIGN.md §9 item 3; recipe: INTEGRATION.md §4).

The rasterizer's forward normally reads the frame's instance count and longest tile list on the host: they size the binning
buffer and the per-tile sort.  With a ``BinningReserve`` it bins into capacities fixed ahead of the frame instead
(``GaussianRasterizer(settings, reserve)``), so a whole step -- forward, losses, ``backward()`` -- has no host read and can be
captured once and replayed:

    reserve = BinningReserve("cuda")
    steps = StepGraph(reserve)
    loss = steps.run(key, step, params)      # step(): forward, losses, loss.backward(); returns the loss

A frame larger than the reserve sets a bit in the reserve's device status instead of writing past its buffers; the step is
then discarded and run again eagerly with a grown reserve.
"""
from __future__ import annotations

from collections import OrderedDict

import torch

__all__ = ["BinningReserve", "StepGraph"]

INSTANCE_ROUND = 65536   # instance capacity granule
LIST_ROUND = 256         # longest-list capacity granule: the tile sort's shared-memory buffers grow in steps of 256 keys
HEADROOM = (5, 4)        # capacity = observed * 5 / 4, rounded up


def _round_up(n: int, granule: int) -> int:
    return -(-n // granule) * granule


class BinningReserve:
    """The binning capacities of the rasterizer's graph path, and its device status: int32 [4] = overflow bits (1: instances,
    2: longest list), the largest instance count and the longest tile list seen since the last ``clear()``, reserved.  The
    capacities only grow: to the observed counts * 5/4, instances rounded up to 65 536 and the list length to 256."""

    def __init__(self, device, instances: int = 0, longest_list: int = 0):
        self.device = torch.device(device)
        self.instances, self.longest_list = 0, 0
        self.fit(instances, longest_list)
        self.status = torch.zeros(4, dtype=torch.int32, device=self.device)

    def fit(self, instances: int, longest_list: int) -> bool:
        """Grow the capacities to hold `instances` and `longest_list` with headroom; True when they grew."""
        if instances < 0 or longest_list < 0:
            raise ValueError("instance counts and list lengths are non-negative")
        num, den = HEADROOM
        grown = (max(self.instances, _round_up(-(-instances * num // den), INSTANCE_ROUND)),
                 max(self.longest_list, _round_up(-(-longest_list * num // den), LIST_ROUND)))
        changed = grown != (self.instances, self.longest_list)
        self.instances, self.longest_list = grown
        return changed

    def clear(self) -> None:
        """Zero the status (stream-ordered; captured when called under capture)."""
        self.status.zero_()

    def read(self) -> tuple[int, int, int]:
        """(overflow bits, largest instance count, longest tile list) since the last clear.  Synchronizes."""
        bits, instances, longest = (v & 0xFFFFFFFF for v in self.status[:3].tolist())
        return bits, instances, longest

    def overflowed(self) -> bool:
        """The status's one host read (synchronizes): True when a frame since the last clear did not fit; the capacities are
        then grown to fit what was seen."""
        bits, instances, longest = self.read()
        if bits:
            self.fit(instances, longest)
        return bits != 0


def _zero_grads(params) -> None:
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        else:
            p.grad.zero_()


class _Captured:
    def __init__(self, graph: torch.cuda.CUDAGraph, out):
        self.graph, self.out = graph, out

    def replay(self):
        self.graph.replay()
        return self.out


class StepGraph:
    """Replay of a training step captured per key, at most `max_graphs` graphs (least recently used dropped).

    ``run(key, fn, params)``: `fn()` runs the step (forward, losses, ``backward()``) and returns its outputs; `params` are the
    tensors whose ``.grad`` the step fills.  `key` must hold everything the captured graph bakes in: every Python scalar the step
    passes (image size, tan-FoV, SH degree, kernel size, require flags, P) and the data pointers of every tensor it reads.  A new
    key warms the step up eagerly on a side stream (which also fits the reserve), captures it and replays it; a known key replays.
    The graph clears the reserve's status and zeroes the ``.grad`` tensors in place at its start, so the gradients are the step's
    own and the ``.grad`` tensors stay the graph's static tensors: do not set them to None between replays.  Returns the outputs
    of the capture, overwritten by the next replay of the same key.

    After each replay the reserve's status is read once.  When a frame did not fit, the reserve grows, every graph is dropped
    (they were sized by the old capacities), the ``.grad`` tensors are zeroed and `fn` runs eagerly; its outputs are returned and
    the key is captured again on its next run."""

    def __init__(self, reserve: BinningReserve, max_graphs: int = 4):
        if max_graphs < 1:
            raise ValueError("max_graphs must be at least 1")
        self.reserve, self.max_graphs = reserve, max_graphs
        self._graphs: OrderedDict = OrderedDict()
        self.captures = 0
        self.fallbacks = 0

    def __len__(self) -> int:
        return len(self._graphs)

    def __contains__(self, key) -> bool:
        return key in self._graphs

    def run(self, key, fn, params):
        params = list(params)
        g = self._graphs.get(key)
        if g is None:
            while len(self._graphs) >= self.max_graphs:
                self._graphs.popitem(last=False)
            g = self._capture(fn, params)
            self._graphs[key] = g
            self.captures += 1
        else:
            self._graphs.move_to_end(key)
        out = g.replay()
        if not self.reserve.overflowed():
            return out
        self._graphs.clear()
        self.fallbacks += 1
        _zero_grads(params)
        return fn()

    def _capture(self, fn, params) -> _Captured:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            _zero_grads(params)
            fn()   # warm-up: one-time set-up of every kernel the step launches, and the reserve fitted to this frame
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self.reserve.clear()
            _zero_grads(params)
            out = fn()
        return _Captured(graph, out)
