"""CUDA-graph capture of the layers' steady state (DESIGN section 8).

A layer step on a graph that has already run once eagerly enqueues only stream work, so it can be captured with
``torch.cuda.graph`` or ``torch.cuda.make_graphed_callables`` and replayed.  This module holds the three rules that make
that safe, and is the one place that asks whether the current stream is capturing:

* **guard** -- work that synchronises or builds per-graph state (a CSR, a light view, a dense batch's graphs, a
  readout's graph count) raises :class:`CaptureError` inside a capture, before it enqueues anything;
* **cache bypass** -- weight packs cached on parameter versions are rebuilt on every call while capturing (the packing
  kernels become part of the graph, so a replay follows the weights through optimizer steps) and the cache is neither
  read nor written;
* **pinning** -- every per-graph object a captured call touches (CSRs with their scratch and transposed CSRs, dense
  graphs, row scales, work buffers) is recorded by the active :func:`pinned` handle, so evicting it from a cache can never
  free memory a captured graph still reads.

Usage::

    with pna_b200.capture.pinned() as keep, torch.cuda.graph(g):
        out = model(x, edge_index)
    # keep `keep` as long as `g`
"""
from __future__ import annotations

import contextlib

import torch

__all__ = ["CaptureError", "Pinned", "capturing", "guard", "pin", "pinned"]


class CaptureError(RuntimeError):
    """A call inside a CUDA graph capture needed work that cannot be captured (a synchronisation, or building per-graph
    state).  Raised before anything was enqueued: the capture is left as it was."""


def capturing() -> bool:
    """Is the current CUDA stream capturing a graph?  (No CUDA context yet: nothing can be capturing.)"""
    return torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()


def guard(what: str, hint: str = "run one eager step on this graph first") -> None:
    """CaptureError naming ``what`` when called inside a capture; nothing outside one."""
    if capturing():
        raise CaptureError(f"{what} cannot run inside a CUDA graph capture: {hint}")


class Pinned:
    """The per-graph objects a capture touched.  Keep it alive as long as the captured graph."""

    def __init__(self):
        self.objects: list = []
        self._ids: set = set()

    def add(self, obj) -> None:
        if obj is not None and id(obj) not in self._ids:
            self._ids.add(id(obj))
            self.objects.append(obj)


_ACTIVE: list = []


@contextlib.contextmanager
def pinned():
    """Record, while capturing, every per-graph object the captured calls touch; yields the :class:`Pinned` handle."""
    handle = Pinned()
    _ACTIVE.append(handle)
    try:
        yield handle
    finally:
        _ACTIVE.remove(handle)


def pin(*objects) -> None:
    """Record ``objects`` in every active :func:`pinned` handle when the current stream is capturing."""
    if _ACTIVE and capturing():
        for h in _ACTIVE:
            for o in objects:
                h.add(o)
