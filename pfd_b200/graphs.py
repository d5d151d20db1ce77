"""CUDA-graph caching for fixed-shape pieces of the pipeline (SeeCoder encode, VAE decode, the
sampling loops of loop.py).  The pipeline launches ~600 kernels per UNet evaluation and ~1100 per
SeeCoder encode; replaying captured graphs removes the Python / ctypes / tensor-map-encode cost from
the request path.  Graphs are keyed on input shapes and on a signature of the weights they baked in
(storage pointer + version of every parameter), so load_state_dict / .half() / .to() invalidate them.
"""
from __future__ import annotations

import gc
from typing import Callable, Dict, Hashable, List, Sequence, Tuple

import torch
import torch.nn as nn

from . import native as nv


class CapturedGraph:
    """fn() captured into a CUDA graph, with the library kernels it launched counted so that every replay adds them
    to nv.launch_count().  replay() returns fn's output of the capture, which each replay rewrites in place.
    The Python garbage collector is held off during the capture: a cyclic-garbage sweep in the middle of a capture may
    run the destructor of an older CUDAGraph (cudaGraphExecDestroy), which is illegal while a stream is capturing in
    the global capture mode and invalidates the capture."""

    def __init__(self, fn: Callable):
        self.graph = torch.cuda.CUDAGraph()
        gc.collect()
        was = gc.isenabled()
        gc.disable()
        n0 = nv.launch_count()
        try:
            with torch.cuda.graph(self.graph):
                self.out = fn()
        finally:
            if was:
                gc.enable()
        self.n_kernels = nv.launch_count() - n0

    def replay(self):
        self.graph.replay()
        nv.note_replay(self.n_kernels)
        return self.out


_generation = 0


def _bump_generation(*_a, **_k) -> None:
    global _generation
    _generation += 1


def watch(module: nn.Module) -> None:
    """Make `load_state_dict` on `module` (or any of its sub-modules) bump the process-wide weight generation,
    which is folded into every graph / packed-weight signature: (data_ptr, _version) pairs alone can collide when
    a module is rebuilt and the caching allocator hands out the same addresses (r1 advisor finding)."""
    for m in module.modules():
        if "_pfd_watched" not in m.__dict__:
            m.__dict__["_pfd_watched"] = True
            m.register_load_state_dict_post_hook(_bump_generation)


def generation() -> int:
    return _generation


def invalidate(module: nn.Module = None) -> None:
    """Explicitly drop every packed-weight cache under `module` and force graph re-capture — for callers that
    modify weights behind autograd's version counter (e.g. `p.data.copy_(...)`)."""
    _bump_generation()
    if module is not None:
        for m in module.modules():
            m.__dict__.pop("_pfd_pk", None)


def weights_signature(*modules: nn.Module) -> Tuple:
    sig = [_generation]
    for m in modules:
        if m is None:
            continue
        watch(m)
        for p in m.parameters():
            sig.append((p.data_ptr(), p._version))
        for b in m.buffers():
            sig.append((b.data_ptr(), b._version))
    return tuple(sig)


class GraphedFunction:
    """fn(*static_inputs) -> tensor | tuple of tensors, captured once and replayed with new input
    values copied into the static input buffers."""

    def __init__(self, fn: Callable, example_inputs: Sequence[torch.Tensor]):
        self.static_in: List[torch.Tensor] = [t.clone() for t in example_inputs]
        # eager warm-up builds every lazily packed weight / mask so capture sees only kernel launches
        self.first_out = fn(*self.static_in)
        torch.cuda.synchronize()
        self.graph = CapturedGraph(lambda: fn(*self.static_in))

    def __call__(self, *inputs: torch.Tensor):
        for s, t in zip(self.static_in, inputs):
            s.copy_(t, non_blocking=True)
        return self.graph.replay()


class GraphCache:
    def __init__(self, max_entries: int = 4):
        self.entries: Dict[Hashable, GraphedFunction] = {}
        self.max_entries = max_entries

    def get(self, key: Hashable, build: Callable[[], GraphedFunction]) -> Tuple[GraphedFunction, bool]:
        hit = key in self.entries
        if not hit:
            if len(self.entries) >= self.max_entries:
                self.entries.pop(next(iter(self.entries)))
            self.entries[key] = build()
        return self.entries[key], hit

    def clear(self):
        self.entries.clear()
