"""CUDA-graph replay of the fixed-shape encoder forwards.

One filter() is ~450 kernel launches of 5-50 us each; issued one by one from Python the launch gaps cost several
milliseconds per image, and NormalNet runs 100 times per image in the reference's SMPL-fitting loop
(apps/infer.py:168-210).  `GraphedForward` runs a module's tensor -> tensor(s) function eagerly the first time a
(shape, weights) combination is seen (which also fills the packed-weight caches), captures it into a
`torch.cuda.CUDAGraph` the second time and replays it afterwards.  Inputs are copied into the graph's static input
buffer and results are returned as fresh clones, so callers see ordinary tensors.

The key carries the identity and version of every parameter / buffer of the module: loading a checkpoint or moving
the module invalidates the captured graphs (they hold the old packed-weight pointers).
"""
import os

import torch

_ENABLED = os.environ.get("ICON_B200_CUDA_GRAPHS", "1") != "0"
MAX_GRAPHS_PER_MODULE = 4


_CONCURRENT = os.environ.get("ICON_B200_CONCURRENT", "1") != "0"
_SIDE = {}
_SLOT = [0]           # which of the two concurrent chains is being enqueued: a module called on both (HGFilter on the front
                      # and the back map) needs one captured graph (= one set of static buffers) per chain


def concurrent(flag=None):
    """Run independent encoder forwards of one call (NormalNet's two generators, HGFilter on the front / back normal
    maps) on two CUDA streams.  Each is a chain of several hundred short kernels, most of them smaller than the GPU:
    side by side they fill SMs the other leaves idle.  Environment ICON_B200_CONCURRENT=0 disables."""
    global _CONCURRENT
    if flag is not None:
        _CONCURRENT = bool(flag)
    return _CONCURRENT


def run_pair(fn_a, fn_b):
    """(fn_a(), fn_b()) -- fn_b on a side stream forked from the current one and joined afterwards, when concurrency
    is on.  Works eagerly and INSIDE a CUDA-graph capture (the fork / join become graph edges, so a replay runs the two
    branches side by side).  Nesting is fine: every stream has its own side stream.  Discipline that keeps the caching
    allocator safe without record_stream during capture: a side stream always first waits for its parent, and the
    parent always joins it before using the results."""
    if not (_CONCURRENT and torch.cuda.is_available()):
        return fn_a(), fn_b()
    cur = torch.cuda.current_stream()
    capturing = torch.cuda.is_current_stream_capturing()
    key = (cur.device_index, cur.cuda_stream)
    side = _SIDE.get(key)
    if side is None:
        side = _SIDE[key] = torch.cuda.Stream(device=cur.device_index)
    side.wait_stream(cur)
    prev, _SLOT[0] = _SLOT[0], 1
    try:
        with torch.cuda.stream(side):
            b = fn_b()
    finally:
        _SLOT[0] = prev
    a = fn_a()
    cur.wait_stream(side)

    def mark(t):
        if isinstance(t, torch.Tensor) and t.is_cuda:
            t.record_stream(cur)
        elif isinstance(t, (list, tuple)):
            for u in t:
                mark(u)
        elif hasattr(t, "__dict__"):                     # nhwc.Raw / Operand: tensors in attributes
            for u in vars(t).values():
                if isinstance(u, torch.Tensor) and u.is_cuda:
                    u.record_stream(cur)
    if not capturing:
        mark(b)
    return a, b


def enable(flag=True):
    """Process-wide switch (also: environment ICON_B200_CUDA_GRAPHS=0)."""
    global _ENABLED
    _ENABLED = bool(flag)


def enabled():
    return _ENABLED


class GraphedForward:
    def __init__(self, module, method):
        self.module, self.method = module, method
        self.entries = {}            # key -> None (seen once, eager) | (graph, static_in, static_out)
        self.disabled = False
        self.replays = 0

    def fn(self, x):
        return getattr(self.module, self.method)(x)

    def __deepcopy__(self, memo):     # graphs are not copied: the copy captures its own
        import copy
        return GraphedForward(copy.deepcopy(self.module, memo), self.method)

    def _key(self, x):
        m = self.module
        weights = tuple((t.data_ptr(), t._version) for t in list(m.parameters()) + list(m.buffers()))
        return (tuple(x.shape), x.dtype, str(x.device), _SLOT[0], weights)

    def __call__(self, x):
        usable = (_ENABLED and not self.disabled and x.is_cuda and not self.module.training
                  and not torch.cuda.is_current_stream_capturing())
        if not usable:
            return self.fn(x)
        key = self._key(x)
        if key not in self.entries:
            if len(self.entries) >= MAX_GRAPHS_PER_MODULE:
                self.entries.clear()
            self.entries[key] = None
            return self.fn(x)                                   # first sight: eager (fills the weight-pack caches)
        ent = self.entries[key]
        if ent is None:
            try:
                static_in = x.detach().clone()
                torch.cuda.current_stream().synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_out = self.fn(static_in)
                ent = self.entries[key] = (graph, static_in, static_out)
            except Exception:                                   # capture not possible here: stay eager from now on
                self.disabled = True
                self.entries.clear()
                return self.fn(x)
        graph, static_in, static_out = ent
        static_in.copy_(x)
        graph.replay()
        self.replays += 1
        if isinstance(static_out, (list, tuple)):
            return type(static_out)(t.clone() for t in static_out)
        return static_out.clone()
