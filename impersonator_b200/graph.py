"""CUDA-graph replay of a fixed launch sequence (``LWB_GRAPH``).

One step of the hot path is ~90-170 kernel launches issued from Python through ctypes; at ~15-25 us of interpreter time per
launch the host becomes the bottleneck once the GPU side drops below ~4 ms (and immediately with ``LWB_STREAMS`` > 1).
``CapturedStep`` records the launches of a callable once -- every buffer is persistent (conv plans, activation buffers) or
allocated from the graph's private pool (outputs), inputs are copied into static tensors -- and replays them with one
``cudaGraphLaunch`` per step.  Programmatic dependent launches and the side-stream fork /
join of ``LWB_STREAMS`` are all captured as graph nodes / edges.  PyTorch supplies the capture plumbing
(``torch.cuda.CUDAGraph``); the graph contains this library's kernels plus a few copy / fill nodes.
"""
import os
import warnings

import torch

from . import kernels as K
from ._lib import _OPEN, pin  # noqa: F401 -- pin lives beside the library binding, which kernels' caches import too


def graphs_enabled():
    """LWB_GRAPH (default 1): replay the per-chunk launch sequence as a CUDA graph where the caller supports it."""
    return os.environ.get("LWB_GRAPH", "1") != "0"


class CapturedStep(object):
    """``step = CapturedStep(fn, example_inputs)``; ``outputs = step(**inputs)``.

    ``fn(**static_inputs)`` must launch only on torch's current stream (and streams forked from / joined to it), must not
    synchronise, and must return a tensor / tuple / dict of tensors (None allowed).  It is run ``warmup`` times eagerly first
    (lazy plan / stream construction, function-attribute set-up), then captured.  The returned outputs are STATIC tensors
    that the next call overwrites: consume (or copy) them before calling again.  If capture fails the object falls back to
    calling ``fn`` eagerly (with a warning) -- same results, only slower.
    """

    def __init__(self, fn, example_inputs, warmup=2):
        self.fn = fn
        self.static_in = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in example_inputs.items()}
        self.graph = None
        self.static_out = None
        self.launches = 0
        self.pinned = []                                         # stream objects (buffers, plans) the graph replays into
        _OPEN.append(self.pinned)
        try:
            self._build(fn, warmup)
        finally:
            _OPEN.pop()
        self.pinned[:] = list({id(o): o for o in self.pinned}.values())

    def _build(self, fn, warmup):
        dev = next(v.device for v in self.static_in.values() if torch.is_tensor(v))
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                fn(**self.static_in)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        try:
            g = torch.cuda.CUDAGraph()
            n0 = K.launch_count()
            # thread_local: other threads of the process (e.g. the NCCL watchdog of a torchrun job) may call the CUDA API
            # while this thread captures
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                out = fn(**self.static_in)
            self.launches = K.launch_count() - n0
            self.graph, self.static_out = g, out
        except Exception as e:                                   # noqa: BLE001 -- any capture failure means "run eagerly"
            torch.cuda.synchronize(dev)
            warnings.warn("lwb_b200: CUDA graph capture failed (%s: %s); running the step eagerly" % (type(e).__name__, e))
            self.graph = None

    @property
    def captured(self):
        return self.graph is not None

    def __call__(self, **inputs):
        if self.graph is None:
            return self.fn(**inputs)
        for k, v in inputs.items():
            dst = self.static_in[k]
            if torch.is_tensor(dst):
                if v.data_ptr() != dst.data_ptr():
                    dst.copy_(v, non_blocking=True)
            elif v != dst:
                raise ValueError("CapturedStep: non-tensor argument %r changed (%r -> %r)" % (k, dst, v))
        self.graph.replay()
        K._count(self.launches)                                  # the replay launches the captured kernels again
        return self.static_out
