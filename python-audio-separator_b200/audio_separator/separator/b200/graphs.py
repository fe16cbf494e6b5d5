"""CUDA-graph replay of a fixed launch list.

The network forwards of this package are launch sequences over the C ABI (several hundred kernels per HTDemucs / Roformer / TFC_TDF_net
forward, all on the caller's stream, no host synchronisation in between).  `GraphedForward` captures that sequence once per input shape
with stream capture and replays it with one cudaGraphLaunch: the ctypes / Python cost per kernel disappears, which matters when a rank
of a time-sharded run gets only a few segments per forward.

PyTorch is used for what it is here for -- device memory and streams: `torch.cuda.graph` provides the capture stream and a private
memory pool, so every intermediate tensor of the captured forward keeps its address for the lifetime of the graph.  The kernels in the
graph are libb200sep's own; nothing is traced or compiled.  A C host does the same with b200sep_capture_begin / _end / _graph_launch
(include/b200sep.h) around its own sequence of operator calls.
"""
from __future__ import annotations

import torch


class GraphedForward:
    """fn(x) -> tensor, captured per (shape, dtype) of x.  The returned tensor is the graph's static output buffer: consume (copy) it before the
    next call.  Inside a capture that is already running, fn runs directly and becomes part of the caller's graph."""

    def __init__(self, fn, warmup: int = 2, max_graphs: int = 8):
        self.fn, self.warmup, self.max_graphs = fn, warmup, max_graphs
        self.cache = {}

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if torch.cuda.is_current_stream_capturing():
            return self.fn(x)
        key = (tuple(x.shape), x.dtype, x.device.index)
        ent = self.cache.get(key)
        if ent is None:
            if len(self.cache) >= self.max_graphs:  # each graph pins its activations: bound the number of resident shapes
                self.cache.pop(next(iter(self.cache)))
            static_in = torch.empty_like(x).copy_(x)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):  # warm-up off the capture: weight packing, tensor maps, func attributes, scratch allocations happen here
                for _ in range(self.warmup):
                    self.fn(static_in)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            # thread-local capture mode: the NCCL watchdog / other threads of a multi-rank run may touch the CUDA API while this thread captures
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                static_out = self.fn(static_in)
            ent = (graph, static_in, static_out)
            self.cache[key] = ent
        graph, static_in, static_out = ent
        static_in.copy_(x)
        graph.replay()
        return static_out
