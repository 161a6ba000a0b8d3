"""CUDA-graph capture of a fixed-shape callable (one `apply_model`, or a whole DDIM step).

One apply_model is ~1000 kernel launches issued through ctypes; at batch 4 the GPU finishes them faster than Python
can enqueue them, so the launch-bound inner loop is captured once and replayed (the graph also pins the TMA tensor
maps and tile schedules that the C ABI computed at capture time).
"""
import gc

import torch


class GraphedCallable:
    """`fn(*tensors) -> tensor | tuple[tensor]` with static shapes, replayed from a CUDA graph.

    Inputs are copied into static buffers before each replay; outputs are static buffers (clone them if they must
    survive the next call)."""

    def __init__(self, fn, example_inputs, warmup=2, adopt_inputs=False):
        self.fn = fn
        # adopt_inputs: the caller's tensors ARE the static buffers (it keeps them alive and refills them in place), so a
        # call with the same tensors copies nothing
        self.static_in = [(t if adopt_inputs else t.clone()) if torch.is_tensor(t) else t for t in example_inputs]
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):  # builds weight caches, sets kernel attributes, warms the allocator
            for _ in range(warmup):
                fn(*self.static_in)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        # A dropped graph that is cyclic garbage (a callable closing over the graph's owner), collected in the middle of
        # this capture, is destroyed by an illegal call while capturing and invalidates the capture; so collect now,
        # and not during the capture.
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.static_out = fn(*self.static_in)
        finally:
            if gc_was_enabled:
                gc.enable()

    def __call__(self, *inputs):
        for s, i in zip(self.static_in, inputs):
            if torch.is_tensor(s) and s.data_ptr() != i.data_ptr():
                s.copy_(i, non_blocking=True)
        self.graph.replay()
        return self.static_out
