"""One training step of the plugin contract -- ``zero_grad``, ``forward(feed_dict)``, ``loss``, ``backward``,
``optimizer.step()``: the loop body of helpers/BaseRunner.py:193-206 -- captured ONCE in a CUDA graph and replayed per
batch.  The step of the dense models is ~70 (NeuMF) to ~150 (SASRec) small launches from Python; as a graph the host
pays one launch and the GPU sees them back to back.

What makes the capture legal: every kernel of this package is enqueued on ``torch.cuda.current_stream()`` without host
synchronisation, scratch memory comes from torch's caching allocator (graph-private pool during capture), and the
optimizer's per-step scalars (Adam's bias corrections) live on the device (``RowSparseOptimizer(device_clock=True)``,
``b2r_optim_tick``) instead of in kernel parameters.  Batches are copied into static device buffers before each replay
(or, with ``replay()``, written there by the caller's own device collate); shapes are fixed at capture time (a ragged last
batch goes through the eager path).

One precondition comes from autograd, not from this package: a parameter's AccumulateGrad node is bound to the stream
that was current when the node was created and lives as long as any autograd graph that reaches it.  If the caller still
holds the (non-detached) loss of an eager step that ran on the legacy default stream, the capture's backward would make
the legacy stream wait on the capturing stream (cudaErrorStreamCaptureImplicit).  Drop or ``detach()`` such losses before
building a GraphedStep; the constructor turns that CUDA error into a message that says so.
"""
from __future__ import annotations

from typing import Dict

import torch

from .optim import RowSparseOptimizer


class GraphedStep:
    def __init__(self, model: torch.nn.Module, example_feed: Dict, warmup: int = 2):
        opt = model.optimizer
        if not isinstance(opt, RowSparseOptimizer) or not opt._want_clock:
            raise ValueError("GraphedStep needs model.optimizer = RowSparseOptimizer(..., device_clock=True)")
        self.model, self.opt = model, opt
        self.static = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in example_feed.items()}
        self.shapes = {k: tuple(v.shape) for k, v in self.static.items() if isinstance(v, torch.Tensor)}
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        self.warmup_losses = []
        with torch.cuda.stream(side):               # eager warm-up steps (real steps: they train) off the default stream
            for _ in range(max(1, warmup)):
                self.warmup_losses.append(self._step().clone())
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(self.graph, capture_error_mode="relaxed"):
                self.loss = self._step()
        except Exception as e:
            if "legacy stream" in repr(e) or "previous error during capture" in repr(e):
                raise RuntimeError("GraphedStep: the capture was invalidated -- most likely an autograd graph of an earlier eager "
                                   "step on the default stream is still alive (a loss tensor kept without .detach()); see the "
                                   "module docstring") from e
            raise
        self.steps_outside_graph = max(1, warmup) + 1      # the capture itself does not execute the step

    def _step(self) -> torch.Tensor:
        self.opt.zero_grad()
        loss = self.model.loss(self.model(self.static))
        loss.backward()
        self.opt.step()
        return loss.detach()

    def matches(self, feed: Dict) -> bool:
        return all(isinstance(feed.get(k), torch.Tensor) and tuple(feed[k].shape) == s for k, s in self.shapes.items())

    def __call__(self, feed: Dict) -> torch.Tensor:
        """copy the batch into the static buffers (H2D if it is on the host), replay; returns the step's loss (a static
        device scalar: read or clone it before the next replay)"""
        for k, s in self.shapes.items():
            self.static[k].copy_(feed[k], non_blocking=True)
        self.graph.replay()
        return self.loss

    def replay(self) -> torch.Tensor:
        """replay on whatever the static input tensors (``self.static``) hold now, with no copy: for a producer that writes
        each batch straight into them on the current stream (runner.fit_on_device).  Returns the step's loss, as ``__call__``"""
        self.graph.replay()
        return self.loss
