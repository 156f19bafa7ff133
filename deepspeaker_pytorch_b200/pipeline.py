"""Host-to-host (or device-to-device) embedding extraction with copy/compute overlap and several forwards in flight.

The reference's ``test()`` loop (reference train_triplet.py:337-350) moves every batch to the GPU, runs the
model and pulls the distances back, all serialised on one stream.  ``EmbeddingPipeline`` keeps the same per-batch
call but

* runs the H2D copy of batch i+1 and the D2H copy of batch i-1 on their own streams while batch i is in the ResCNN
  kernels (PCIe is full duplex; 2.6 MB in, 128 KB out per 64 utterances), and
* alternates batches between ``lanes`` compute streams, each with its own engine handle and activation workspace
  (all lanes read one packed weight image): a layer of a 64-utterance batch has only 1-2.4 tiles per SM, and a
  kernel's set-up and last-tile epilogue leave the tensor pipe idle, so a second and third forward in flight fill
  what the first one leaves.

The queueing itself is native (``dsk_pipeline_*`` in libdsk.so): one C call per batch issues the ~12 CUDA runtime calls
(copies, event waits / records, the forward's graph launch), so the Python cost per batch is one ctypes call
(~10 us) instead of the 0.12-0.18 ms the stream / event bookkeeping cost when it was written in Python - which at
8 processes per box was as long as the GPU step itself.
"""
from __future__ import annotations

import collections
import ctypes

import torch

from . import _lib as L


class EmbeddingPipeline:
    def __init__(self, model, lanes: int = 3, depth: int = 4, check_every: int = 1):
        """``check_every``: the parameter / BatchNorm-buffer versions are compared (and the packed weights refreshed when
        they changed) before every ``check_every``-th batch; 0 = never (a frozen model; call ``refresh()`` yourself)."""
        p = next(model.parameters())
        if not p.is_cuda:
            raise RuntimeError("EmbeddingPipeline needs the model on a CUDA device")
        if model.training:
            raise RuntimeError("EmbeddingPipeline is an inference helper: call model.eval() first")
        self.model = model
        self.device = p.device
        self.depth = depth
        self.lib = L.load()
        self.engine = model._get_engine(self.device)
        self.engine.sync_weights(eval_mode=True)
        self.handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_create(ctypes.byref(self.handle), self.engine.handle, lanes, depth),
                    "dsk_pipeline_create")
        self.embedding_size = model.embedding_size

        def _stream(i):
            s = ctypes.c_void_p()
            L.check(self.lib.dsk_pipeline_lane_stream(self.handle, i, ctypes.byref(s)), "dsk_pipeline_lane_stream")
            return torch.cuda.ExternalStream(s.value, device=self.device)

        self.lanes = [_stream(i) for i in range(lanes)]     # torch views of the native streams (event timing, joins)
        self.h2d, self.d2h = _stream(-1), _stream(-2)
        self._ticket = ctypes.c_int64(-1)
        self._calls = 0
        self.check_every = check_every
        # device-resident batches in flight: the pipeline keeps the input and output tensors alive until the lane has
        # finished with them (torch's record_stream cannot be used: the lane streams belong to libdsk, and the caching
        # allocator would try to record events on them after the pipeline is gone)
        self._inflight = collections.deque()

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.dsk_pipeline_destroy(self.handle)      # synchronises the lanes first
                self.handle = ctypes.c_void_p()
            self._inflight.clear()
        except Exception:
            pass

    def refresh(self):
        """Pick up parameter / BatchNorm-buffer changes now (the lanes re-adopt the primary's packed weights at their
        next forward).  Writes through ``param.data`` are invisible to the version check: call
        ``model.refresh_weights()`` first in that case."""
        self.engine.sync_weights(eval_mode=True)

    def _maybe_refresh(self):
        if self.check_every and self._calls % self.check_every == 0:
            self.engine.sync_weights(eval_mode=True)

    @torch.no_grad()
    def embed_device(self, x: torch.Tensor) -> torch.Tensor:
        """Queue one device-resident batch on the next compute lane; returns the (asynchronously produced) embeddings.

        Lifetimes: ``x`` may be dropped by the caller right after this call - the pipeline holds a reference until the
        lane has read it.  The returned ``emb`` is produced on the lane stream: order the consuming stream with
        ``wait_lanes()`` / ``synchronize()`` before reading it."""
        if not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous():
            x = x.to(self.device, torch.float32).contiguous()
        B, _, T, _ = x.shape
        self._maybe_refresh()
        lane = self.lanes[self._calls % len(self.lanes)]
        self._calls += 1
        emb = torch.empty(B, self.embedding_size, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_submit_device(self.handle, x.data_ptr(), B, T, emb.data_ptr(), L.cur_stream(),
                                                        ctypes.byref(self._ticket)), "dsk_pipeline_submit_device")
        done = torch.cuda.Event()
        done.record(lane)
        self._inflight.append((done, x, emb))
        while len(self._inflight) > 2 * len(self.lanes) * self.depth:
            ev, _, _ = self._inflight.popleft()
            if not ev.query():
                ev.synchronize()
        return emb

    def wait_lanes(self, stream=None):
        """Make ``stream`` (default: the current stream) wait for everything queued on the compute lanes."""
        stream = stream or torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_join(self.handle, stream.cuda_stream), "dsk_pipeline_join")

    @torch.no_grad()
    def embed(self, x_host: torch.Tensor, out_host: torch.Tensor) -> int:
        """Queue one batch: ``x_host`` (B,1,T,64) pinned fp32 -> ``out_host`` (B,E) pinned fp32.  Asynchronous: returns
        the batch's ticket; ``wait(ticket)`` blocks until ``out_host`` is complete (or call ``synchronize()``).  Both
        tensors must stay alive and untouched until then."""
        if not (x_host.is_pinned() and out_host.is_pinned()):
            raise RuntimeError("EmbeddingPipeline.embed needs pinned host tensors (asynchronous copies)")
        if x_host.dtype != torch.float32 or out_host.dtype != torch.float32 or not x_host.is_contiguous() or not out_host.is_contiguous():
            raise RuntimeError("EmbeddingPipeline.embed needs contiguous float32 tensors")
        B, _, T, _ = x_host.shape
        if out_host.shape != (B, self.embedding_size):
            raise RuntimeError(f"out_host must be ({B}, {self.embedding_size}), got {tuple(out_host.shape)}")
        self._maybe_refresh()
        self._calls += 1
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_submit(self.handle, x_host.data_ptr(), B, T, out_host.data_ptr(),
                                                 ctypes.byref(self._ticket)), "dsk_pipeline_submit")
        return self._ticket.value

    def wait(self, ticket: int):
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_wait(self.handle, int(ticket)), "dsk_pipeline_wait")

    def synchronize(self):
        with torch.cuda.device(self.device):
            L.check(self.lib.dsk_pipeline_sync(self.handle), "dsk_pipeline_sync")
        self._inflight.clear()
