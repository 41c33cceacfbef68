"""Host-buffer streaming front end of ``VQVAE.forward`` (models/vqvae.py:29-44 called in a loop,
as main.py:60-75 does with its DataLoader batches).

The reference's caller hands the model one host batch after another.  A cfg2 step's input and output
cross PCIe in each direction next to its kernels, so a caller that copies, runs and reads back
synchronously leaves the GPU idle while the copies run.  ``HostPipeline`` keeps
``depth`` batches in flight on three streams -- host->device copy, the captured forward graph,
device->host copy -- with one set of device buffers (and one captured graph) per slot.  Every
batch still goes host -> HBM -> kernels -> host; only the waiting is overlapped.

    pipe = HostPipeline(model, (256, 3, 32, 32), depth=3)
    for x in batches:                       # pinned (or pageable) host tensors
        done = pipe.push(x)                 # None until the pipe is full, then the oldest result
        if done is not None: consume(done)  # done.loss, done.x_hat (host), done.perplexity
    for done in pipe.drain(): consume(done)

A result's host tensors belong to a slot that the NEXT ``push`` reuses: read (or copy) them before
pushing again.  (``depth`` + 1 slots exist so that the result handed out by a push is not the slot
that push refills.)
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass
from typing import Deque, List, Optional

import torch

from ._lib import check, lib
from .modules import _INVALIDATIONS


@dataclass
class HostResult:
    index: int                   # running number of the batch this result belongs to
    loss: torch.Tensor           # 0-d host tensor (models/vqvae.py:44 embedding_loss)
    x_hat: torch.Tensor          # host tensor, same shape as the input batch
    perplexity: torch.Tensor     # 0-d host tensor


def _packed_scalars_ptr(loss, perp):
    """Address of [loss, perplexity] when the two 0-d tensors are adjacent fp32 views of one buffer
    (ops.vq_finish returns them that way): one device->host copy instead of two."""
    if (loss.dtype == torch.float32 and perp.dtype == torch.float32 and loss.numel() == 1 and perp.numel() == 1
            and perp.data_ptr() == loss.data_ptr() + 4):
        return loss.data_ptr()
    return None


class _Slot:
    def __init__(self, model, shape, device, use_graph):
        self.x_dev = torch.zeros(shape, dtype=torch.float32, device=device)
        self.x_hat_host = torch.empty(shape, dtype=torch.float32).pin_memory()
        self.scalars_host = torch.empty((2,), dtype=torch.float32).pin_memory()
        self.h2d_done = torch.cuda.Event()
        self.compute_done = torch.cuda.Event()
        self.d2h_done = torch.cuda.Event()
        self.busy = False
        self.index = -1
        self.graph = None
        self.out = None
        self.x_hat_ptr = None        # graph mode: fixed output addresses -> raw stream-ordered copies
        self.scalars_ptr = None
        self.x_ref = None
        self.model = model
        if use_graph:
            warm = torch.cuda.Stream(device=device)
            warm.wait_stream(torch.cuda.current_stream(device))
            with torch.cuda.stream(warm), torch.no_grad():
                for _ in range(2):                       # packs weights, sizes workspaces
                    model(self.x_dev)
            torch.cuda.current_stream(device).wait_stream(warm)
            torch.cuda.synchronize(device)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph), torch.no_grad():
                self.out = model(self.x_dev)
            torch.cuda.synchronize(device)
            loss, x_hat, perp = self.out
            self.x_hat_ptr = x_hat.data_ptr() if x_hat.is_contiguous() else None
            self.scalars_ptr = _packed_scalars_ptr(loss, perp)

    def run(self):
        if self.graph is not None:
            self.graph.replay()
            return self.out
        with torch.no_grad():
            return self.model(self.x_dev)


class HostPipeline:
    """``depth`` host batches in flight through ``model`` (a vqvae_b200 ``VQVAE`` on a CUDA device)."""

    def __init__(self, model, batch_shape, depth: int = 3, use_graph: bool = True, raw_copies: bool = True):
        p = next(model.parameters())
        if p.device.type != "cuda":
            raise RuntimeError("HostPipeline needs the model on a CUDA device (there is no CPU path)")
        if depth < 1:
            raise ValueError("depth must be >= 1")
        self.device = p.device
        self.shape = tuple(int(s) for s in batch_shape)
        self.h2d_bytes = 4 * int(torch.Size(self.shape).numel())
        self.d2h_bytes = self.h2d_bytes + 8
        with torch.cuda.device(self.device):
            self._copy_in = torch.cuda.Stream()
            self._compute = torch.cuda.Stream()
            self._copy_out = torch.cuda.Stream()
            # depth in flight + the one whose result the caller is still reading
            self._slots = [_Slot(model, self.shape, self.device, use_graph) for _ in range(depth + 1)]
        self.depth = depth
        self.model = model
        self._params = list(model.parameters())
        self._pstate = self._param_versions()
        self._pstate_fast = self._param_versions(False)
        self._inflight: Deque[_Slot] = deque()
        self._count = 0
        self._lib = lib()
        self._raw = bool(raw_copies)

    # -- internals ---------------------------------------------------------------------------
    def _param_versions(self, full=True):
        """Fingerprint of the weights the captured graphs depend on.  ``full``: version counters AND storage addresses
        (``.to()``, re-assigned ``.data``); the cheap form (version counters only: ~2 us for the 23 tensors) runs on
        every push, the full one on every 32nd -- a push must stay far below the 140 us the device needs per step."""
        try:
            if full:
                return (_INVALIDATIONS["n"],) + tuple((p._version, p.data_ptr()) for p in self._params)
            return (_INVALIDATIONS["n"],) + tuple([p._version for p in self._params])
        except RuntimeError:                     # inference tensors carry no version counter: always refresh
            return None

    def _refresh_weights(self):
        """The captured graphs read the packed-weight buffers, which only a Python-side forward refreshes: after a
        load_state_dict / optimizer step, repack IN PLACE (same buffers) on the compute stream before the next replay
        (``param.data`` edits are invisible to torch's version counters: call vqvae_b200.invalidate_packed first)."""
        full = (self._count & 31) == 0
        st = self._param_versions(full)
        if st is not None and st == (self._pstate if full else self._pstate_fast):
            return
        if not full:
            st = self._param_versions(True)
        prev = torch.cuda.current_stream(self.device)
        torch.cuda.set_stream(self._compute)
        try:
            self.model.repack()
        finally:
            torch.cuda.set_stream(prev)
        self._pstate = st
        self._pstate_fast = self._param_versions(False)

    def _finish(self, slot: _Slot) -> HostResult:
        slot.d2h_done.synchronize()
        slot.busy = False
        return HostResult(slot.index, slot.scalars_host[0], slot.x_hat_host, slot.scalars_host[1])

    # -- public ------------------------------------------------------------------------------
    def push(self, x_host: torch.Tensor) -> Optional[HostResult]:
        """Queue one host batch; returns the oldest outstanding result once ``depth`` are in flight."""
        if (tuple(x_host.shape) != self.shape or x_host.dtype != torch.float32 or x_host.device.type != "cpu"
                or not x_host.is_contiguous()):
            raise ValueError(f"expected a contiguous float32 host tensor of shape {self.shape}")
        done = None
        if len(self._inflight) == self.depth:
            done = self._finish(self._inflight.popleft())
        self._refresh_weights()
        slot = self._slots[self._count % len(self._slots)]
        assert not slot.busy
        slot.busy, slot.index = True, self._count
        self._count += 1
        nbytes = self.h2d_bytes
        if self._raw and slot.graph is not None and slot.x_hat_ptr is not None and slot.scalars_ptr is not None:
            # graph mode: every address is fixed, so the step is a dozen cheap calls (event waits/records, three
            # stream-ordered copies through the C ABI, one graph launch) -- no stream contexts, no Tensor.copy_
            L = self._lib
            cin, comp, cout = self._copy_in, self._compute, self._copy_out
            cin.wait_event(slot.compute_done)            # the slot's previous forward has read x_dev
            slot.x_ref = x_host                          # keep the source alive until this slot is reused
            check(L.vqb_memcpy_async(slot.x_dev.data_ptr(), x_host.data_ptr(), nbytes, 1, cin.cuda_stream), "h2d")
            slot.h2d_done.record(cin)
            comp.wait_event(slot.h2d_done)
            comp.wait_event(slot.d2h_done)               # previous outputs of this slot are on the host
            prev = torch.cuda.current_stream(self.device)
            torch.cuda.set_stream(comp)
            try:
                slot.graph.replay()
            finally:
                torch.cuda.set_stream(prev)
            slot.compute_done.record(comp)
            cout.wait_event(slot.compute_done)
            check(L.vqb_memcpy_async(slot.x_hat_host.data_ptr(), slot.x_hat_ptr, nbytes, 2, cout.cuda_stream), "d2h")
            check(L.vqb_memcpy_async(slot.scalars_host.data_ptr(), slot.scalars_ptr, 8, 2, cout.cuda_stream), "d2h")
            slot.d2h_done.record(cout)
            self._inflight.append(slot)
            return done
        with torch.cuda.stream(self._copy_in):
            # the slot's previous forward has read x_dev (its result was handed out above or earlier)
            self._copy_in.wait_event(slot.compute_done)
            slot.x_dev.copy_(x_host, non_blocking=True)
            slot.h2d_done.record()
        with torch.cuda.stream(self._compute):
            self._compute.wait_event(slot.h2d_done)
            self._compute.wait_event(slot.d2h_done)      # previous outputs of this slot are on the host
            loss, x_hat, perp = slot.run()
            slot.compute_done.record()
            if slot.graph is None:                       # eager outputs come from the caching allocator
                for t in (loss, x_hat, perp):
                    t.record_stream(self._copy_out)
        with torch.cuda.stream(self._copy_out):
            self._copy_out.wait_event(slot.compute_done)
            slot.x_hat_host.copy_(x_hat, non_blocking=True)
            slot.scalars_host[0:1].copy_(loss.reshape(1), non_blocking=True)
            slot.scalars_host[1:2].copy_(perp.reshape(1), non_blocking=True)
            slot.d2h_done.record()
        self._inflight.append(slot)
        return done

    def drain(self) -> List[HostResult]:
        """Wait for everything in flight; results in submission order."""
        out = []
        while self._inflight:
            out.append(self._finish(self._inflight.popleft()))
        return out

    def run(self, batches, on_result=None) -> int:
        """Push every batch of an iterable; ``on_result`` sees each result in order.  Returns the count."""
        n = 0
        for x in batches:
            r = self.push(x)
            n += 1
            if r is not None and on_result is not None:
                on_result(r)
        for r in self.drain():
            if on_result is not None:
                on_result(r)
        return n
