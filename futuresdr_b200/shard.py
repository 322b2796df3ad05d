"""Multi-GPU sharding of one logical sample stream (SURVEY.md §8e; new design -- the reference
is single-process, single-device).

One process per GPU.  The stream is cut into contiguous time ranges: at step ``t`` rank ``r``
of ``W`` owns samples ``[(t*W + r)*S, (t*W + r + 1)*S)``.  A FIR output needs the ``ntaps-1``
inputs before it, so the only data-path exchange is the *overlap region*: every rank
contributes the last ``H = ceil((ntaps-1)/D)*D`` samples of its chunk to one fixed-size NCCL
all-gather (2 KiB per rank for 256 taps) and installs its left neighbour's tail as history in
front of its own chunk (rank 0 takes rank ``W-1``'s tail of the previous step; at the very start
of the stream there is no history, so the first chunk yields ``S-(ntaps-1)`` outputs exactly like
the reference, perf/fir/fir.rs:97).

The exchange is latency-bound (~tens of microseconds), so it is taken off the critical path: the
all-gather is launched asynchronously, the outputs whose window lies entirely inside the rank's
own chunk (all but the first ``split/D``, split = H rounded up to an aligned slice) are computed meanwhile, and only a small second launch for
the first ``H/D`` outputs waits for the neighbour's tail.

The per-rank compute is the same C-ABI FIR plan as the single-GPU path; ``compute`` can be
replaced (tests run this file's logic on CPU over gloo with the oracle as the kernel).

``exchange="peer"`` (the default on GPUs) removes even that from the step: every rank keeps its chunks in a
C-ABI device ring (``b2s_ring_*``) exported to its right neighbour through CUDA IPC, and the FIR kernel's
TMA loader fetches the left neighbour's last ``H`` samples straight from the neighbour's HBM over NVLink in
front of its first tile (``b2s_fir_exec_hist``) -- ONE launch per step, no copy, no collective, no host
synchronisation.  Ordering is two u32 counters per ring in device memory: ``ready`` (chunks published by the
owner, release store) which the neighbour's kernel spins on before it reads the tail, and ``consumed``
(written back by that kernel) which the owner's stream waits on before it refills the slot.  NCCL is only
used to bootstrap (exchange of the 64-byte IPC handles).  ``exchange="nccl"`` keeps the all-gather variant
(the north star's wording; also what the gloo tests exercise on CPU).
"""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np
import torch
import torch.distributed as dist

from . import _lib


class ShardedFir:
    def __init__(self, taps, chunk_items: int, sample_dtype=np.complex64, decim: int = 1,
                 device: Optional[torch.device] = None, group=None,
                 compute: Optional[Callable] = None, algo: int = 0, overlap: bool = True,
                 exchange: str = "auto", n_slots: int = 2):
        self.taps = np.ascontiguousarray(taps)
        self.ntaps = int(self.taps.size)
        self.S = int(chunk_items)
        self.decim = int(decim)
        # History a chunk needs so its first output continues the global output sequence without
        # gap or overlap: H = ceil((ntaps-1)/D)*D  (== ntaps-1 for D == 1).  The reference keeps
        # slice starts at multiples of D because it consumes n*D items per call
        # (decimating_fir.rs:94); H being a multiple of D preserves that phase across shards.
        self.halo = ((self.ntaps + self.decim - 2) // self.decim) * self.decim
        if self.S % self.decim:
            raise ValueError("chunk_items must be a multiple of decim so shard phases align")
        # Split point of the overlapped step: outputs [0, split/D) need the neighbour's tail, the rest only
        # the rank's own chunk.  It is H rounded up so that both xbuf[split:] and out[split/D:] stay 16-byte
        # aligned -- an unaligned slice would push the FIR plan onto its scalar fallback kernel.
        isz = np.dtype(sample_dtype).itemsize
        q = self.decim * max(1, 16 // isz)
        self.split = ((self.halo + q - 1) // q) * q
        if self.S < self.split + self.ntaps:
            raise ValueError("chunk shorter than the FIR history")
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.tdtype = torch.complex64 if np.dtype(sample_dtype) == np.complex64 else torch.float32
        self.sample_dtype = np.dtype(sample_dtype)
        if exchange == "none":              # independent replicas: every rank runs its own stream (diagnostics)
            self.rank, self.world, exchange = 0, 1, "peer"
        if exchange == "auto":
            exchange = "peer" if (compute is None and self.device.type == "cuda") else "nccl"
        if exchange not in ("peer", "nccl"):
            raise ValueError("exchange must be 'auto', 'peer', 'nccl' or 'none'")
        self.exchange = exchange
        self.have_history = False          # becomes True after the first step of the stream
        self.step_index = 0
        self.overlap = bool(overlap)
        self.on_kernel = None              # optional callable("begin" | "end") around the FIR launch (bench timing)
        if exchange == "peer":
            self._init_peer(algo, int(n_slots))
            return
        # [halo | chunk] contiguous so the kernel sees history + new samples as one slice
        self.xbuf = torch.zeros(self.halo + self.S, dtype=self.tdtype, device=self.device)
        self.tails = torch.zeros(self.world, max(self.halo, 1), dtype=self.tdtype, device=self.device)
        self.my_tail = torch.zeros(max(self.halo, 1), dtype=self.tdtype, device=self.device)
        self.prev_last_tail = torch.zeros(max(self.halo, 1), dtype=self.tdtype, device=self.device)
        if compute is None:
            from .filters import DecimatingFirFilter
            ctx = self._make_ctx()
            self._filter = DecimatingFirFilter(self.decim, self.taps, sample_dtype, ctx=ctx, algo=algo)
            compute = self._filter.filter
            # the split/D outputs behind the exchange are a few hundred items: the CUDA-core kernel has no
            # tap-table prologue, so that second launch costs ~half of a tensor-kernel launch
            self._head_filter = DecimatingFirFilter(self.decim, self.taps, sample_dtype, ctx=ctx, algo=_lib.ALGO_DIRECT)
            head_compute = self._head_filter.filter
        else:
            head_compute = compute
        self.compute = compute
        self.head_compute = head_compute

    def _make_ctx(self):
        """The context of THIS object's device and of torch's current stream there (not whatever device happens
        to be current): buffers, kernels and collectives must share one device and one stream order."""
        from .context import Context
        return Context(self.device.index if self.device.index is not None else torch.cuda.current_device(),
                       stream=torch.cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------------------------------------
    # exchange == "peer": device ring + CUDA-IPC peer mapping + in-kernel history fetch
    # ------------------------------------------------------------------------------------------------
    def _init_peer(self, algo: int, n_slots: int):
        import ctypes as C
        from ._lib import lib, check
        from .filters import DecimatingFirFilter
        if n_slots < 2:
            raise ValueError("the peer exchange needs at least two ring slots")
        self.ctx = self._make_ctx()
        self._filter = DecimatingFirFilter(self.decim, self.taps, self.sample_dtype, ctx=self.ctx, algo=algo)
        self.n_slots = n_slots
        isz = self.sample_dtype.itemsize
        if (self.S * isz) % 16:
            raise ValueError("chunk_items must be a whole number of 16-byte units for the peer exchange")
        self._ring = C.c_void_p()
        check(lib.b2s_ring_create(self.ctx.handle, isz, self.S, max(self.halo, 1), n_slots, 0, C.byref(self._ring)),
              self.ctx.handle)
        self._base = lib.b2s_ring_base(self._ring)
        self._slot_off = [lib.b2s_ring_slot_offset(self._ring, i) for i in range(n_slots)]
        self._flags_off = lib.b2s_ring_flags_offset(self._ring)
        self._ready = self._base + self._flags_off            # chunks this rank has published
        self._consumed = self._base + self._flags_off + 4     # chunks whose tail the right neighbour has read
        self._left_base = self._base                          # world == 1: the "neighbour" is this ring
        self._left_mapped = None
        if self.world > 1:
            h = (C.c_uint8 * 64)()
            check(lib.b2s_ipc_export(self.ctx.handle, C.c_void_p(self._base), h), self.ctx.handle)
            mine = {"handle": bytes(h), "slot_off": self._slot_off, "flags_off": self._flags_off, "pid": __import__("os").getpid(),
                    "device": self.ctx.device}
            allh = [None] * self.world
            dist.all_gather_object(allh, mine, group=self.group)
            left = allh[(self.rank - 1) % self.world]
            if left["slot_off"] != self._slot_off or left["flags_off"] != self._flags_off:
                raise RuntimeError("ring geometry differs between ranks")
            if left["pid"] == mine["pid"]:
                raise RuntimeError("peer exchange needs one process per rank")
            p = C.c_void_p()
            hb = (C.c_uint8 * 64).from_buffer_copy(left["handle"])
            check(lib.b2s_ipc_open(self.ctx.handle, hb, C.byref(p)), self.ctx.handle)
            self._left_base = self._left_mapped = p.value
        self._cur = None          # slot index being filled for the coming step
        self._slots = [None] * n_slots

    def close(self):
        if getattr(self, "exchange", None) == "peer" and getattr(self, "_ring", None):
            from ._lib import lib
            self.ctx.sync()
            if self.world > 1 and dist.is_initialized():
                dist.barrier(group=self.group)            # nobody may still be reading this ring
            if self._left_mapped:
                lib.b2s_ipc_close(self.ctx.handle, self._left_mapped)
                self._left_mapped = None
            lib.b2s_ring_destroy(self._ring)
            self._ring = None

    def _slot_tensor(self, index: int) -> torch.Tensor:
        from .edges import _DevView
        return torch.as_tensor(_DevView(self._base + self._slot_off[index], self.S, self.sample_dtype), device=self.device)

    def slot_tensors(self):
        """All ring slots as tensors (benchmarks pre-fill them once so that the timed steps find their
        input resident in HBM)."""
        return [self._slot_tensor(i) for i in range(self.n_slots)]

    def begin_chunk(self) -> torch.Tensor:
        """Writable view of the slot of the coming step.  Before the slot is handed out the stream waits until
        the right neighbour has read the tail of the chunk that last lived in it (``consumed`` counter)."""
        if self.exchange != "peer":
            return self.xbuf[self.halo:]
        if self._cur is None:
            from ._lib import lib, check
            t = self.step_index
            self._cur = t % self.n_slots
            if self.world > 1 and t >= self.n_slots and self.halo:
                check(lib.b2s_flag_wait(self.ctx.handle, self._consumed, t - self.n_slots + 1), self.ctx.handle)
        return self._slot_tensor(self._cur)

    @property
    def chunk(self) -> torch.Tensor:
        """The rank's writable chunk (fill this with the step's samples)."""
        return self.begin_chunk()

    def _step_peer(self, out: torch.Tensor):
        import ctypes as C
        from ._lib import lib, check
        self.begin_chunk()
        t, W, r, H, S = self.step_index, self.world, self.rank, self.halo, self.S
        isz = self.sample_dtype.itemsize
        cur = self._cur
        d_in = self._base + self._slot_off[cur]
        from ._lib import Handshake
        hs = Handshake()
        if W > 1 and H:
            hs.publish_flag, hs.publish_value = self._ready, t + 1                            # publish chunk t
        first_of_stream = r == 0 and t == 0
        c, p, st = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
        if self.on_kernel:
            self.on_kernel("begin")
        if first_of_stream or H == 0:
            check(lib.b2s_fir_exec_hist(self._filter._h, None, 0, C.c_void_p(d_in), S, C.c_void_p(out.data_ptr()),
                                        out.numel(), C.byref(hs), C.byref(c), C.byref(p), C.byref(st)), self.ctx.handle)
        else:
            if r == 0:      # history = the tail of rank W-1's chunk of the PREVIOUS step
                src_slot, need = (t - 1) % self.n_slots, t
            else:           # history = the tail of rank r-1's chunk of THIS step
                src_slot, need = cur, t + 1
            d_hist = self._left_base + self._slot_off[src_slot] + (S - H) * isz
            if W > 1:
                hs.wait_flag, hs.wait_value = self._left_base + self._flags_off, need
                hs.done_flag, hs.done_value = self._left_base + self._flags_off + 4, need
            check(lib.b2s_fir_exec_hist(self._filter._h, C.c_void_p(d_hist), H, C.c_void_p(d_in), S,
                                        C.c_void_p(out.data_ptr()), out.numel(), C.byref(hs),
                                        C.byref(c), C.byref(p), C.byref(st)), self.ctx.handle)
        if self.on_kernel:
            self.on_kernel("end")
        self._cur = None
        self.have_history = True
        self.step_index += 1
        from .filters import ComputationStatus
        return c.value, p.value, ComputationStatus(st.value)

    def _exchange(self, async_op: bool):
        """All-gather of the overlap region (every rank's last H samples). Returns a work handle or None."""
        if self.halo == 0:
            return None
        my_tail = self.xbuf[self.S:]                     # last `halo` samples of [halo|chunk], contiguous
        if self.world == 1:
            self.tails[0].copy_(my_tail)
            return None
        # complex tensors travel as their (re, im) float view
        real = (lambda t: torch.view_as_real(t) if t.is_complex() else t)
        return dist.all_gather_into_tensor(real(self.tails).reshape(-1), real(my_tail).reshape(-1),
                                           group=self.group, async_op=async_op)

    def step(self, out: torch.Tensor):
        """Filter this step's chunk (already written into ``self.chunk``).

        Returns (consumed, produced, status).  ``out`` must hold ``S // decim`` items.
        """
        if self.exchange == "peer":
            return self._step_peer(out)
        H, D, N = self.halo, self.decim, self.ntaps
        first_of_stream = self.rank == 0 and not self.have_history
        if self.world == 1:
            # single rank: the history of step t+1 is the tail of step t's own chunk -- one device copy
            # per step, no gather buffers
            res = self.compute(self.xbuf[H:] if first_of_stream else self.xbuf, out)
            if H:
                self.xbuf[:H].copy_(self.xbuf[self.S:])
            self.have_history = True
            self.step_index += 1
            return res
        work = self._exchange(async_op=self.overlap)
        if first_of_stream:
            res = self.compute(self.xbuf[H:], out)                       # no history: S-(ntaps-1) outputs
        elif self.rank == 0:
            # history = rank W-1's tail of the PREVIOUS step (saved before this step's gather started)
            if H:
                self.xbuf[:H].copy_(self.prev_last_tail[:H])
            res = self.compute(self.xbuf, out)
        elif H == 0:
            res = self.compute(self.xbuf, out)
        elif self.overlap:
            A = self.split
            nh = A // D                                                  # outputs that (may) need the neighbour's tail
            c1, p1, st = self.compute(self.xbuf[A:], out[nh:])           # windows fully inside the own chunk
            if work is not None:
                work.wait()
                work = None
            self.xbuf[:H].copy_(self.tails[self.rank - 1][:H])
            c0, p0, _ = self.head_compute(self.xbuf[:A + N - 1], out[:nh])   # the first split/D outputs
            res = (c0 + c1, p0 + p1, st)
        else:
            if work is not None:
                work.wait()
                work = None
            self.xbuf[:H].copy_(self.tails[self.rank - 1][:H])
            res = self.compute(self.xbuf, out)
        if work is not None:
            work.wait()
        if self.rank == 0 and H:
            self.prev_last_tail.copy_(self.tails[self.world - 1])        # history for the next step
        self.have_history = True
        self.step_index += 1
        return res
