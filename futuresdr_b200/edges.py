"""Host edges and wire format for the hot-path blocks (SURVEY.md §8f row 4).

What the reference has, and what mirrors it here:

  * ``VectorSource`` / ``VectorSink``   src/blocks/vector_source.rs:25-75, vector_sink.rs:20-70
  * ``FileSource`` / ``FileSink``       src/blocks/file_source.rs:24-100, file_sink.rs:33-95 -- raw native-endian
    items, i.e. interleaved ``f32 re, f32 im`` for ``Complex<f32>`` (the ``*.cf32`` captures under
    examples/wlan/data); ``repeat`` re-opens the file at EOF exactly like file_source.rs:66-70
  * the H2D / D2H stream edges          src/runtime/buffer/vulkan/h2d.rs:161-232, d2h.rs:66-74, :270-299:
    pinned staging per slot, asynchronous copy, an event per slot (the Vulkan fence) -- here the
    C-ABI ring (``b2s_ring_*``, ``b2s_slot_*``).  The host fills slot k+1 while the GPU still works on k.
  * a device stream buffer between two blocks (``StreamBuffer``): the role of buffer/slab.rs on the CPU --
    a reader sees its unconsumed items plus everything produced since, contiguously, in HBM.

``run_chain`` is NOT a scheduler (the reference's runtime is out of scope, SURVEY.md §8): it is the
Mocker idea (src/runtime/mocker.rs) extended to a linear chain -- call ``work`` on every stage in turn
until all report finished -- so the edges and the finish rules can be tested end to end.  ``Flowgraph``
does the same for branching graphs (fan-out through ``MultiStreamBuffer``, fan-in through multi-input
blocks such as Combine) with the reference's StreamInputDone / StreamOutputDone finish rules.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import lib, check
from .blocks import Block, WorkIo, _tdtype
from .context import Context, default_context


# ---------------------------------------------------------------------------------------------------
# device stream buffer + the two port views blocks use (same methods as mocker::Reader / Writer)
# ---------------------------------------------------------------------------------------------------
class StreamBuffer:
    """Linear device buffer shared by one writer and one reader; unconsumed items are moved to the front
    when the free tail gets short (slab.rs keeps history the same way)."""

    def __init__(self, dtype, capacity_items: int, device="cuda"):
        self.dtype = np.dtype(dtype)
        self.data = torch.empty(int(capacity_items), dtype=_tdtype(dtype), device=device)
        self.rd = 0
        self.wr = 0
        self.writer_finished = False

    def _compact(self):
        rem = self.wr - self.rd
        if self.rd == 0:
            return
        if rem:
            src = self.data[self.rd:self.wr]
            if rem > self.rd:                       # source and destination overlap
                src = src.clone()
            self.data[:rem].copy_(src)
        self.rd, self.wr = 0, rem

    # writer side
    def write_slice(self) -> torch.Tensor:
        if self.rd and (self.data.numel() - self.wr) < self.data.numel() // 2:
            self._compact()
        return self.data[self.wr:]

    def produce(self, n: int):
        assert self.wr + n <= self.data.numel()
        self.wr += n

    # reader side
    def read_slice(self) -> torch.Tensor:
        return self.data[self.rd:self.wr]

    def consume(self, n: int):
        assert self.rd + n <= self.wr
        self.rd += n


class _ReaderPort:
    def __init__(self, buf: StreamBuffer):
        self.buf, self.dtype, self.min_items = buf, buf.dtype, 1

    def slice(self):
        return self.buf.read_slice()

    def consume(self, n):
        self.buf.consume(n)

    def finished(self):
        return self.buf.writer_finished

    def set_min_items(self, n):
        self.min_items = max(self.min_items, n)


class _WriterPort:
    def __init__(self, buf: StreamBuffer):
        self.buf, self.dtype, self.min_items = buf, buf.dtype, 1

    def slice(self):
        return self.buf.write_slice()

    def produce(self, n):
        self.buf.produce(n)

    def set_min_items(self, n):
        self.min_items = max(self.min_items, n)


class MultiStreamBuffer:
    """Linear device buffer with one writer and ``n_readers`` readers, each with its own read cursor (the reference's
    buffers let one output feed several inputs).  The writer's free space is bounded by the slowest reader that is
    still running: unconsumed items from the smallest live read cursor on are moved to the front when the free tail
    gets short.  A reader whose block has finished no longer holds items back."""

    def __init__(self, dtype, capacity_items: int, n_readers: int, device="cuda"):
        self.dtype = np.dtype(dtype)
        self.data = torch.empty(int(capacity_items), dtype=_tdtype(dtype), device=device)
        self.rd = [0] * int(n_readers)
        self.live = [True] * int(n_readers)
        self.wr = 0
        self.shift = 0                              # items dropped from the front by compaction so far
        self.writer_finished = False

    def _low(self) -> int:
        live = [r for r, a in zip(self.rd, self.live) if a]
        return min(live) if live else self.wr

    def _compact(self):
        lo = self._low()
        if lo == 0:
            return
        rem = self.wr - lo
        if rem:
            src = self.data[lo:self.wr]
            if rem > lo:                            # source and destination overlap
                src = src.clone()
            self.data[:rem].copy_(src)
        self.rd = [max(r - lo, 0) for r in self.rd]
        self.wr = rem
        self.shift += lo

    # writer side
    def write_slice(self) -> torch.Tensor:
        if self._low() and (self.data.numel() - self.wr) < self.data.numel() // 2:
            self._compact()
        return self.data[self.wr:]

    def produce(self, n: int):
        assert self.wr + n <= self.data.numel()
        self.wr += n

    # reader side
    def read_slice(self, k: int) -> torch.Tensor:
        return self.data[self.rd[k]:self.wr]

    def consume(self, k: int, n: int):
        assert self.rd[k] + n <= self.wr
        self.rd[k] += n

    def cursors(self) -> tuple:
        """Stream positions of the write and read cursors (unchanged by compaction)."""
        return (self.wr + self.shift, *(r + self.shift for r in self.rd))


class _MultiReaderPort:
    def __init__(self, buf: MultiStreamBuffer, k: int):
        self.buf, self.k, self.dtype, self.min_items = buf, k, buf.dtype, 1

    def slice(self):
        return self.buf.read_slice(self.k)

    def consume(self, n):
        self.buf.consume(self.k, n)

    def finished(self):
        return self.buf.writer_finished

    def set_min_items(self, n):
        self.min_items = max(self.min_items, n)


class _DevView:
    """Zero-copy torch view of ``n`` items at a raw device pointer (a ring slot's buffer)."""

    def __init__(self, ptr: int, n: int, dtype):
        dt = np.dtype(dtype)
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": dt.str, "data": (int(ptr), False), "version": 2}


def _slot_tensor(slot, n: int, dtype) -> torch.Tensor:
    return torch.as_tensor(_DevView(lib.b2s_slot_device_ptr(slot), n, dtype), device="cuda")


def _slot_host(slot, n: int, dtype) -> np.ndarray:
    dt = np.dtype(dtype)
    raw = (C.c_char * (n * dt.itemsize)).from_address(lib.b2s_slot_host_ptr(slot))
    return np.frombuffer(raw, dtype=dt, count=n)


class _Ring:
    def __init__(self, ctx: Context, dtype, chunk_items: int, n_slots: int):
        self.ctx, self.dtype, self.chunk = ctx, np.dtype(dtype), int(chunk_items)
        self.h = C.c_void_p()
        check(lib.b2s_ring_create(ctx.handle, self.dtype.itemsize, self.chunk, 0, n_slots, 1, C.byref(self.h)), ctx.handle)

    def acquire_empty(self):
        s = C.c_void_p()
        rc = lib.b2s_ring_acquire_empty(self.h, C.byref(s))
        if rc == _lib.EAGAIN:
            return None
        check(rc, self.ctx.handle)
        return s

    def close(self):
        if self.h:
            lib.b2s_ring_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


# ---------------------------------------------------------------------------------------------------
# sources: host items -> pinned staging -> async H2D -> device stream
# ---------------------------------------------------------------------------------------------------
class _HostSource(Block):
    """Common H2D edge (buffer/vulkan/h2d.rs): one ring slot per chunk; the slot's event guards its pinned
    staging, so refilling slot k+n_slots only ever waits for a copy issued n_slots chunks ago."""

    def __init__(self, dtype, chunk_items: int = 1 << 20, n_slots: int = 3, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.out_dtype = np.dtype(dtype)
        self.in_dtype = None
        self.chunk = int(chunk_items)
        self._ring = _Ring(self.ctx, dtype, self.chunk, n_slots)
        self.output = None
        self.h2d_bytes = 0

    def _fill(self, host: np.ndarray) -> tuple[int, bool]:
        """Write up to host.size items into ``host``; return (items written, end of data)."""
        raise NotImplementedError

    def work(self, io: WorkIo):
        out = self.output.slice()
        room = min(out.numel(), self.chunk)
        if room == 0:
            return
        slot = self._ring.acquire_empty()
        assert slot is not None, "H2D ring exhausted: a slot was not released"
        check(lib.b2s_slot_wait(slot), self.ctx.handle)            # staging free again (its last H2D completed)
        n, eof = self._fill(_slot_host(slot, room, self.out_dtype))
        check(lib.b2s_ring_submit_full(self._ring.h, slot, n, 1), self.ctx.handle)      # async H2D + event
        full, valid = C.c_void_p(), C.c_size_t(0)
        check(lib.b2s_ring_acquire_full(self._ring.h, C.byref(full), C.byref(valid)), self.ctx.handle)
        if n:
            out[:n].copy_(_slot_tensor(full, n, self.out_dtype))  # stream-ordered behind the H2D
            self.output.produce(n)
            self.h2d_bytes += n * self.out_dtype.itemsize
        check(lib.b2s_ring_release(self._ring.h, full), self.ctx.handle)
        if eof:
            io.finished = True


class VectorSource(_HostSource):
    """blocks::VectorSource (vector_source.rs:38-75): emits ``items`` once, then finishes."""

    def __init__(self, items, chunk_items: int = 1 << 20, ctx: Optional[Context] = None):
        items = np.ascontiguousarray(items)
        super().__init__(items.dtype, chunk_items, ctx=ctx)
        self.items, self.pos = items, 0

    def _fill(self, host):
        n = min(host.size, self.items.size - self.pos)
        host[:n] = self.items[self.pos:self.pos + n]
        self.pos += n
        return n, self.pos == self.items.size


class FileSource(_HostSource):
    """blocks::FileSource<T> (file_source.rs:24-100): raw items of ``dtype`` (cf32 = interleaved f32 pairs)
    read straight into the pinned staging buffer; ``repeat`` re-opens the file at EOF (:66-70)."""

    def __init__(self, file_path, dtype=np.complex64, repeat: bool = False, chunk_items: int = 1 << 20,
                 ctx: Optional[Context] = None):
        super().__init__(dtype, chunk_items, ctx=ctx)
        self.file_path, self.repeat = os.fspath(file_path), bool(repeat)
        self.file = open(self.file_path, "rb", buffering=0)        # init(): file_source.rs:94-97

    def _fill(self, host):
        raw = memoryview(host.view(np.uint8))
        i, eof = 0, False
        while i < len(raw):
            got = self.file.readinto(raw[i:])
            if not got:
                if self.repeat:
                    self.file.close()
                    self.file = open(self.file_path, "rb", buffering=0)
                    if os.fstat(self.file.fileno()).st_size == 0:
                        eof = True
                        break
                else:
                    eof = True
                    break
            else:
                i += got
        return i // self.out_dtype.itemsize, eof                  # produce(i / item_size), :86


# ---------------------------------------------------------------------------------------------------
# sinks: device stream -> slot -> async D2H into pinned staging -> host
# ---------------------------------------------------------------------------------------------------
class _HostSink(Block):
    """Common D2H edge (buffer/vulkan/d2h.rs): the copy of chunk k is in flight while chunk k+1 is being
    produced; the host touches a slot's staging only after ``b2s_slot_wait`` on it."""

    def __init__(self, dtype, chunk_items: int = 1 << 20, n_slots: int = 3, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.in_dtype = np.dtype(dtype)
        self.out_dtype = None
        self.chunk = int(chunk_items)
        self._ring = _Ring(self.ctx, dtype, self.chunk, n_slots)
        self._inflight: List[tuple] = []
        self._depth = max(1, n_slots - 1)
        self.input = None
        self.d2h_bytes = 0

    def _take(self, host: np.ndarray):
        raise NotImplementedError

    def _drain(self, keep: int):
        while len(self._inflight) > keep:
            slot, n = self._inflight.pop(0)
            check(lib.b2s_slot_wait(slot), self.ctx.handle)
            self._take(_slot_host(slot, n, self.in_dtype))
            check(lib.b2s_ring_release(self._ring.h, slot), self.ctx.handle)

    def work(self, io: WorkIo):
        i = self.input.slice()
        n = min(i.numel(), self.chunk)
        if n:
            self._drain(self._depth - 1)
            slot = self._ring.acquire_empty()
            assert slot is not None, "D2H ring exhausted"
            _slot_tensor(slot, n, self.in_dtype).copy_(i[:n])
            check(lib.b2s_ring_submit_full(self._ring.h, slot, n, 0), self.ctx.handle)
            full, valid = C.c_void_p(), C.c_size_t(0)
            check(lib.b2s_ring_acquire_full(self._ring.h, C.byref(full), C.byref(valid)), self.ctx.handle)
            check(lib.b2s_slot_fetch_to_host(full, n), self.ctx.handle)       # async D2H + event
            self._inflight.append((full, n))
            self.input.consume(n)
            self.d2h_bytes += n * self.in_dtype.itemsize
        if self.input.finished() and n == i.numel():
            self._drain(0)
            self._finish()
            io.finished = True

    def _finish(self):
        pass


class VectorSink(_HostSink):
    """blocks::VectorSink (vector_sink.rs:20-70): collects everything it receives; ``items()`` afterwards."""

    def __init__(self, dtype, capacity: int = 0, chunk_items: int = 1 << 20, ctx: Optional[Context] = None):
        super().__init__(dtype, chunk_items, ctx=ctx)
        self._parts: List[np.ndarray] = []

    def _take(self, host):
        self._parts.append(host.copy())

    def items(self) -> np.ndarray:
        return np.concatenate(self._parts) if self._parts else np.zeros(0, self.in_dtype)


class FileSink(_HostSink):
    """blocks::FileSink<T> (file_sink.rs:33-95): raw items appended to ``file_path`` (created / truncated in
    init, :88-91); ``n_written`` counts items like the reference's log line (:80)."""

    def __init__(self, file_path, dtype=np.complex64, chunk_items: int = 1 << 20, ctx: Optional[Context] = None):
        super().__init__(dtype, chunk_items, ctx=ctx)
        self.file_path = os.fspath(file_path)
        self.file = open(self.file_path, "wb")
        self.n_written = 0

    def _take(self, host):
        self.file.write(memoryview(host.view(np.uint8)))
        self.n_written += host.size

    def _finish(self):
        self.file.flush()
        self.file.close()


# ---------------------------------------------------------------------------------------------------
# linear chain driver
# ---------------------------------------------------------------------------------------------------
def run_chain(stages: Sequence[Block], buffer_items: int = 4 << 20, max_rounds: int = 1 << 24, device="cuda"):
    """Connect ``stages[0] -> stages[1] -> ...`` with device stream buffers and call ``work`` round-robin until
    the last stage reports finished.  A stage finishing marks its output stream finished, which is what the
    next stage's ``input.finished()`` reports (the reference's port ``finished`` flag, buffer/mod.rs:295-353).
    Returns the number of work() calls made."""
    assert len(stages) >= 2
    bufs = []
    for up, down in zip(stages[:-1], stages[1:]):
        assert np.dtype(up.out_dtype) == np.dtype(down.in_dtype), \
            f"{type(up).__name__} -> {type(down).__name__}: item types differ"
        b = StreamBuffer(up.out_dtype, buffer_items, device)
        up.output, down.input = _WriterPort(b), _ReaderPort(b)
        bufs.append(b)
    done = [False] * len(stages)
    calls = 0
    for _ in range(max_rounds):
        progressed = False
        for k, st in enumerate(stages):
            if done[k]:
                continue
            before = tuple((b.rd, b.wr) for b in bufs)
            io = WorkIo()
            st.work(io)
            calls += 1
            if io.finished:
                done[k] = True
                if k < len(bufs):
                    bufs[k].writer_finished = True
                progressed = True
            progressed |= before != tuple((b.rd, b.wr) for b in bufs)
        if done[-1]:
            break
        if not progressed:
            raise RuntimeError("run_chain: no stage can make progress (buffer_items too small for a stage's minimum?)")
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize()
    return calls


# ---------------------------------------------------------------------------------------------------
# fan-out / fan-in graph driver
# ---------------------------------------------------------------------------------------------------
def _port_key(p):
    return tuple(p) if isinstance(p, (tuple, list)) else p


def _set_port(blk: Block, port, obj):
    if isinstance(port, tuple):
        getattr(blk, port[0])[port[1]] = obj
    else:
        setattr(blk, port, obj)


class Flowgraph:
    """A graph of blocks joined by device stream buffers, driven like ``run_chain`` (the Mocker idea, not a scheduler:
    the reference's runtime is out of scope, SURVEY.md §8) but with any topology:

      * ``connect(src, "port", dst, "port")``; ports default to ``"output"`` / ``"input"`` (``connect(src, dst)``),
        a port of a list of ports is ``("outputs", k)``.  Item types must agree on every edge.
      * one output port may feed several inputs (``MultiStreamBuffer``); an input port has exactly one writer.
      * finish rules of the reference's block loop (runtime/wrapped_kernel.rs:133-138, :188-191): a block that finishes
        marks each of its output streams finished for the readers (StreamInputDone) and finishes every block writing
        to one of its inputs (StreamOutputDone), even when that writer has other readers.  The run ends when every
        block has finished; a round in which no block moves a cursor, changes state or finishes raises.

    Blocks run round-robin in the order they first appear in ``connect`` calls."""

    def __init__(self):
        self.blocks: List[Block] = []
        self.edges: List[tuple] = []                 # (src, src_port, dst, dst_port)

    def add(self, blk: Block) -> Block:
        if not any(b is blk for b in self.blocks):
            self.blocks.append(blk)
        return blk

    def connect(self, src: Block, *args):
        """connect(src, dst) | connect(src, src_port, dst) | connect(src, dst, dst_port) |
        connect(src, src_port, dst, dst_port)."""
        a = list(args)
        src_port = _port_key(a.pop(0)) if a and not isinstance(a[0], Block) else "output"
        if not a or not isinstance(a[0], Block):
            raise TypeError("Flowgraph.connect: the destination block is missing")
        dst = a.pop(0)
        dst_port = _port_key(a.pop(0)) if a else "input"
        if a:
            raise TypeError("Flowgraph.connect: too many arguments")
        if src_port not in src.stream_outputs():
            raise ValueError(f"{type(src).__name__} has no stream output {src_port!r}")
        if dst_port not in dst.stream_inputs():
            raise ValueError(f"{type(dst).__name__} has no stream input {dst_port!r}")
        if any(d is dst and dp == dst_port for _, _, d, dp in self.edges):
            raise ValueError(f"{type(dst).__name__}.{dst_port} is already connected")
        st, dt = np.dtype(src.port_dtype(src_port)), np.dtype(dst.port_dtype(dst_port))
        if st != dt:
            raise TypeError(f"{type(src).__name__}.{src_port} ({st}) -> {type(dst).__name__}.{dst_port} ({dt}): "
                            "item types differ")
        self.add(src)
        self.add(dst)
        self.edges.append((src, src_port, dst, dst_port))

    def run(self, buffer_items: int = 4 << 20, max_rounds: int = 1 << 24, device="cuda") -> int:
        """Run until every block has finished; returns the number of work() calls made."""
        idx = {id(b): k for k, b in enumerate(self.blocks)}
        for b in self.blocks:
            for p in b.stream_inputs():
                if not any(d is b and dp == p for _, _, d, dp in self.edges):
                    raise ValueError(f"{type(b).__name__}.{p} is not connected")
            for p in b.stream_outputs():
                if not any(s is b and sp == p for s, sp, _, _ in self.edges):
                    raise ValueError(f"{type(b).__name__}.{p} is not connected")
        writers = {}                                 # (src index, port) -> [(dst, dst_port), ...]
        for s, sp, d, dp in self.edges:
            writers.setdefault((idx[id(s)], sp), []).append((d, dp))
        out_bufs = [[] for _ in self.blocks]         # block -> buffers it writes
        in_bufs = [[] for _ in self.blocks]          # block -> (buffer, reader index, writer block index)
        bufs = []
        for (si, sp), readers in writers.items():
            src = self.blocks[si]
            b = MultiStreamBuffer(src.port_dtype(sp), buffer_items, len(readers), device)
            _set_port(src, sp, _WriterPort(b))
            for k, (d, dp) in enumerate(readers):
                _set_port(d, dp, _MultiReaderPort(b, k))
                in_bufs[idx[id(d)]].append((b, k, si))
            out_bufs[si].append(b)
            bufs.append(b)
        done = [False] * len(self.blocks)

        def finish(k):
            if done[k]:
                return
            done[k] = True
            for b in out_bufs[k]:                    # StreamInputDone to every reader
                b.writer_finished = True
            for b, r, w in in_bufs[k]:               # StreamOutputDone to every writer
                b.live[r] = False
                finish(w)

        calls = 0
        for _ in range(max_rounds):
            progressed = False
            for k, blk in enumerate(self.blocks):
                if done[k]:
                    continue
                before = tuple(b.cursors() for b in bufs)
                io = WorkIo()
                blk.work(io)
                calls += 1
                if io.finished:
                    finish(k)
                    progressed = True
                progressed |= io.call_again or before != tuple(b.cursors() for b in bufs)
            if all(done):
                break
            if not progressed:
                stuck = [type(b).__name__ for k, b in enumerate(self.blocks) if not done[k]]
                raise RuntimeError(f"Flowgraph.run: no block can make progress (still running: {stuck})")
        if torch.device(device).type == "cuda":
            torch.cuda.synchronize()
        return calls
