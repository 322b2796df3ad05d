"""CPU tests of the host side the record-producing blocks share (futuresdr_b200.blocks): the record reader, driven by a
fake drain function in place of a block's b2s_*_drain_* call, and the payload batch of the transmitters' push and
encode calls."""
import ctypes as C

import numpy as np
import pytest

from futuresdr_b200._lib import B200SdrError, EINVAL
from futuresdr_b200.blocks import LORA_BURST, _payload_batch, _Records

_DRAIN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t))
_H = 0x5EED


class _FakeList:
    """A block's record list as its drain call hands it out: up to ``cap`` queued records per call, oldest first.
    ``fail_at`` makes that call (counting from 1) return EINVAL."""

    def __init__(self, fail_at=None):
        self.queue, self.added = np.zeros(0, LORA_BURST), 0
        self.calls, self.fail_at = 0, fail_at
        self.fn = _DRAIN(self._drain)

    def add(self, n):
        self.queue = np.concatenate([self.queue, _bursts(self.added, n)])
        self.added += n

    def _drain(self, h, host, cap, n):
        assert h == _H
        self.calls += 1
        if self.calls == self.fail_at:
            return EINVAL
        k = min(cap, self.queue.size)
        C.memmove(host, self.queue.ctypes.data, k * LORA_BURST.itemsize)
        self.queue = self.queue[k:].copy()
        n[0] = k
        return 0


def _bursts(start, n):
    r = np.zeros(n, LORA_BURST)
    r["index"] = np.arange(start, start + n)
    r["len"] = 3 * r["index"] + 1
    return r


def test_no_records_read_as_an_empty_array_of_the_record_type():
    fake = _FakeList()
    out = _Records(fake.fn, LORA_BURST).read(_H, None)
    assert out.dtype == LORA_BURST and out.size == 0
    assert fake.calls == 1


def test_a_read_over_several_chunks_returns_every_record_in_order():
    fake = _FakeList()
    n = 3 * _Records.chunk + 5
    fake.add(n)
    out = _Records(fake.fn, LORA_BURST).read(_H, None)
    assert np.array_equal(out, _bursts(0, n))
    assert fake.calls == 4


def test_reads_are_cumulative_and_clear_empties_them():
    fake = _FakeList()
    rec = _Records(fake.fn, LORA_BURST)
    fake.add(10)
    assert np.array_equal(rec.read(_H, None), _bursts(0, 10))
    fake.add(7)
    assert np.array_equal(rec.read(_H, None), _bursts(0, 17))
    assert np.array_equal(rec.read(_H, None), _bursts(0, 17))
    rec.clear()
    out = rec.read(_H, None)
    assert out.dtype == LORA_BURST and out.size == 0
    fake.add(4)
    assert np.array_equal(rec.read(_H, None), _bursts(17, 4))


def test_a_failed_drain_raises_and_keeps_the_records_drained_before_it():
    fake = _FakeList(fail_at=2)
    rec = _Records(fake.fn, LORA_BURST)
    fake.add(_Records.chunk + 3)
    with pytest.raises(B200SdrError):
        rec.read(_H, None)
    assert np.array_equal(rec.read(_H, None), _bursts(0, _Records.chunk + 3))


def test_payload_batch():
    data, buf, lens = _payload_batch(["hé", b"\x00\x01", b"", bytearray(b"xyz"), np.arange(4, dtype=np.uint8)])
    assert data == ["hé".encode(), b"\x00\x01", b"", b"xyz", b"\x00\x01\x02\x03"]
    assert buf == b"".join(data)
    assert lens._type_ is C.c_size_t and list(lens) == [3, 2, 0, 3, 4]
    data, buf, lens = _payload_batch([])
    assert data == [] and buf == b""
    assert lens._type_ is C.c_size_t and list(lens) == [0]            # one element: a valid pointer for n = 0
