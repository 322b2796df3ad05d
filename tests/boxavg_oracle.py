"""CPU oracle of the WLAN and M17 receivers' MovingAverage (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/boxavg_oracle.c``, the C restatement of one work() call of
examples/wlan/src/moving_average.rs:67-107 and examples/m17/src/moving_average.rs:41-81, compiled by
``native.load_oracle`` on first use.

``BoxAvgRef.work`` is one reference call; ``BoxAvgRef.run`` emulates what one device exec covers: the calls the
reference makes back to back on what is left of the slices, until a call makes no progress or ``max_calls`` calls have
run.  ``np_work`` is an independent numpy float32 transcription of one call, for cross-checking the C file.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_szp = C.POINTER(C.c_size_t)
_ip = C.POINTER(C.c_int)
MAX_ITER = 4000

SIGNATURES = {
    "orc_boxavg_work_f32": (C.c_int, [C.c_size_t, C.c_int, C.c_float, _szp, _f32p, C.c_size_t, C.c_int, _f32p,
                                      C.c_size_t, _szp, _szp, _ip, _ip]),
    "orc_boxavg_work_c32": (C.c_int, [C.c_size_t, _szp, _f32p, C.c_size_t, C.c_int, _f32p, C.c_size_t, _szp, _szp,
                                      _ip, _ip]),
}


def lib() -> C.CDLL:
    return load_oracle("boxavg_oracle", SIGNATURES)


@dataclass
class Call:
    consumed: int
    produced: int
    call_again: bool
    finished: bool
    out: np.ndarray


@dataclass
class Exec:
    consumed: int
    produced: int
    calls: int
    call_again: bool
    done: bool
    out: np.ndarray


class BoxAvgRef:
    """MovingAverage<f32> / MovingAverage<Complex32> (wlan) or m17::MovingAverage (f32, ``divisor=4800.0``)."""

    def __init__(self, dtype, length: int, divisor=None):
        self.dtype = np.dtype(dtype)
        assert self.dtype in (np.dtype(np.float32), np.dtype(np.complex64))
        assert divisor is None or self.dtype == np.float32
        self.len = int(length)
        assert self.len > 0
        self.divisor = divisor
        self.pad = self.len - 1

    def work(self, x, out_cap: int, finished: bool = True) -> Call:
        x = np.ascontiguousarray(np.asarray(x, self.dtype).reshape(-1))
        out = np.zeros(max(min(out_cap, max(self.pad, MAX_ITER)), 1), self.dtype)    # a call writes no more
        pad = C.c_size_t(self.pad)
        c, p, ca, fin = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_int(0)
        xp = x.ctypes.data_as(_f32p) if x.size else C.cast(C.c_void_p(0), _f32p)
        if self.dtype == np.float32:
            rc = lib().orc_boxavg_work_f32(self.len, self.divisor is not None, float(self.divisor or 1.0),
                                           C.byref(pad), xp, x.size, int(finished), out.ctypes.data_as(_f32p),
                                           out_cap, C.byref(c), C.byref(p), C.byref(ca), C.byref(fin))
        else:
            rc = lib().orc_boxavg_work_c32(self.len, C.byref(pad), xp, x.size, int(finished),
                                           out.ctypes.data_as(_f32p), out_cap, C.byref(c), C.byref(p), C.byref(ca),
                                           C.byref(fin))
        assert rc == 0
        self.pad = pad.value
        return Call(c.value, p.value, bool(ca.value), bool(fin.value), out[: p.value].copy())

    def run(self, x, out_cap: int, max_calls: int = 0) -> Exec:
        """One device exec: calls back to back on the remaining slices until one makes no progress or max_calls
        (0: no limit) have run.  ``done`` is the last call's finish rule with the input taken as finished."""
        x = np.asarray(x, self.dtype).reshape(-1)
        c = p = calls = 0
        outs = []
        last = None
        while max_calls == 0 or calls < max_calls:
            last = self.work(x[c:], out_cap - p, True)
            calls += 1
            c += last.consumed
            p += last.produced
            outs.append(last.out)
            if last.produced == 0:
                break
        out = np.concatenate(outs) if outs else np.zeros(0, self.dtype)
        return Exec(c, p, calls, bool(last and last.call_again), bool(last and last.finished), out)


def np_work(dtype, length: int, divisor, pad: int, x, out_cap: int, finished: bool = True):
    """numpy float32 transcription of one work() call -> (pad, consumed, produced, call_again, finished, out)."""
    dtype = np.dtype(dtype)
    x = np.asarray(x, dtype).reshape(-1)
    if pad > 0:
        m = min(pad, out_cap)
        return pad - m, 0, m, m < out_cap, False, np.zeros(m, dtype)
    avail = max(x.size + 1 - length, 0)
    m = min(MAX_ITER, avail, out_cap)
    out = np.zeros(m, dtype)
    if m > 0:
        comps = [x.view(np.float32)] if dtype == np.float32 else [x.real.copy(), x.imag.copy()]
        res = []
        for comp in comps:
            with np.errstate(all="ignore"):
                res.append(_chain(comp, length, m, divisor, dtype == np.float32))
        if dtype == np.float32:
            out = res[0]
        else:
            out.real, out.imag = res[0], res[1]
    return pad, m, m, False, bool(finished and m == avail), out


def _chain(comp, length, m, divisor, neg_zero):
    """One component's running sum: the fold of the prefix from -0.0 (f32) or +0.0 (Complex32), then m steps."""
    f32 = np.float32
    s = f32(-0.0) if neg_zero else f32(0.0)
    for k in range(length - 1):
        s = f32(s + comp[k])
    o = np.zeros(m, np.float32)
    for i in range(m):
        s = f32(s + comp[i + length - 1])
        o[i] = f32(s / f32(divisor)) if divisor is not None else s
        s = f32(s - comp[i])
    return o


def replay(dtype, length: int, divisor, stream, execs):
    """The outputs of a block whose execs saw the slices ``execs`` = [(n_in, n_out_cap, max_calls), ...] of the input
    ``stream``, each slice starting where the previous execs' consumption left it.  Returns (outputs, per-exec
    (consumed, produced))."""
    ref = BoxAvgRef(dtype, length, divisor)
    stream = np.asarray(stream, np.dtype(dtype))
    pos, outs, counts = 0, [], []
    for n_in, cap, mc in execs:
        e = ref.run(stream[pos:pos + n_in], cap, mc)
        pos += e.consumed
        outs.append(e.out)
        counts.append((e.consumed, e.produced))
    return (np.concatenate(outs) if outs else np.zeros(0, np.dtype(dtype))), counts
