"""Kernel time of the quadrature demodulators (Apply QuadDemodC32 and QuadDemod) against a device-to-device copy that
moves the same bytes, measured in one process on 64 Mi samples of the FM receiver benchmark's input signal.

The demodulator reads 8 B and writes 8 B (C32) or 4 B (F32) per sample, so the copy ceiling is a cudaMemcpy of 8 B
(resp. 6 B) per sample: 16 (12) B of HBM traffic per sample either way.  Prints one JSON line per op with the kernel
and copy times (median over rounds of >= 50 back-to-back launches each, CUDA events), their ratio, the SHA-256 of the
output after a reset, and the GPU's name and power limit.  With --out DIR the raw outputs are written there
(demod_c32.bin, demod_f32.bin) for a bitwise comparison between two builds (B2S_LIB=... selects a library).

    python scripts/apply_demod_timing.py [--n 67108864] [--launches 50] [--rounds 5] [--out DIR]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import futuresdr_b200  # noqa: E402
from futuresdr_b200.blocks import Apply, ApplyOp  # noqa: E402


def fm_signal(n, dev):
    """The first n samples of bench.py's configs[2] input: a sinusoidally modulated FM carrier (phase in float64) plus
    white noise at -26 dB, from the same generator seed and in the same 16 Mi-sample segments."""
    x = torch.empty(n, dtype=torch.complex64, device=dev)
    g = torch.Generator(device=dev).manual_seed(0x5EED + 3)
    seg = 16 * 1024 * 1024
    for c0 in range(0, n, seg):
        m = min(seg, n - c0)
        tt = torch.arange(c0, c0 + m, dtype=torch.float64, device=dev)
        ph = (-(0.05 / 0.0007)) * torch.cos(2 * np.pi * 0.0007 * tt)
        xs = torch.view_as_real(x[c0:c0 + m])
        xs.normal_(generator=g)
        xs.mul_(0.05)
        xs[:, 0] += torch.cos(ph).float()
        xs[:, 1] += torch.sin(ph).float()
    return x


def time_ms(fn, launches):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / launches


def power_limit_w(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=64 * 1024 * 1024)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    dev = torch.device("cuda", torch.cuda.current_device())
    gpu = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
           "lib": os.path.relpath(futuresdr_b200._lib.SO_PATH)}
    x = fm_signal(a.n, dev)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    for op, out_dtype, name in ((ApplyOp.QuadDemodC32, torch.complex64, "demod_c32"),
                                (ApplyOp.QuadDemod, torch.float32, "demod_f32")):
        blk = Apply(op)
        out = torch.empty(a.n, dtype=out_dtype, device=dev)
        copy_bytes = a.n * (8 + out.element_size()) // 2
        src = torch.empty(copy_bytes, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        kern, copy = [], []
        for _ in range(a.warmup):
            blk.apply(x, out)
            dst.copy_(src)
        for _ in range(a.rounds):                         # alternate the two so drift in clocks hits both alike
            copy.append(time_ms(lambda: dst.copy_(src), a.launches))
            kern.append(time_ms(lambda: blk.apply(x, out), a.launches))
        blk.reset()
        blk.apply(x, out)
        torch.cuda.synchronize()
        host = out.cpu().numpy()
        if a.out:
            host.tofile(os.path.join(a.out, name + ".bin"))
        k, c = statistics.median(kern), statistics.median(copy)
        print(json.dumps({"op": name, "samples": a.n, "kernel_ms": round(k, 4), "copy_ms": round(c, 4),
                          "ratio": round(k / c, 4), "kernel_ms_rounds": [round(v, 4) for v in kern],
                          "copy_ms_rounds": [round(v, 4) for v in copy], "bytes_per_sample": 8 + out.element_size(),
                          "sha256": hashlib.sha256(host.tobytes()).hexdigest(), **gpu}), flush=True)
        del out, src, dst


if __name__ == "__main__":
    main()
