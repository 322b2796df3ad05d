"""Tensor vs CUDA-core FIR on SMALL slices (the perf/fir regime: 1 M samples per call): where does the tensor kernel's
fixed cost (Toeplitz fill, one persistent CTA per SM) stop paying?  Prints microseconds per call."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import futuresdr_b200 as fb

def timeit(fn, iters=200, warm=20):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3

rng = np.random.default_rng(1)
for dtype, td in ((np.float32, torch.float32), (np.complex64, torch.complex64)):
    for ntaps in (32, 64, 128, 256):
        taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
        ft = fb.FirFilter(taps, sample_dtype=dtype, algo=fb.ALGO_TENSOR)
        fd = fb.FirFilter(taps, sample_dtype=dtype, algo=fb.ALGO_DIRECT)
        row = []
        for n in (1 << 14, 1 << 16, 1 << 18, 1 << 20, 1 << 22, 1 << 24):
            x = torch.randn(n + ntaps - 1, device="cuda").to(td)
            y = torch.empty(n, dtype=td, device="cuda")
            a = timeit(lambda: ft.filter(x, y)); b = timeit(lambda: fd.filter(x, y))
            row.append(f"n=2^{n.bit_length()-1}: tc {a:.1f} / direct {b:.1f} us")
        print(np.dtype(dtype).name, ntaps, " | ".join(row), flush=True)
