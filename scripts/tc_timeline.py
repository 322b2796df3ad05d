"""Per-CTA timeline of the headline tensor-FIR launch (c32, 256 taps, 64 Mi samples through the ring, as bench.py).

Builds the library with -DB2S_TC_TIMELINE (scripts/build_variant.sh tc_timeline), runs the headline shape and
reads back, after each of --launches launches, the %globaltimer stamps every CTA wrote (fir_tc.cu, TcStamp):
kernel entry, first and last bulk copy issued, first tile's full barrier (+ its MMAs issued), first store, start of
the last tile's store, converter exit and exit.  All figures are fractions of the launch span (first entry to last
exit over all CTAs), averaged over CTAs, median over launches:

  fill        entry of the launch -> the CTA's first bulk copy (no byte of this SM moves)
  first store entry of the launch -> the CTA's first store
  drain       the CTA's last bulk copy -> its exit (no more reads from this SM)
  tail idle   the CTA's exit -> the launch's last exit (the SM has nothing left to do: last wave)
  edge idle   fill + drain + tail idle: the part of the launch in which the SM's read stream is not running

    python scripts/tc_timeline.py [--launches 20] [--lib path/to/libb200sdr_X.so] [--json out.json]

The stamps add a few global stores per CTA; the default build compiles to the same SASS without them.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TL = ["entry", "first_copy", "last_copy", "first_full", "first_store", "last_store", "conv_exit", "exit"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", default=None, help="an already built -DB2S_TC_TIMELINE library (default: build one)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    lib_path = args.lib
    if lib_path is None:
        subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_variant.sh"), "tc_timeline", "-DB2S_TC_TIMELINE"],
                       check=True, stdout=subprocess.DEVNULL)
        lib_path = os.path.join(ROOT, "futuresdr_b200", "variants", "libb200sdr_tc_timeline.so")
    os.environ["B2S_LIB"] = os.path.abspath(lib_path)
    sys.path.insert(0, ROOT)

    import numpy as np
    import torch

    import bench
    import futuresdr_b200 as fb
    from futuresdr_b200._lib import lib
    from futuresdr_b200.shard import ShardedFir

    read = lib.b2s_tc_timeline_read            # only in a -DB2S_TC_TIMELINE build
    read.restype = C.c_int
    read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sh = ShardedFir(bench._taps(), bench.CHUNK, np.complex64, device=dev, algo=fb.ALGO_TENSOR, exchange="peer")
    g = torch.Generator(device=dev).manual_seed(bench.SEED)
    for t in sh.slot_tensors():
        torch.view_as_real(t).normal_(generator=g)
    out = torch.empty(bench.CHUNK, dtype=torch.complex64, device=dev)
    ctas = min(torch.cuda.get_device_properties(dev).multi_processor_count, -(-bench.CHUNK // 8192))
    buf = (C.c_ulonglong * (ctas * len(TL)))()

    for _ in range(args.warmup):
        sh.step(out)
    torch.cuda.synchronize()
    per_launch = []
    for _ in range(args.launches):
        read(buf, ctas)                                      # clear
        sh.step(out)
        torch.cuda.synchronize()
        if read(buf, ctas) != len(TL):
            raise RuntimeError("b2s_tc_timeline_read failed: not a -DB2S_TC_TIMELINE build?")
        s = np.array(buf, dtype=np.float64).reshape(ctas, len(TL))
        if (s == 0).any():
            raise RuntimeError("a CTA left a stamp unwritten")
        t0, t1 = s[:, 0].min(), s[:, 7].max()
        span = t1 - t0
        st = {k: s[:, i] for i, k in enumerate(TL)}
        r = {
            "span_us": span / 1e3,
            "fill": float(np.mean(st["first_copy"] - t0) / span),
            "first_full": float(np.mean(st["first_full"] - t0) / span),
            "first_store": float(np.mean(st["first_store"] - t0) / span),
            "drain": float(np.mean(st["exit"] - st["last_copy"]) / span),
            "tail_idle": float(np.mean(t1 - st["exit"]) / span),
            "entry_skew_max_us": float((st["entry"].max() - t0) / 1e3),
            "exit_spread_us": float((t1 - st["exit"].min()) / 1e3),
        }
        r["edge_idle"] = r["fill"] + r["drain"] + r["tail_idle"]
        per_launch.append(r)
    med = {k: statistics.median(r[k] for r in per_launch) for k in per_launch[0]}
    res = {"gpu": torch.cuda.get_device_name(dev), "launches": args.launches, "ctas": ctas, "median": med,
           "lib": os.path.basename(lib_path)}
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({**res, "per_launch": per_launch}, f, indent=1)


if __name__ == "__main__":
    main()
