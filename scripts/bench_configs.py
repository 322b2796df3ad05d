"""Secondary measurements for the non-headline BASELINE configs (parity-tested elsewhere; these
are NOT bench.py lines): per-kernel device-resident throughput with CUDA events, reported as
Msamples/s (input samples) and algorithmic GB/s vs the HBM peak.

    python scripts/bench_configs.py [--quick]
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import futuresdr_b200 as fb  # noqa: E402
from futuresdr_b200 import blocks as B  # noqa: E402

PEAK = 3350.0   # H100 SXM data-sheet HBM3 bandwidth (GB/s), used without MEASURED_PEAKS.json
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def report(name, n_in, bytes_alg, sec, extra=""):
    gbs = bytes_alg / sec / 1e9
    print(json.dumps({"kernel": name, "Msamples_s": round(n_in / sec / 1e6, 1), "ms": round(sec * 1e3, 4),
                      "alg_GBs": round(gbs, 1), "frac_hbm": round(gbs / PEAK, 4), "note": extra}), flush=True)


def want(section):
    """--only a,b,c runs just the named sections (fir, f32, chain, fft, resamp, next, iir, sigsrc, stream, boxavg, adsb,
    zigbee, keyfob, ssb, lora, wlan, zigbee_tx, scale)."""
    for i, a in enumerate(sys.argv):
        if a == "--only" and i + 1 < len(sys.argv):
            return section in sys.argv[i + 1].split(",")
    return True


def iir_section(quick):
    """IirFilter: SCAN on 64 Mi samples per call, DIRECT (sequential, bit-exact) on 1 Mi, and the oracle's one-thread
    rate (the recurrence cannot be split across host threads).  8 B/sample of HBM traffic (4 in, 4 out)."""
    from scipy import signal
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import iir_oracle as orc
    n = (16 if quick else 64) << 20
    bb, aa = signal.butter(2, 0.1)
    b6, a6 = signal.butter(6, 0.1)
    poles = 0.9 * np.exp(1j * np.linspace(0.3, 2.8, 3))
    a7 = -np.real(np.poly(np.concatenate([poles, poles.conj(), [0.5]])))[1:]
    shapes = {"biquad": (-aa[1:], bb), "dc_blocker": ([0.995], [1.0, -1.0]), "butter6": (-a6[1:], b6),
              "na7_nb1": (a7, [1.0])}
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n + 64, generator=g, device="cuda")
    y = torch.empty(n + 64, device="cuda")
    for name, (a, b) in shapes.items():
        f = fb.IirFilter(np.float32(a), np.float32(b), np.float32, algo=fb.ALGO_SCAN)
        sec = timeit(lambda: f.filter(x[: n + len(b) - 1], y[:n]), iters=10, warm=3)
        report(f"iir_scan_{name}", n, 8 * n, sec, extra=f"Gsamples_s={n / sec / 1e9:.2f}")
    nd = 1 << 20
    for name, (a, b) in shapes.items():
        f = fb.IirFilter(np.float32(a), np.float32(b), np.float32, algo=fb.ALGO_DIRECT)
        sec = timeit(lambda: f.filter(x[: nd + len(b) - 1], y[:nd]), iters=3, warm=1)
        report(f"iir_direct_{name}", nd, 8 * nd, sec, extra=f"Gsamples_s={nd / sec / 1e9:.4f}")
    x64 = torch.randn(nd + 64, dtype=torch.float64, generator=g, device="cuda")
    y64 = torch.empty(nd + 64, dtype=torch.float64, device="cuda")
    f = fb.IirFilter(-aa[1:], bb, np.float64)
    sec = timeit(lambda: f.filter(x64[: nd + 2], y64[:nd]), iters=3, warm=1)
    report("iir64_direct_biquad", nd, 16 * nd, sec, extra=f"Gsamples_s={nd / sec / 1e9:.4f}")
    xc = x[:nd].cpu().numpy()
    orc.lib()                                   # compile the oracle outside the timed window
    for name, (a, b) in shapes.items():
        t0 = time.perf_counter()
        orc.iir(np.float32(a), np.float32(b), xc)
        sec = time.perf_counter() - t0
        report(f"iir_oracle_1thread_{name}", nd, 8 * nd, sec, extra=f"CPU, one thread; Gsamples_s={nd / sec / 1e9:.4f}")


def sigsrc_section(quick):
    """SignalSource: 64 Mi items per call, write-only traffic (4 B/sample f32, 8 B/sample Complex32) against the
    3.35 TB/s data-sheet figure.  fs/64 is in the set because its increment (2^26) puts neighbouring samples 16 table
    entries apart, the stride that would collapse an unpadded shared-memory table onto one bank; fs/4 makes every
    lane of a warp read the same entry.  The oracle's one-thread CPU rate is given for context."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import sigsrc_oracle as orc
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"kernel": "sigsrc_device", "gpu": q[torch.cuda.current_device()] if q else "unknown"}), flush=True)
    n = (16 if quick else 64) << 20
    fs = 48000.0
    freqs = {"1k": 1000.0, "48k": 48000.0, "fs4": fs / 4, "fs64": fs / 64}
    cases = [("f32_sin", fb.SignalWave.Sin, np.float32), ("c32_sin", fb.SignalWave.Sin, np.complex64),
             ("c32_square", fb.SignalWave.Square, np.complex64)]
    out = {np.float32: torch.empty(n, dtype=torch.float32, device="cuda"),
           np.complex64: torch.empty(n, dtype=torch.complex64, device="cuda")}
    for name, wave, dt in cases:
        bps = np.dtype(dt).itemsize
        for fname, f in freqs.items():
            src = fb.SignalSource(wave, f, fs, 0.5, 0.0, dt)
            sec = timeit(lambda: src.generate(out[dt]), iters=20, warm=3)
            gbs = bps * n / sec / 1e9
            print(json.dumps({"kernel": f"sigsrc_{name}_{fname}", "items": n, "ms": round(sec * 1e3, 4),
                              "Gsamples_s": round(n / sec / 1e9, 2), "bytes_written": bps * n,
                              "write_GBs": round(gbs, 1), "frac_3350GBs": round(gbs / 3350.0, 4)}), flush=True)
    nc = 4 << 20
    for name, wave, dt in cases:
        ref = orc.Source(int(wave), 1000.0, fs, 0.5, 0.0, dt)
        ref.work(1024)                              # compile the oracle outside the timed window
        t0 = time.perf_counter()
        ref.work(nc)
        sec = time.perf_counter() - t0
        print(json.dumps({"kernel": f"sigsrc_oracle_1thread_{name}", "items": nc,
                          "Gsamples_s": round(nc / sec / 1e9, 4), "note": "CPU, one thread"}), flush=True)


def stream_section(quick):
    """Combine / Split / StreamDuplicator / StreamDeinterleaver kernels on 64 Mi items per call, as fractions of the
    3.35 TB/s data-sheet figure computed from algorithmic bytes; the numpy restatement on one CPU thread beside each;
    and the WLAN receiver front end (rx.rs:73-93) as an end-to-end graph rate through edges.Flowgraph."""
    import subprocess
    import ctypes as C
    from futuresdr_b200 import _lib
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"kernel": "stream_device", "gpu": q[torch.cuda.current_device()] if q else "unknown"}), flush=True)
    n = (16 if quick else 64) << 20
    nc = 4 << 20
    g = torch.Generator(device="cuda").manual_seed(5)
    ctx = fb.default_context().handle

    def line(name, nbytes, sec, cpu_sec):
        gbs = nbytes / sec / 1e9
        print(json.dumps({"kernel": name, "items": n, "ms": round(sec * 1e3, 4), "Gitems_s": round(n / sec / 1e9, 2),
                          "alg_GBs": round(gbs, 1), "frac_3350GBs": round(gbs / 3350.0, 4),
                          "cpu_1thread_Gitems_s": round(nc / cpu_sec / 1e9, 4)}), flush=True)

    def cpu_time(fn):
        fn()
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    c64 = lambda m: torch.view_as_complex(torch.randn(m, 2, generator=g, device="cuda"))  # noqa: E731
    a, b = c64(n), c64(n)
    bf = torch.rand(n, generator=g, device="cuda") + 0.5
    oc = torch.empty(n, dtype=torch.complex64, device="cuda")
    of = torch.empty(n, device="cuda")
    ha, hb, hf = a[:nc].cpu().numpy(), b[:nc].cpu().numpy(), bf[:nc].cpu().numpy()
    cb, cp = C.c_size_t(0), C.c_size_t(0)

    def comb(op, x, y, o):
        return lambda: _lib.lib.b2s_combine_exec(ctx, op, C.c_void_p(x.data_ptr()), n, C.c_void_p(y.data_ptr()), n,
                                                 C.c_void_p(o.data_ptr()), n, C.byref(cb), C.byref(cp))

    def np_conj_mul():
        r = np.empty(nc, np.complex64)
        r.real = ha.real * hb.real - ha.imag * (-hb.imag)
        r.imag = ha.real * (-hb.imag) + ha.imag * hb.real
    sec = timeit(comb(_lib.COMBINE_CONJ_MUL_C32, a, b, oc), iters=20, warm=3)
    line("combine_conj_mul_c32", 24 * n, sec, cpu_time(np_conj_mul))
    sec = timeit(comb(_lib.COMBINE_MAG_DIV_C32_F32, a, bf, of), iters=20, warm=3)
    line("combine_mag_div_c32_f32", 16 * n, sec, cpu_time(lambda: np.hypot(ha.real, ha.imag) / hf))
    o1 = torch.empty(n, device="cuda")
    sec = timeit(lambda: _lib.lib.b2s_split_exec(ctx, _lib.SPLIT_RE_IM, C.c_void_p(a.data_ptr()), n,
                                                 C.c_void_p(of.data_ptr()), C.c_void_p(o1.data_ptr()), n, C.byref(cb),
                                                 C.byref(cp)), iters=20, warm=3)
    line("split_re_im", 16 * n, sec, cpu_time(lambda: (ha.real.copy(), ha.imag.copy())))
    del o1
    for dt, s in ((torch.float32, 4), (torch.complex64, 8)):
        src = (torch.randn(n, generator=g, device="cuda") if dt == torch.float32 else a)
        hsrc = src[:nc].cpu().numpy()
        for N in (2, 4):
            outs = [torch.empty(n, dtype=dt, device="cuda") for _ in range(N)]
            ptrs = (C.c_void_p * N)(*[o.data_ptr() for o in outs])
            sec = timeit(lambda: _lib.lib.b2s_fanout_exec(ctx, 0, s, C.c_void_p(src.data_ptr()), n, ptrs, N, n,
                                                          C.byref(cb), C.byref(cp)), iters=10, warm=2)
            line(f"duplicate_{'f32' if s == 4 else 'c32'}_N{N}", (1 + N) * s * n, sec,
                 cpu_time(lambda: [hsrc.copy() for _ in range(N)]))
            del outs
        for N in (2, 4, 16, 256):
            per = n // N
            outs = [torch.empty(per, dtype=dt, device="cuda") for _ in range(N)]
            ptrs = (C.c_void_p * N)(*[o.data_ptr() for o in outs])
            sec = timeit(lambda: _lib.lib.b2s_fanout_exec(ctx, 1, s, C.c_void_p(src.data_ptr()), per * N, ptrs, N, per,
                                                          C.byref(cb), C.byref(cp)), iters=10, warm=2)
            line(f"deinterleave_{'f32' if s == 4 else 'c32'}_N{N}", 2 * s * per * N, sec,
                 cpu_time(lambda: [hsrc[k::N].copy() for k in range(N)]))
            del outs
    del a, b, bf, oc, of
    torch.cuda.empty_cache()
    # whole graph, end to end: source stream already on the device is not possible through VectorSource, so the rate
    # includes the host -> device copy of the source and the device -> host copies of the sink
    from futuresdr_b200.blocks import Apply, ApplyOp, Fir
    from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource
    ns = (4 if quick else 16) << 20
    x = (np.random.default_rng(0).standard_normal(2 * ns).astype(np.float32).view(np.complex64))
    best = None
    for _ in range(3):
        fg = Flowgraph()
        src, delay = VectorSource(x), fb.Delay(np.complex64, 16)
        mag2, mult = Apply(ApplyOp.NormSqr), fb.Combine(fb.CombineOp.ConjMulC32)
        favg = Fir(fb.FirFilter(np.ones(64, np.float32), sample_dtype=np.float32))
        cavg = Fir(fb.FirFilter(np.ones(48, np.float32), sample_dtype=np.complex64))
        div, snk = fb.Combine(fb.CombineOp.MagDivC32F32), VectorSink(np.float32)
        for args in ((src, delay), (src, mag2), (src, mult, "in0"), (delay, mult, "in1"), (mag2, favg),
                     (mult, cavg), (cavg, div, "in0"), (favg, div, "in1"), (div, snk)):
            fg.connect(*args)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "wlan_rx_front_end_graph", "items": ns, "s": round(best, 4),
                      "Gsamples_s_end_to_end": round(ns / best / 1e9, 4),
                      "note": "whole graph, end to end: VectorSource H2D + Delay + NormSqr + 2 FIR + 2 Combine + "
                              "VectorSink D2H, driven by edges.Flowgraph from Python"}), flush=True)


def boxavg_section(quick):
    """The WLAN / M17 MovingAverage (csrc/boxavg.cu) on 64 Mi items per exec: f32 len 64, c32 len 48 (the WLAN rx
    shapes) and f32 len 4800 / 4800 (M17), as fractions of the 3.35 TB/s data-sheet figure computed from algorithmic
    bytes (input + output once each); the C oracle on one thread beside each; and the WLAN receiver front end with the
    real MovingAverage blocks as an end-to-end graph rate through edges.Flowgraph."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from boxavg_oracle import BoxAvgRef
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"kernel": "boxavg_device", "gpu": q[torch.cuda.current_device()] if q else "unknown"}), flush=True)
    n = (16 if quick else 64) << 20
    nc = 4 << 20
    g = torch.Generator(device="cuda").manual_seed(7)
    for dt, length, div in ((np.float32, 64, None), (np.complex64, 48, None), (np.float32, 4800, 4800.0)):
        cplx = dt == np.complex64
        x = (torch.view_as_complex(torch.randn(n, 2, generator=g, device="cuda")) if cplx
             else torch.randn(n, generator=g, device="cuda"))
        o = torch.empty_like(x)
        blk = fb.MovingAverage(dt, length, div)
        blk.average(x, o)                                        # the pad: later execs are all sums

        def run():
            blk.average(x, o)
        sec = timeit(run, iters=20, warm=3)
        nbytes = 2 * x.element_size() * (n + 1 - length)
        gbs = nbytes / sec / 1e9
        hx = x[:nc].cpu().numpy()
        ref = BoxAvgRef(dt, length, div)
        ref.pad = 0
        t0 = time.perf_counter()
        ref.run(hx, nc)
        cpu = time.perf_counter() - t0
        name = f"boxavg_{'c32' if cplx else 'f32'}_len{length}" + ("_div" if div else "")
        print(json.dumps({"kernel": name, "items": n, "ms": round(sec * 1e3, 4), "Gitems_s": round(n / sec / 1e9, 2),
                          "alg_GBs": round(gbs, 1), "frac_3350GBs": round(gbs / 3350.0, 4),
                          "cpu_oracle_1thread_Gitems_s": round(nc / cpu / 1e9, 4)}), flush=True)
        del x, o, blk
        torch.cuda.empty_cache()
    from futuresdr_b200.blocks import Apply, ApplyOp
    from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource
    ns = (4 if quick else 16) << 20
    x = (np.random.default_rng(0).standard_normal(2 * ns).astype(np.float32).view(np.complex64))
    best = None
    for _ in range(3):
        fg = Flowgraph()
        src, delay = VectorSource(x), fb.Delay(np.complex64, 16)
        mag2, mult = Apply(ApplyOp.NormSqr), fb.Combine(fb.CombineOp.ConjMulC32)
        favg, cavg = fb.MovingAverage(np.float32, 64), fb.MovingAverage(np.complex64, 48)
        div, snk = fb.Combine(fb.CombineOp.MagDivC32F32), VectorSink(np.float32)
        for args in ((src, delay), (src, mag2), (src, mult, "in0"), (delay, mult, "in1"), (mag2, favg),
                     (mult, cavg), (cavg, div, "in0"), (favg, div, "in1"), (div, snk)):
            fg.connect(*args)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "wlan_rx_front_end_graph_moving_average", "items": ns, "s": round(best, 4),
                      "Gsamples_s_end_to_end": round(ns / best / 1e9, 4),
                      "note": "whole graph, end to end: VectorSource H2D + Delay + NormSqr + 2 MovingAverage + "
                              "2 Combine + VectorSink D2H, driven by edges.Flowgraph from Python"}), flush=True)


def adsb_section(quick):
    """The ADS-B detector / demodulator (csrc/adsb.cu) on 64 Mi positions per exec, with sparse triggers and with a
    trigger at every position, as fractions of the 3.35 TB/s data-sheet figure from 12 B of algorithmic bytes per
    position (three f32 reads); and the receive front end (listen_adsb.rs:85-120) end to end through edges.Flowgraph."""
    import subprocess
    from futuresdr_b200 import adsb
    from futuresdr_b200.edges import Flowgraph, VectorSource
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"kernel": "adsb_device", "gpu": q[torch.cuda.current_device()] if q else "unknown"}), flush=True)
    n = (16 if quick else 64) << 20
    g = torch.Generator(device="cuda").manual_seed(11)
    s = torch.rand(n, generator=g, device="cuda")
    nf = torch.rand(n, generator=g, device="cuda") + 0.25
    for name, density in (("sparse", 1e-4), ("every_position", 1.0)):
        hit = torch.rand(n, generator=g, device="cuda") < density
        corr = torch.where(hit, nf * 20.0, nf * 5.0)
        blk = fb.AdsbDemod(10.0)

        def run():
            blk.reset()                                          # lists restart: no growth inside the timing
            blk.exec(s, nf, corr)
        sec = timeit(run, iters=20, warm=3)
        gbs = 12 * n / sec / 1e9
        n_det = blk.detections().size
        print(json.dumps({"kernel": f"adsb_{name}", "positions": n, "detections": int(n_det),
                          "ms": round(sec * 1e3, 4), "alg_GBs": round(gbs, 1), "frac_3350GBs": round(gbs / 3350.0, 4)}),
              flush=True)
        del corr, blk
    del s, nf
    torch.cuda.empty_cache()
    ns = (4 if quick else 16) << 20
    x = (np.random.default_rng(0).standard_normal(2 * ns).astype(np.float32).view(np.complex64))
    best = None
    for _ in range(3):
        fg = Flowgraph()
        src = VectorSource(x)
        fg.add(src)
        adsb.front_end(fg, src, 4_000_000)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "adsb_rx_front_end_graph", "items": ns, "s": round(best, 4),
                      "Gsamples_s_end_to_end": round(ns / best / 1e9, 4),
                      "note": "whole graph, end to end: VectorSource H2D + resampler + NormSqr + 2 FIR + AdsbDemod, "
                              "driven by edges.Flowgraph from Python"}), flush=True)


def zigbee_section(quick):
    """The ZigBee receive chain (csrc/apply.cu DcBlockF32, csrc/zigbee.cu ClockRecoveryMm and ZigbeeDecoder) at 64 Mi
    items per exec in Msamples/s, each serial kernel also as SM cycles per step at the card's maximum SM clock; the
    front end (rx.rs:66-92) end to end through edges.Flowgraph; and the C oracle of each stage on one CPU thread."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import zigbee_oracle as zo
    from futuresdr_b200 import zigbee
    from futuresdr_b200.edges import Flowgraph, VectorSource
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "zigbee_device", "gpu": gpu}), flush=True)
    try:
        mhz = float(gpu.split(",")[2].split()[0])
    except Exception:
        mhz = float("nan")
    n = (16 if quick else 64) << 20
    rng = np.random.default_rng(0)
    ph = torch.from_numpy((np.sin(np.arange(n) * 0.7) * 1.2 + 0.3 * rng.standard_normal(n)).astype(np.float32)).cuda()
    out = torch.empty(n, device="cuda")

    def line(name, items, sec, steps=None):
        d = {"kernel": f"zigbee_{name}", "items": items, "ms": round(sec * 1e3, 3),
             "Msamples_s": round(items / sec / 1e6, 2)}
        if steps is not None:
            d["steps"] = steps
            d["cycles_per_step_at_max_sm_clock"] = round(sec * mhz * 1e6 / steps, 2)
        print(json.dumps(d), flush=True)

    dc = B.Apply(B.ApplyOp.DcBlockF32, zigbee.DC_ALPHA)
    line("dc_block", n, timeit(lambda: dc.apply(ph, out), iters=3, warm=1), n)
    mm = B.ClockRecoveryMm(zigbee.MM_OMEGA, zigbee.MM_GAIN_OMEGA, zigbee.MM_MU, zigbee.MM_GAIN_MU,
                           zigbee.MM_OMEGA_RELATIVE_LIMIT)
    mm.exec(ph[:1 << 20], out)
    best, produced, clocks = None, 0, []
    import threading
    stop = threading.Event()

    def sample():                                                # the SM clock while the one-CTA kernel runs
        while not stop.wait(0.25):
            r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm",
                                "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.strip()
            if r.isdigit():
                clocks.append(int(r))
    th = threading.Thread(target=sample)
    th.start()
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c, produced = mm.exec(ph, out)                           # synchronises
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    stop.set()
    th.join()
    line("clock_recovery_mm", n, best, produced)
    if clocks:
        med = float(np.median(clocks))
        print(json.dumps({"kernel": "zigbee_clock_recovery_mm_sm_clock", "samples": len(clocks), "median_mhz": med,
                          "min_mhz": min(clocks), "max_mhz": max(clocks),
                          "cycles_per_step_at_median_clock": round(best * med * 1e6 / produced, 2)}), flush=True)
    dec = B.ZigbeeDecoder(zigbee.DECODER_THRESHOLD)
    noise = torch.randn(n, device="cuda")
    pre = zo.chips_of(bytes(4))[:256]
    dense = torch.from_numpy(np.where(np.resize(pre, n) > 0, 1.0, -1.0).astype(np.float32)).cuda()
    for name, x in (("decoder_noise", noise), ("decoder_all_preamble", dense)):
        def run():
            dec.reset()
            dec.exec(x)
        line(name, n, timeit(run, iters=5, warm=1))
    del noise, dense, ph, out
    torch.cuda.empty_cache()
    ns = (4 if quick else 16) << 20
    x = (np.random.default_rng(1).standard_normal(2 * ns).astype(np.float32).view(np.complex64))
    best = None
    for _ in range(3):
        fg = Flowgraph()
        src = VectorSource(x)
        fg.add(src)
        zigbee.front_end(fg, src)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "zigbee_rx_front_end_graph", "items": ns, "s": round(best, 4),
                      "Msamples_s_end_to_end": round(ns / best / 1e6, 2),
                      "note": "whole graph, end to end: VectorSource H2D + QuadDemod + DcBlockF32 + ClockRecoveryMm + "
                              "ZigbeeDecoder, driven by edges.Flowgraph from Python"}), flush=True)
    m = 4 << 20
    xs = (np.sin(np.arange(m) * 0.7) * 1.2 + 0.3 * rng.standard_normal(m)).astype(np.float32)
    t0 = time.perf_counter()
    zo.DcBlock(zigbee.DC_ALPHA).work(xs)
    t1 = time.perf_counter()
    zo.Mm(zigbee.MM_OMEGA, zigbee.MM_GAIN_OMEGA, zigbee.MM_MU, zigbee.MM_GAIN_MU,
          zigbee.MM_OMEGA_RELATIVE_LIMIT).work(xs, m)
    t2 = time.perf_counter()
    zo.Decoder(zigbee.DECODER_THRESHOLD).work(rng.standard_normal(m).astype(np.float32))
    t3 = time.perf_counter()
    for name, sec in (("dc_block", t1 - t0), ("clock_recovery_mm", t2 - t1), ("decoder_noise", t3 - t2)):
        print(json.dumps({"kernel": f"zigbee_oracle_cpu_1thread_{name}", "items": m, "ms": round(sec * 1e3, 2),
                          "Msamples_s": round(m / sec / 1e6, 2)}), flush=True)


def keyfob_section(quick):
    """The keyfob receive chain (csrc/apply.cu SliceF32U8, csrc/keyfob.cu KeyfobDecoder) at 64 Mi items per exec: the
    slicer as a fraction of 3.35 TB/s at 5 B per item, the decoder on all zeros, on the slicer output of noise and on
    the densest valid-pulse stream as items/s and as a fraction of 3.35 TB/s at 1 B per item; the front end
    (main.rs:39-79) end to end through edges.Flowgraph; and the C oracle on one CPU thread."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import keyfob_oracle as ko
    from futuresdr_b200 import keyfob
    from futuresdr_b200.edges import Flowgraph, VectorSource
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "keyfob_device", "gpu": gpu}), flush=True)
    n = (16 if quick else 64) << 20
    peak = 3.35e12

    def line(name, items, sec, bytes_per_item):
        print(json.dumps({"kernel": f"keyfob_{name}", "items": items, "ms": round(sec * 1e3, 3),
                          "Gitems_s": round(items / sec / 1e9, 2),
                          "frac_of_3p35_TBs": round(items * bytes_per_item / sec / peak, 3)}), flush=True)

    x = torch.randn(n, device="cuda")
    u = torch.empty(n, dtype=torch.uint8, device="cuda")
    sl = B.Apply(B.ApplyOp.SliceF32U8)
    line("slicer", n, timeit(lambda: sl.apply(x, u), iters=10, warm=2), 5)
    lp = torch.from_numpy(np.convolve(np.random.default_rng(2).standard_normal(n + 127).astype(np.float32),
                                      keyfob.lowpass_taps(), "valid").astype(np.float32)).cuda()
    noise = torch.empty(n, dtype=torch.uint8, device="cuda")
    sl.apply(lp, noise)
    del x, lp
    zeros = torch.zeros(n, dtype=torch.uint8, device="cuda")
    dense = torch.from_numpy(np.resize(np.repeat(np.array([0, 1], np.uint8), 63), n)).cuda()
    dec = B.KeyfobDecoder()
    for name, s in (("decoder_zeros", zeros), ("decoder_noise_slicer", noise), ("decoder_dense_63", dense)):
        def run():
            dec.reset()
            dec.exec(s)
        line(name, n, timeit(run, iters=10, warm=2), 1)
    del zeros, noise, dense, u
    torch.cuda.empty_cache()
    ns = (4 if quick else 16) << 20
    xc = (np.random.default_rng(1).standard_normal(2 * ns).astype(np.float32).view(np.complex64))
    best = None
    for _ in range(3):
        fg = Flowgraph()
        src = VectorSource(xc)
        fg.add(src)
        keyfob.front_end(fg, src)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "keyfob_rx_front_end_graph", "items": ns, "s": round(best, 4),
                      "Msamples_s_end_to_end": round(ns / best / 1e6, 2),
                      "note": "whole graph at 4 Msps in: VectorSource H2D + resampler 1/16 + NormSqr + DcBlockF32 + "
                              "128-tap FIR + SliceF32U8 + KeyfobDecoder, driven by edges.Flowgraph from Python"}),
          flush=True)
    m = 16 << 20
    xs = np.random.default_rng(3).standard_normal(m).astype(np.float32)
    ys = np.convolve(xs, keyfob.lowpass_taps(), "same").astype(np.float32)
    t0 = time.perf_counter()
    bits = ko.slice_u8(ys)
    t1 = time.perf_counter()
    ko.Decoder().work(bits)
    t2 = time.perf_counter()
    ko.Decoder().work(np.resize(np.repeat(np.array([0, 1], np.uint8), 63), m))
    t3 = time.perf_counter()
    for name, sec in (("slicer", t1 - t0), ("decoder_noise_slicer", t2 - t1), ("decoder_dense_63", t3 - t2)):
        print(json.dumps({"kernel": f"keyfob_oracle_cpu_1thread_{name}", "items": m, "ms": round(sec * 1e3, 2),
                          "Msamples_s": round(m / sec / 1e6, 2)}), flush=True)


def ssb_section(quick):
    """The SSB transceiver's device closures at 64 Mi items per exec: each oscillator mixer (csrc/rotator.cu) as kernel
    time (torch.profiler, the record ring filled before the exec) and as sustained exec time (host clock over back-to-
    back execs, paced by the host replay of the recurrence), the record H2D copies, Apply(DivC32) and
    ApplyNM(C32ToI16Iq) (csrc/apply.cu); fractions of 3.35 TB/s from algorithmic bytes (a mixer: 8 B in, 8 or 4 B out
    and 1 B of records per sample).  Then the receive graph (receive.rs:54-87) end to end from a FileSource, and the C
    oracle on one CPU thread."""
    import subprocess
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ssb_oracle as so
    from futuresdr_b200 import ssb
    from futuresdr_b200.edges import FileSource, Flowgraph, VectorSink
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "ssb_device", "gpu": gpu}), flush=True)
    n = (16 if quick else 64) << 20
    peak = 3.35e12

    def line(name, items, sec, bytes_per_item, **extra):
        print(json.dumps({"kernel": f"ssb_{name}", "items": items, "ms": round(sec * 1e3, 3),
                          "Gitems_s": round(items / sec / 1e9, 3),
                          "frac_of_3p35_TBs": round(items * bytes_per_item / sec / peak, 3), **extra}), flush=True)

    def device_us(prof, needle):
        tot, cnt = 0.0, 0
        for e in prof.key_averages():
            if needle in e.key:
                tot += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                cnt += e.count
        return tot, cnt

    x = torch.view_as_complex(torch.randn(n, 2, device="cuda"))
    for op, out_b in ((B.MixOp.RotateC32, 8), (B.MixOp.RotateScaleC32, 8), (B.MixOp.WeaverF32, 4)):
        o = torch.empty(n, dtype=torch.float32 if op == B.MixOp.WeaverF32 else torch.complex64, device="cuda")
        m = B.Mixer(op, float(ssb.xlating_phase()), 0.5)
        m.mix(x[:1 << 20], o[:1 << 20])                          # warm-up (module load, record buffers)
        torch.cuda.synchronize()
        m.reset()
        time.sleep(0.5)                                          # the worker fills its 32 Mi-sample ring meanwhile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.mix(x, o)
            torch.cuda.synchronize()
        k_us, k_n = device_us(prof, "rotator_kernel")
        c_us, c_n = device_us(prof, "Memcpy HtoD")
        line(f"mixer_{op.name}_kernel", n, k_us * 1e-6, 8 + out_b + 1, launches=k_n,
             records_h2d_ms=round(c_us * 1e-3, 3), h2d_copies=c_n)
        execs = 2 if quick else 4
        m.mix(x, o)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(execs):
            m.mix(x, o)
        torch.cuda.synchronize()
        line(f"mixer_{op.name}_sustained", n, (time.perf_counter() - t0) / execs, 8 + out_b + 1,
             note="exec rate with the replay worker running: paced by the host recurrence, not by the GPU")
        m.close()
        del o
    y = torch.empty_like(x)
    div = B.Apply(B.ApplyOp.DivC32, 0.0001)
    line("apply_DivC32", n, timeit(lambda: div.apply(x, y), iters=10, warm=2), 16)
    del y
    q16 = torch.empty(2 * n, dtype=torch.int16, device="cuda")
    conv = B.ApplyNM(B.ApplyNMOp.C32ToI16Iq, 0.9)
    line("applynm_C32ToI16Iq", n, timeit(lambda: conv.apply(x, q16), iters=10, warm=2), 12)
    q16u = q16[1:]                                               # output 2-byte but not 4-byte aligned
    line("applynm_C32ToI16Iq_out_unaligned", n - 1, timeit(lambda: conv.apply(x[:n - 1], q16u), iters=10, warm=2), 12)
    del x, q16, q16u
    torch.cuda.empty_cache()
    ns = (4 if quick else 16) << 20
    xc = (np.random.default_rng(1).standard_normal(2 * ns).astype(np.float32) * 5000).view(np.complex64)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ssb_lsb_256k.dat")
        xc.tofile(path)
        for rate in (48_000, 8_000):
            best = None
            for _ in range(2):
                fg = Flowgraph()
                src = FileSource(path, np.complex64, repeat=False, chunk_items=1 << 20)
                fg.add(src)
                b = ssb.receiver(fg, src, rate)
                fg.connect(b["weaver"], VectorSink(np.float32))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fg.run(buffer_items=4 << 20)
                sec = time.perf_counter() - t0
                best = sec if best is None else min(best, sec)
            print(json.dumps({"kernel": f"ssb_rx_graph_{rate // 1000}k", "items": ns, "s": round(best, 4),
                              "Msamples_s_end_to_end": round(ns / best / 1e6, 2),
                              "note": "FileSource (256 kHz c32 file) + xlating mixer + resampler + Weaver mixer + "
                                      "VectorSink, driven by edges.Flowgraph from Python"}), flush=True)
    m = 16 << 20
    xs = xc[:m]
    for name, fn in (("mixer_RotateC32", lambda: so.Mixer(so.ROTATE, 0.1).work(xs)),
                     ("mixer_RotateScaleC32", lambda: so.Mixer(so.ROTATE_SCALE, 0.1, 1e-4).work(xs)),
                     ("mixer_WeaverF32", lambda: so.Mixer(so.WEAVER, 0.1, 0.5).work(xs)),
                     ("file_level", lambda: so.file_level(xs)), ("to_i16_iq", lambda: so.to_i16_iq(xs))):
        t0 = time.perf_counter()
        fn()
        sec = time.perf_counter() - t0
        print(json.dumps({"kernel": f"ssb_oracle_cpu_1thread_{name}", "items": m, "ms": round(sec * 1e3, 2),
                          "Msamples_s": round(m / sec / 1e6, 2)}), flush=True)


def lora_section(quick):
    """The LoRa transmitter (csrc/lora.cu): the modulator over many queued frames as kernel time (CUDA events around one
    exec that produces every queued sample) in Gsamples/s and as a fraction of 3.35 TB/s at 8 B/sample written; one SF7
    frame in cycles per sample at the SM clock nvidia-smi reports as the maximum; the device encoder in frames/s; the C
    oracle (encode + modulate with libm) on one CPU thread; and the transmit graph into a VectorSink end to end."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import lora_oracle as lo
    from futuresdr_b200 import lora
    from futuresdr_b200.edges import Flowgraph, VectorSink
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "lora_device", "gpu": gpu}), flush=True)
    try:
        mhz = float(gpu.split(",")[2].split()[0])
    except (IndexError, ValueError):
        mhz = float("nan")
    rng = np.random.default_rng(7)
    peak = 3.35e12

    def modulate_rate(name, n_frames, sf, os_, payload_len, reps):
        tx = B.LoraTransmitter(sf, 1, True, sf >= 11, False, os_, (8, 16), 8, 0)
        pays = [rng.integers(0, 256, payload_len, dtype=np.uint8).tobytes() for _ in range(n_frames)]
        tx.push(*pays)
        total = tx.pending()
        out = torch.empty(total, dtype=torch.complex64, device="cuda")
        best = None
        for r in range(reps + 1):
            if r:
                tx.push(*pays)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            tx.exec(out)
            e1.record()
            torch.cuda.synchronize()
            sec = e0.elapsed_time(e1) * 1e-3
            if r:                                             # the first exec warms up (module load)
                best = sec if best is None else min(best, sec)
        print(json.dumps({"kernel": f"lora_modulate_{name}", "frames": n_frames, "samples": total,
                          "ms": round(best * 1e3, 3), "Gsamples_s": round(total / best / 1e9, 3),
                          "frac_of_3p35_TBs": round(total * 8 / best / peak, 3),
                          "cycles_per_sample_per_chain": round(best * mhz * 1e6 / (total / n_frames), 2)}),
              flush=True)
        tx.close()
        del out
        torch.cuda.empty_cache()

    modulate_rate("4096x_sf7_os4_16B", 4096, 7, 4, 16, 2 if quick else 5)
    modulate_rate("1024x_sf7_os4_16B", 1024, 7, 4, 16, 2 if quick else 5)
    modulate_rate("256x_sf12_os8_255B", 256 if not quick else 32, 12, 8, 255, 1 if quick else 2)
    modulate_rate("1x_sf7_os4_16B", 1, 7, 4, 16, 5)
    modulate_rate("1x_sf7_os1_255B", 1, 7, 1, 255, 5)
    nf = 4096 if quick else 65536
    pays = [rng.integers(0, 256, 64, dtype=np.uint8).tobytes() for _ in range(nf)]
    lora.encode(pays[:16], 7, 1, True, False, False)
    torch.cuda.synchronize()
    best = None
    for _ in range(3):
        t0 = time.perf_counter()
        lora.encode(pays, 7, 1, True, False, False)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "lora_encode_64B_sf7_cr1", "frames": nf, "ms": round(best * 1e3, 3),
                      "frames_s": round(nf / best, 1), "note": "host clock: upload, one launch, synchronise"}),
          flush=True)
    t0 = time.perf_counter()
    for p in pays[:1000]:
        lo.encode(p, 7, 1, True, False, False)
    sec = time.perf_counter() - t0
    print(json.dumps({"kernel": "lora_oracle_cpu_1thread_encode_64B", "frames_s": round(1000 / sec, 1)}), flush=True)
    sym = lo.encode(pays[0][:16], 7, 1, True, False, False)
    t0 = time.perf_counter()
    out, _ = lo.modulate(sym, 7, 4, (8, 16), 8, 0)
    sec = time.perf_counter() - t0
    print(json.dumps({"kernel": "lora_oracle_cpu_1thread_modulate_sf7_os4", "samples": out.size,
                      "Msamples_s": round(out.size / sec / 1e6, 2)}), flush=True)
    n_graph = 256 if quick else 2048
    best = None
    for _ in range(2):
        fg = Flowgraph()
        tx = lora.transmitter(fg, sf=lora.SpreadingFactor.SF7, os_factor=4)
        sink = VectorSink(np.complex64)
        fg.connect(tx, sink)
        tx.push(*[rng.integers(0, 256, 16, dtype=np.uint8).tobytes() for _ in range(n_graph)])
        total = tx.pending()
        tx.finish()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "lora_tx_graph_sf7_os4_16B", "frames": n_graph, "samples": total,
                      "s": round(best, 4), "Msamples_s_end_to_end": round(total / best / 1e6, 2),
                      "note": "LoraTransmitter + VectorSink (D2H to host memory) driven by edges.Flowgraph"}),
          flush=True)


def wlan_section(quick):
    """The WLAN transmitter (csrc/wlan.cu): the OFDM exec kernel over 4096 queued frames of 1500 bytes at BPSK 1/2 and
    64-QAM 3/4 with pads of 5000 (tx.rs) as kernel time (CUDA events around one exec that produces every queued sample),
    in Gsamples/s and as a fraction of 3.35 TB/s at 8 B/sample written; the same exec cut into 1 Mi-sample execs; the
    device encoder in frames/s; and the transmit graph into a VectorSink end to end."""
    import subprocess
    from futuresdr_b200 import wlan
    from futuresdr_b200.edges import Flowgraph, VectorSink
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "wlan_device", "gpu": gpu}), flush=True)
    rng = np.random.default_rng(8)
    peak = 3.35e12
    nf = 512 if quick else 4096
    pays = [rng.integers(0, 256, 1500, dtype=np.uint8).tobytes() for _ in range(nf)]

    def exec_rate(name, mcs, reps, cap=None):
        tx = B.WlanTransmitter(wlan.SRC_MAC, wlan.DST_MAC, wlan.BSS_MAC, int(mcs), 5000, 5000)
        tx.push(*pays)
        total = tx.pending()
        out = torch.empty(total, dtype=torch.complex64, device="cuda")
        best = None
        for r in range(reps + 1):
            if r:
                tx.push(*pays)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            if cap is None:
                tx.exec(out)
            else:
                for o in range(0, total, cap):
                    tx.exec(out[o:o + cap])
            e1.record()
            torch.cuda.synchronize()
            sec = e0.elapsed_time(e1) * 1e-3
            if r:                                             # the first exec warms up (module load)
                best = sec if best is None else min(best, sec)
        print(json.dumps({"kernel": f"wlan_exec_{name}", "frames": nf, "samples": total,
                          "execs": 1 if cap is None else -(-total // cap), "ms": round(best * 1e3, 3),
                          "Gsamples_s": round(total / best / 1e9, 3),
                          "frac_of_3p35_TBs": round(total * 8 / best / peak, 3)}), flush=True)
        tx.close()
        del out
        torch.cuda.empty_cache()

    exec_rate(f"{nf}x1500B_bpsk12_pad5000", wlan.Mcs.BPSK_1_2, 2 if quick else 5)
    exec_rate(f"{nf}x1500B_qam64_34_pad5000", wlan.Mcs.QAM64_3_4, 2 if quick else 5)
    exec_rate(f"{nf}x1500B_qam64_34_pad5000_1Mi_execs", wlan.Mcs.QAM64_3_4, 2 if quick else 3, cap=1 << 20)
    for mcs in (wlan.Mcs.BPSK_1_2, wlan.Mcs.QAM64_3_4):
        wlan.encode(pays[:16], mcs)
        torch.cuda.synchronize()
        best = None
        for _ in range(3):
            t0 = time.perf_counter()
            wlan.encode(pays, mcs)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            best = sec if best is None else min(best, sec)
        print(json.dumps({"kernel": f"wlan_encode_1500B_{mcs.name.lower()}", "frames": nf, "ms": round(best * 1e3, 3),
                          "frames_s": round(nf / best, 1), "note": "host clock: upload, three launches, synchronise"}),
              flush=True)
    n_graph = 128 if quick else 1024
    best = None
    for _ in range(2):
        fg = Flowgraph()
        tx = wlan.transmitter(fg, default_mcs=wlan.Mcs.QAM16_1_2)
        sink = VectorSink(np.complex64)
        fg.connect(tx, sink)
        tx.push(*pays[:n_graph])
        total = tx.pending()
        tx.finish()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "wlan_tx_graph_qam16_12_1500B_pad5000", "frames": n_graph, "samples": total,
                      "s": round(best, 4), "Msamples_s_end_to_end": round(total / best / 1e6, 2),
                      "note": "WlanTransmitter + VectorSink (D2H to host memory) driven by edges.Flowgraph"}),
          flush=True)


def zigbee_tx_section(quick):
    """The ZigBee transmitter (csrc/zigbee_tx.cu): the exec kernel as kernel time (CUDA events around the execs that
    produce every queued sample, 64 Mi samples per exec) in Gsamples/s and as a fraction of 3.35 TB/s at 8 B/sample
    written, over 4096 frames of 116 bytes at the reference's pad of 40000 (mostly zero stores) and at pad 0 (all
    body), and the pad-40000 stream in 1 Mi-sample execs; push in frames/s for 4096-frame batches; and, end to end, the
    transmit graph into a VectorSink and the transceiver loop into the receive front end."""
    import subprocess
    from futuresdr_b200 import zigbee
    from futuresdr_b200.edges import Flowgraph, VectorSink
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[torch.cuda.current_device()] if q else "unknown"
    print(json.dumps({"kernel": "zigbee_tx_device", "gpu": gpu}), flush=True)
    rng = np.random.default_rng(9)
    peak = 3.35e12
    nf = 512 if quick else 4096
    pays = [rng.integers(0, 256, 116, dtype=np.uint8).tobytes() for _ in range(nf)]

    def exec_rate(name, pad, reps, cap):
        tx = B.ZigbeeTransmitter(pad)
        tx.push(*pays)
        total = tx.pending()
        out = torch.empty(min(total, cap), dtype=torch.complex64, device="cuda")
        best = None
        for r in range(reps + 1):
            if r:
                tx.push(*pays)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(0, total, cap):
                tx.exec(out)
            e1.record()
            torch.cuda.synchronize()
            sec = e0.elapsed_time(e1) * 1e-3
            if r:                                             # the first pass warms up (module load)
                best = sec if best is None else min(best, sec)
        print(json.dumps({"kernel": f"zigbee_tx_exec_{name}", "frames": nf, "samples": total,
                          "execs": -(-total // cap), "ms": round(best * 1e3, 3),
                          "Gsamples_s": round(total / best / 1e9, 3),
                          "frac_of_3p35_TBs": round(total * 8 / best / peak, 3)}), flush=True)
        tx.close()
        del out
        torch.cuda.empty_cache()

    reps = 2 if quick else 5
    exec_rate(f"{nf}x116B_pad40000", 40000, reps, 64 << 20)
    exec_rate(f"{nf}x116B_pad0", 0, reps, 64 << 20)
    exec_rate(f"{nf}x116B_pad40000_1Mi_execs", 40000, reps, 1 << 20)
    tx = B.ZigbeeTransmitter()
    tx.push(*pays[:16])
    best = None
    for _ in range(5):
        tx.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tx.push(*pays)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "zigbee_tx_push_116B", "frames": nf, "ms": round(best * 1e3, 3),
                      "frames_s": round(nf / best, 1), "note": "host clock: framing, FCS, upload, synchronise"}),
          flush=True)
    tx.close()
    n_graph = 64 if quick else 512
    best = None
    for _ in range(2):
        fg = Flowgraph()
        tx = zigbee.transmitter(fg)
        sink = VectorSink(np.complex64)
        fg.connect(tx, sink)
        tx.push(*pays[:n_graph])
        total = tx.pending()
        tx.finish()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fg.run(buffer_items=4 << 20)
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    print(json.dumps({"kernel": "zigbee_tx_graph_116B_pad40000", "frames": n_graph, "samples": total,
                      "s": round(best, 4), "Msamples_s_end_to_end": round(total / best / 1e6, 2),
                      "note": "ZigbeeTransmitter + VectorSink (D2H to host memory) driven by edges.Flowgraph"}),
          flush=True)
    n_loop = 16 if quick else 64
    fg = Flowgraph()
    tx = zigbee.transmitter(fg)
    b = zigbee.front_end(fg, tx)
    tx.push(*pays[:n_loop])
    total = tx.pending()
    tx.finish()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fg.run(buffer_items=1 << 20)
    sec = time.perf_counter() - t0
    fr = b["decoder"].frames()
    print(json.dumps({"kernel": "zigbee_trx_loop_116B_pad40000", "frames": n_loop, "samples": total,
                      "decoded_crc_ok": int(fr["crc_ok"].sum()), "s": round(sec, 4),
                      "Msamples_s_end_to_end": round(total / sec / 1e6, 2),
                      "note": "ZigbeeTransmitter -> QuadDemod -> DcBlockF32 -> ClockRecoveryMm -> ZigbeeDecoder"}),
          flush=True)


def main():
    quick = "--quick" in sys.argv
    n = (16 if quick else 64) * 1024 * 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.view_as_complex(torch.randn(n + 4096, 2, generator=g, device="cuda"))
    y = torch.empty(n + 4096, dtype=torch.complex64, device="cuda")
    rng = np.random.default_rng(7)
    import oracle as orc
    xr = torch.view_as_real(x).reshape(-1)[: 2 * n]
    yr = torch.view_as_real(y).reshape(-1)[: 2 * n]

    if want("fir"):
        # FIR tap sweep, direct vs tensor
        for ntaps in (8, 16, 32, 64, 128, 256):
            taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
            for algo, nm in ((fb.ALGO_DIRECT, "direct"), (fb.ALGO_TENSOR, "tensor")):
                if algo == fb.ALGO_TENSOR and ntaps < 16:
                    continue
                f = fb.FirFilter(taps, algo=algo)
                sec = timeit(lambda: f.filter(x[: n + ntaps - 1], y[:n]))
                report(f"fir_c32_{ntaps}taps_{nm}", n, 16 * n, sec)
        # 1024-tap (config 5 per-GPU kernel)
        taps = rng.uniform(-1, 1, 1024).astype(np.float32)
        f = fb.FirFilter(taps)
        nn = n // 4
        sec = timeit(lambda: f.filter(x[: nn + 1023], y[:nn]), iters=3, warm=1)
        report("fir_c32_1024taps_auto", nn, 16 * nn, sec, extra=f"algo={f.algo}")
    if want("fir1024") and not want("fir"):
        taps = rng.uniform(-1, 1, 1024).astype(np.float32)
        f = fb.FirFilter(taps)
        nn = n // 4
        sec = timeit(lambda: f.filter(x[: nn + 1023], y[:nn]), iters=3, warm=1)
        report("fir_c32_1024taps_auto", nn, 16 * nn, sec, extra=f"algo={f.algo}")
    if want("fft4096") and not want("fft"):
        fft = B.Fft(4096)
        sec = timeit(lambda: fft.transform(x[:n], y[:n]))
        report("fft_4096_fwd", n, 16 * n, sec)
    if want("demod") and not want("chain"):
        n4 = n // 4
        dem = B.Apply(B.ApplyOp.QuadDemodC32)
        z = torch.empty(n4, dtype=torch.complex64, device="cuda")
        sec = timeit(lambda: dem.apply(y[:n4], z))
        report("quad_demod_c32", n4, 16 * n4, sec)
    if want("fused"):
        # fused rows of round 2: spectrum pipe in one pass, channelizer in one launch
        for N in (2048, 4096):
            sp = B.SpectrumPipe(N, 0.1, 3)
            po = torch.empty(n // 3 + 2 * N, dtype=torch.float32, device="cuda")
            sec = timeit(lambda: sp.process(x[:n], po), iters=5, warm=2)
            report(f"spectrum_pipe_fused_{N}", n, 8 * n + 4 * (n // 3), sec, extra="FFT + |x|^2 + MovingAvg(0.1, 3): spectrum_kernel + scan + fixup")
        for N, T in ((64, 16), (16, 16), (256, 8), (64, 12)):         # 64 x 12: padded to 16 taps
            ctaps = (orc.kaiser_lowpass(0.4 / N, 0.1 / N, 1e-3)).astype(np.float32)
            ctaps = np.resize(ctaps, N * T)
            ch = B.PfbChannelizer(N, ctaps, 1.0)
            ch.reserve_outputs(n // N + 8)
            ch.input.set(x[:n])
            ch.work(B.WorkIo())                               # window fill

            def run_ch():
                ch.input.pos, ch.produced = 0, 0
                ch.work(B.WorkIo())
            sec = timeit(run_ch, iters=5, warm=1)
            report(f"pfb_channelizer_fused_{N}ch_{T}taps", n, 16 * n, sec, extra="FIR bank + IFFT + transposed store in one launch")
    if want("synth"):
        for N, T in ((64, 16), (16, 16), (64, 12)):                    # 64 x 12: padded to 16 taps
            staps = np.resize((orc.kaiser_lowpass(0.4 / N, 0.1 / N, 1e-3)).astype(np.float32), N * T)
            syn = B.PfbSynthesizer(N, staps)
            nv = n // N
            xin = x[:N * nv].view(N, nv)
            syn.set_inputs(xin[:, :4 * T])                    # window fill
            syn.output.reserve(8 * T * N)
            syn.work(B.WorkIo())
            syn.set_inputs(xin)
            syn.output.reserve(n + 2 * N)

            def run_syn():
                syn.in_pos, syn.output.len = 0, 0
                syn.work(B.WorkIo())
            sec = timeit(run_syn, iters=5, warm=1)
            report(f"pfb_synthesizer_{N}ch_{T}taps", n, 16 * n, sec, extra="gather + IFFT + FIR bank")
    if want("f32"):
        # f32 x f32 64 taps (perf/fir config-1 kernel)
        xr = torch.view_as_real(x).reshape(-1)[: 2 * n]
        yr = torch.view_as_real(y).reshape(-1)[: 2 * n]
        t64 = rng.random(64).astype(np.float32)
        for algo, nm in ((fb.ALGO_DIRECT, "direct"), (fb.ALGO_TENSOR, "tensor")):
            f = fb.FirFilter(t64, sample_dtype=np.float32, algo=algo)
            sec = timeit(lambda: f.filter(xr, yr[: 2 * n - 63]))
            report(f"fir_f32_64taps_{nm}", 2 * n, 8 * 2 * n, sec)

    if want("chain"):
        # config 3 pieces: decimator /4 (52 taps) -> quad demod -> PfbArb 0.768
        dec = B.FirBuilder.decimating(4)
        sec = timeit(lambda: dec.filter.filter(x[:n], y[: n // 4]))
        report("decim4_52taps_c32", n, 8 * n + 8 * (n // 4), sec, extra=f"algo={dec.filter.algo}")
        dtaps = fb.firdes.kaiser.lowpass(0.25, 0.1, 1e-4)
        decd = fb.DecimatingFirFilter(4, dtaps, algo=fb.ALGO_DIRECT)
        sec = timeit(lambda: decd.filter(x[:n], y[: n // 4]))
        report("decim4_52taps_c32_direct", n, 8 * n + 8 * (n // 4), sec)
        n4 = n // 4
        dem = B.Apply(B.ApplyOp.QuadDemodC32)
        z = torch.empty(n4, dtype=torch.complex64, device="cuda")
        sec = timeit(lambda: dem.apply(y[:n4], z))
        report("quad_demod_c32", n4, 16 * n4, sec)
        demf = B.Apply(B.ApplyOp.QuadDemod)
        zf = torch.empty(n4, dtype=torch.float32, device="cuda")
        sec = timeit(lambda: demf.apply(y[:n4], zf))
        report("quad_demod_f32", n4, 12 * n4, sec)
        import oracle as orc
        ptaps = (orc.kaiser_lowpass(0.4 / 32, 0.1 / 32, 1e-3) * 32).astype(np.float32)[: 32 * 16]
        pfb = B.PfbArbResampler(0.768, ptaps, 32)
        w = torch.empty(int(n4 * 0.8) + 1024, dtype=torch.complex64, device="cuda")

        def run_pfb():
            pfb.input.set(z)
            pfb.output.data, pfb.output.len = w, 0
            io = B.WorkIo()
            pfb.work(io)
            if io.call_again:
                pfb.input.data = z
                pfb.input.pos = pfb.input.pos
                pfb.work(B.WorkIo())
        t0 = time.perf_counter()
        sec = timeit(run_pfb, iters=3, warm=1)
        report("pfbarb_0.768_32x16", n4, 8 * n4 + 8 * int(n4 * 0.768), sec, extra="includes the host timing-recurrence replay")

    if want("fft"):
        # config 4: FFT 4096
        for nfft_size in (64, 1024, 2048, 4096, 8192, 16384):
            fft = B.Fft(nfft_size)
            sec = timeit(lambda: fft.transform(x[:n], y[:n]))
            report(f"fft_{nfft_size}_fwd", n, 16 * n, sec)
        fft = B.Fft.with_options(4096, B.FftDirection.Forward, True, 1.0 / 4096)
        sec = timeit(lambda: fft.transform(x[:n], y[:n]))
        report("fft_4096_fwd_shift_norm", n, 16 * n, sec)
    if want("resamp"):
        # rational resampler 3/2 (72 taps) and 48/125
        for L, M in ((3, 2), (48, 125)):
            r = B.FirBuilder.resampling(L, M)
            cap = n // 4 * L // M + L
            sec = timeit(lambda: r.filter.filter(x[: n // 4], y[:cap]), iters=5)
            report(f"resamp_{L}_{M}_c32", n // 4, 8 * (n // 4) + 8 * ((n // 4) * L // M), sec)
    if want("next"):
        # SURVEY §8f rows: XlatingFir, PfbChannelizer, spectrum pipe
        xl = B.XlatingFir(4, 1000.0, 48000.0)
        nx = n // 4

        def run_xl():
            c, p, st = xl.filter.filter(x[:nx], y[: nx // 4])
            xl.rotator.rotate_inplace(y[:p])
        sec = timeit(run_xl, iters=3, warm=1)
        report("xlating_fir_d4_52taps", nx, 8 * nx + 8 * (nx // 4), sec, extra="includes the host replay of the rotator recurrence")
        ctaps = (orc.kaiser_lowpass(0.4 / 64, 0.1 / 64, 1e-3)).astype(np.float32)[: 64 * 16]
        ch = B.PfbChannelizer(64, ctaps, 1.0)
        ch.reserve_outputs(n // 64 + 8)
        ch.input.set(x[:n])
        ch.work(B.WorkIo())                                   # window fill

        def run_ch():
            ch.input.pos, ch.produced = 0, 0
            ch.work(B.WorkIo())
        sec = timeit(run_ch, iters=5, warm=1)
        report("pfb_channelizer_64ch_16taps", n, 16 * n, sec, extra="FIR bank + 64-pt IFFT + transpose (3 kernels)")
        fft2 = B.Fft.with_options(2048, B.FftDirection.Forward, True, None)
        mag = B.Apply(B.ApplyOp.NormSqr)
        keep = B.MovingAvg(2048, 0.1, 3)
        pw = torch.empty(n, dtype=torch.float32, device="cuda")
        po = torch.empty(n // 3 + 4096, dtype=torch.float32, device="cuda")

        def run_spec():
            fft2.transform(x[:n], y[:n])
            mag.apply(y[:n], pw)
            keep.input.set(pw)
            keep.output.data, keep.output.len = po, 0
            keep.work(B.WorkIo())
        sec = timeit(run_spec, iters=5, warm=1)
        report("spectrum_pipe_fft2048_normsqr_mavg", n, 8 * n + 4 * (n // 3), sec, extra="unfused: 3 kernels, 32 B/sample of HBM traffic")
    if want("iir"):
        iir_section(quick)
    if want("sigsrc"):
        sigsrc_section(quick)
    if want("stream"):
        stream_section(quick)
    if want("boxavg"):
        boxavg_section(quick)
    if want("adsb"):
        adsb_section(quick)
    if want("zigbee"):
        zigbee_section(quick)
    if want("keyfob"):
        keyfob_section(quick)
    if want("ssb"):
        ssb_section(quick)
    if want("lora"):
        lora_section(quick)
    if want("wlan"):
        wlan_section(quick)
    if want("zigbee_tx"):
        zigbee_tx_section(quick)
    if want("scale"):
        # element-wise scale (the Vulkan/wgpu shader)
        sc = B.Apply(B.ApplyOp.ScaleF32, 12.0)
        sec = timeit(lambda: sc.apply(xr, yr))
        report("scale_f32_x12", 2 * n, 8 * 2 * n, sec)


if __name__ == "__main__":
    main()
