"""Parity of the wgmma (tensor-core, split-bf16) FIR against the oracle, through the C ABI.
Same tolerance as the direct path: |y - y_ref| <= 1e-5 * ||taps||_1 * max|x|."""
import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fb():
    import futuresdr_b200 as fb
    return fb


def _noise(rng, n, cplx=True):
    if cplx:
        return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    return rng.standard_normal(n).astype(np.float32)


def _check(fb, rng, ntaps, n, cplx, cap=None, taps=None):
    import torch
    x = _noise(rng, n, cplx)
    if taps is None:
        taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
    f = fb.FirFilter(taps, sample_dtype=x.dtype, algo=fb.ALGO_TENSOR)
    assert f.algo == fb.ALGO_TENSOR
    cap = n if cap is None else cap
    xd = torch.from_numpy(x).cuda()
    yd = torch.full((max(cap, 1),), 3.0, dtype=xd.dtype, device="cuda")[:cap]
    c, p, st = f.filter(xd, yd)
    torch.cuda.synchronize()
    c0, p0, s0, ref = orc.fir(taps, x, cap)
    assert (c, p, int(st)) == (c0, p0, s0)
    if p:
        tol = 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
        assert np.max(np.abs(yd[:p].cpu().numpy() - ref)) <= tol


@pytest.mark.parametrize("ntaps", [16, 17, 31, 64, 128, 129, 130, 200, 256, 257])
@pytest.mark.parametrize("cplx", [True, False])
def test_tensor_fir_parity(fb, rng, ntaps, cplx):
    _check(fb, rng, ntaps, 30000 + ntaps, cplx)


def test_tensor_fir_ragged(fb, rng):
    for n in (256, 257, 300, 4096 + 255, 4097 + 255, 8192 + 254, 123457):
        for cap in (n, 1, 4095, 4096, 4097):
            _check(fb, rng, 256, n, True, cap=cap)
    for n in (8192 + 255, 8193 + 255, 70001):
        _check(fb, rng, 256, n, False)


def test_tensor_fir_many_tiles_multiwave(fb, rng):
    # > 132 SMs x 4 stages of tiles: exercises the stage / accumulator ring wrap-around
    _check(fb, rng, 256, 4096 * 1500 + 255 + 17, True)
    _check(fb, rng, 100, 8192 * 700 + 99 + 5, False)


def test_tensor_fir_kaiser_taps_and_impulse(fb, rng):
    taps = orc.kaiser_lowpass(0.1, 0.02, 1e-4)[:257]
    _check(fb, rng, taps.size, 50000, True, taps=taps.astype(np.float32))
    # impulse response == reversed taps placement (exact in bf16 split: 1.0 is exact)
    import torch
    n, ntaps = 9000, 256
    t = rng.uniform(-1, 1, ntaps).astype(np.float32)
    x = np.zeros(n, np.complex64); x[5000] = 1.0 + 0.5j
    f = fb.FirFilter(t, algo=fb.ALGO_TENSOR)
    yd = torch.zeros(n, dtype=torch.complex64, device="cuda")
    c, p, st = f.filter(torch.from_numpy(x).cuda(), yd)
    _, _, _, ref = orc.fir(t, x, n)
    assert np.max(np.abs(yd[:p].cpu().numpy() - ref)) <= 2.0 ** -17   # taps: g_hi + g_lo leaves <= 2^-18 relative


def test_tensor_unsupported_shapes_are_refused(fb):
    with pytest.raises(fb.B200SdrError):       # decimation must divide 128 (the kept output phases are lane-static)
        fb.DecimatingFirFilter(3, np.ones(64, np.float32), algo=fb.ALGO_TENSOR)
    assert fb.DecimatingFirFilter(4, np.ones(64, np.float32), algo=fb.ALGO_TENSOR).algo == fb.ALGO_TENSOR
    ramp = lambda n: np.linspace(0.1, 1.0, n).astype(np.float32)
    assert fb.DecimatingFirFilter(4, ramp(52)).algo == fb.ALGO_TENSOR      # FirBuilder::decimating(4)
    assert fb.DecimatingFirFilter(5, ramp(52)).algo == fb.ALGO_DIRECT
    # AUTO keeps CONSTANT tap vectors (boxcar / moving average) on the CUDA cores: their split-bf16 errors are coherent
    assert fb.DecimatingFirFilter(4, np.ones(52, np.float32)).algo == fb.ALGO_DIRECT
    with pytest.raises(fb.B200SdrError):
        fb.FirFilter(np.ones(64, np.complex64), algo=fb.ALGO_TENSOR)
    with pytest.raises(fb.B200SdrError):       # < 16 taps: split-bf16 error bound too loose, refused
        fb.FirFilter(np.ones(5, np.float32), algo=fb.ALGO_TENSOR)
    with pytest.raises(fb.B200SdrError):       # > 257 taps: Toeplitz operand no longer fits K <= 384
        fb.FirFilter(np.ones(300, np.float32), algo=fb.ALGO_TENSOR)
    # AUTO falls back to the CUDA-core kernel for those shapes
    assert fb.FirFilter(np.ones(300, np.float32)).algo == fb.ALGO_FFT          # long filter: overlap-save
    assert fb.FirFilter(np.ones(300, np.float32), sample_dtype=np.float32).algo == fb.ALGO_DIRECT
    assert fb.FirFilter(np.ones(5, np.float32)).algo == fb.ALGO_DIRECT
    assert fb.FirFilter(ramp(256)).algo == fb.ALGO_TENSOR


def test_tensor_vs_direct_full_chunk(fb):
    """BASELINE chunk size: tensor path == direct path within tolerance on 64 Mi samples."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(0x5EED)
    n = 64 * 1024 * 1024
    x = torch.view_as_complex(torch.randn(n + 255, 2, generator=g, device="cuda"))
    taps = np.random.default_rng(7).uniform(-1, 1, 256).astype(np.float32)
    ft = fb.FirFilter(taps, algo=fb.ALGO_TENSOR)
    fd = fb.FirFilter(taps, algo=fb.ALGO_DIRECT)
    yt = torch.empty(n, dtype=torch.complex64, device="cuda")
    yd = torch.empty(n, dtype=torch.complex64, device="cuda")
    assert ft.filter(x, yt)[:2] == (n, n)
    assert fd.filter(x, yd)[:2] == (n, n)
    scale = float(np.sum(np.abs(taps))) * float(x.abs().max())
    assert float((yt - yd).abs().max()) <= 1e-5 * scale


@pytest.mark.parametrize("cplx", [True, False])
def test_tensor_fir_unaligned_output_and_input(fb, rng, cplx):
    """Outputs that are not 16-byte aligned leave through the per-lane store epilogue instead of the bulk
    (TMA) stores; inputs that are not 16-byte aligned cannot be bulk-copied at all and take the CUDA-core
    kernel.  Both must still match the oracle."""
    import torch
    ntaps, n = 200, 9 * 8192 + 1234
    taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
    x = _noise(rng, n + 1, cplx)
    f = fb.FirFilter(taps, sample_dtype=x.dtype, algo=fb.ALGO_TENSOR)
    tol = 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
    xd = torch.from_numpy(x).cuda()
    for in_off, out_off in ((0, 1), (1, 0), (1, 1)):
        yd = torch.zeros(n + 1, dtype=xd.dtype, device="cuda")
        c, p, st = f.filter(xd[in_off:in_off + n], yd[out_off:out_off + n])
        c0, p0, s0, ref = orc.fir(taps, x[in_off:in_off + n], n)
        assert (c, p, int(st)) == (c0, p0, s0)
        assert np.max(np.abs(yd[out_off:out_off + p].cpu().numpy() - ref)) <= tol
        assert float(yd[out_off + p:].abs().max()) == 0.0 and (out_off == 0 or float(yd[0].abs()) == 0.0)


@pytest.mark.parametrize("decim,ntaps,cplx", [(4, 52, True), (2, 129, True), (8, 200, False), (16, 33, True),
                                              (128, 256, True), (64, 100, False)])
def test_tensor_decimating_fir(fb, rng, decim, ntaps, cplx):
    """Decimating FIR on the tensor path (the epilogue keeps the output phases D-1 mod D): many interior tiles
    (bulk stores), a ragged tail, a small output capacity, against the oracle's decimating_fir.rs restatement."""
    import torch
    n = 40 * 16384 + 12345
    x = _noise(rng, n, cplx)
    taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
    f = fb.DecimatingFirFilter(decim, taps, sample_dtype=x.dtype, algo=fb.ALGO_TENSOR)
    assert f.algo == fb.ALGO_TENSOR
    xd = torch.from_numpy(x).cuda()
    tol = 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
    for cap in (n, 1000, 1):
        yd = torch.full((cap + 8,), 7.0, dtype=xd.dtype, device="cuda")
        c, p, st = f.filter(xd, yd[:cap])
        c0, p0, s0, ref = orc.decim_fir(taps, decim, x, cap)
        assert (c, p, int(st)) == (c0, p0, s0)
        got = yd.cpu().numpy()
        assert np.max(np.abs(got[:p] - ref)) <= tol
        assert np.all(got[cap:] == 7.0)                      # nothing written past the capacity
