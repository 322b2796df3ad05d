"""Fft block options (inverse, fftshift, normalisation; src/blocks/fft.rs:160-221) at the sizes where the first load
and the last store meet a different plan shape: one pass that is both first and last (2, 16), the first two-pass
plan (32), 256 threads capped at 128 registers (8192) and 1024 threads per transform (16384).  The 4096-point case is
tests/test_gpu_blocks.py::test_fft_options; same tolerance."""
import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [2, 16, 32, 8192, 16384])
@pytest.mark.parametrize("inverse,shift,norm", [(False, True, None), (True, False, None), (True, True, None),
                                                (False, False, 1.0 / 4096), (True, True, 0.25)])
def test_fft_options_plan_shapes(rng, inverse, shift, norm, n):
    import torch
    from futuresdr_b200.blocks import Fft, FftDirection
    nfft = 9
    x = (rng.standard_normal(n * nfft) + 1j * rng.standard_normal(n * nfft)).astype(np.complex64)
    fft = Fft.with_options(n, FftDirection.Inverse if inverse else FftDirection.Forward, shift, norm)
    out = torch.zeros(x.size, dtype=torch.complex64, device="cuda")
    m = fft.transform(torch.from_numpy(x).cuda(), out)
    torch.cuda.synchronize()
    m0, ref = orc.fft_block(x, n, inverse=inverse, fft_shift=shift, normalize=norm)
    assert m == m0
    got, ref = out.cpu().numpy().reshape(nfft, n), ref.reshape(nfft, n)
    assert np.all(np.max(np.abs(got - ref), axis=1) <= 1e-5 * np.max(np.abs(ref), axis=1))
