"""The tensor FIR at the edges of its tiles: the CTAs of a launch take whole 64-block (complex) / 128-block (real)
tiles of 128-item blocks from the launch's tile counter as they run, and the output may end anywhere inside a tile or
a block.  Checked against the CUDA-core kernel (ALGO_DIRECT) within the usual 1e-5 * ||taps||_1 * max|x|, and bit for
bit against the same samples filtered one tile per launch: a column of the block-Toeplitz product does not depend on
which CTA, tile or launch computes it.  Many launches of one plan in a row also check that every launch leaves its
tile counter zeroed for the next."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NTAPS = 256


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tile_blocks(cplx):
    return 64 if cplx else 128


def _noise(n, cplx, seed):
    rng = np.random.default_rng(seed)
    if cplx:
        return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    return rng.standard_normal(n).astype(np.float32)


def _taps(ntaps=NTAPS):
    return np.random.default_rng(5).uniform(-1, 1, ntaps).astype(np.float32)


def _filters(cplx, decim, ntaps=NTAPS):
    import futuresdr_b200 as fb
    dt = np.complex64 if cplx else np.float32
    t = _taps(ntaps)
    tc = fb.DecimatingFirFilter(decim, t, dt, algo=fb.ALGO_TENSOR)
    assert tc.algo == fb.ALGO_TENSOR
    return t, tc, fb.DecimatingFirFilter(decim, t, dt, algo=fb.ALGO_DIRECT)


def _run(f, xd, n_out):
    y = torch.full((n_out,), 7.0, dtype=xd.dtype, device="cuda")
    c, p, st = f.filter(xd, y)
    torch.cuda.synchronize()
    return (c, p, int(st)), y


def _close(taps, x, a, b):
    tol = 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
    err = float((a - b).abs().max()) if a.numel() else 0.0
    assert err <= tol, (err, tol)


def _n_in(n_blocks, cplx, decim, ragged, ntaps=NTAPS):
    """input length whose output covers n_blocks full-rate blocks, the last one `ragged` outputs short"""
    n_out = (n_blocks * 128 - ragged * decim) // decim
    return n_out * decim + ntaps - 1, n_out


def _check_direct(cplx, decim, n_blocks, ragged, seed):
    taps, tc, direct = _filters(cplx, decim)
    n, n_out = _n_in(n_blocks, cplx, decim, ragged)
    x = _noise(n, cplx, seed)
    xd = torch.from_numpy(x).cuda()
    r_tc, y_tc = _run(tc, xd, n_out)
    r_d, y_d = _run(direct, xd, n_out)
    assert r_tc == r_d and r_tc[1] == n_out
    _close(taps, x, y_tc, y_d)
    return tc, xd, y_tc, n_out


def _check_tiles_bitwise(tc, xd, y, cplx, decim, tiles):
    """tile t of the whole launch's output == the same samples filtered as one launch of exactly one tile"""
    t_items = _tile_blocks(cplx) * 128
    for t in tiles:
        i0 = t * t_items
        n_out = min(t_items, y.numel() * decim - i0) // decim
        if n_out <= 0:
            continue
        xs = xd[i0:i0 + n_out * decim + NTAPS - 1]
        _, ys = _run(tc, xs, n_out)
        o0 = i0 // decim
        assert torch.equal(_bits(ys), _bits(y[o0:o0 + n_out])), (t, decim)


def _bits(y):
    return (torch.view_as_real(y) if y.is_complex() else y).contiguous().view(torch.int32)


def _sizes(cplx):
    tb = _tile_blocks(cplx)
    # one tile ending at every block; four tiles, the last one ending at every block
    return list(range(1, tb + 1)) + [3 * tb + r for r in range(tb)]


@pytest.mark.parametrize("cplx", [True, False], ids=["c32", "f32"])
@pytest.mark.parametrize("decim", [1, 4, 128])
def test_output_end_at_every_block_of_a_tile(cplx, decim):
    tb = _tile_blocks(cplx)
    for i, nb in enumerate(_sizes(cplx)):
        ragged = (i * 37) % (128 // decim)
        tc, xd, y, _ = _check_direct(cplx, decim, nb, ragged, seed=100 + i)
        if i % 8 == 0:
            _check_tiles_bitwise(tc, xd, y, cplx, decim, range(-(-nb // tb)))


@pytest.mark.parametrize("cplx", [True, False], ids=["c32", "f32"])
@pytest.mark.parametrize("decim", [1, 4, 128])
@pytest.mark.parametrize("n_blocks", [1, 2, 7, 8, 9, 40, 63, 64, 65, 127, 128, 129, 500],
                         ids=lambda b: f"{b}blk")
def test_single_tile_and_fewer_tiles_than_sms(cplx, decim, n_blocks):
    tc, xd, y, _ = _check_direct(cplx, decim, n_blocks, ragged=n_blocks % (128 // decim), seed=n_blocks)
    _check_tiles_bitwise(tc, xd, y, cplx, decim, range(-(-n_blocks // _tile_blocks(cplx))))


@pytest.mark.parametrize("cplx", [True, False], ids=["c32", "f32"])
@pytest.mark.parametrize("decim", [1, 4, 128])
def test_many_tiles_per_cta(cplx, decim):
    """three whole waves and a part of a fourth one, ending inside a block: the raw-slot and operand-stage rings wrap;
    the first and the last tiles checked bit for bit"""
    tb = _tile_blocks(cplx)
    nb = _sm_count() * tb * 3 + 8 * 37 + 5
    tc, xd, y, _ = _check_direct(cplx, decim, nb, ragged=3 % (128 // decim), seed=7)
    nt = -(-nb // tb)
    _check_tiles_bitwise(tc, xd, y, cplx, decim, list(range(16)) + list(range(nt - 16, nt)))


def _exec_hist(fir, hist_t, in_t, out_t):
    from futuresdr_b200._lib import check, lib
    c, p, st = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
    check(lib.b2s_fir_exec_hist(fir._h, C.c_void_p(hist_t.data_ptr()), hist_t.numel(), C.c_void_p(in_t.data_ptr()),
                                in_t.numel(), C.c_void_p(out_t.data_ptr()), out_t.numel(), None, C.byref(c),
                                C.byref(p), C.byref(st)), fir.ctx.handle)
    torch.cuda.synchronize()
    return c.value, p.value, st.value


@pytest.mark.parametrize("cplx", [True, False], ids=["c32", "f32"])
@pytest.mark.parametrize("decim", [1, 4, 128])
@pytest.mark.parametrize("lead", [0, 1])
@pytest.mark.parametrize("n_blocks", [5, 64 * 3 + 17, 132 * 64 + 8 * 11 + 3])
def test_lead_and_detached_history(cplx, decim, lead, n_blocks):
    """`lead` dummy items (a history 0 or 1 items off 16 bytes) with the history in its own allocation, fetched into
    the first raw slot of the tile at item 0; the poisoned items around it must not leak into the result"""
    taps, tc, direct = _filters(cplx, decim)
    n, n_out = _n_in(n_blocks, cplx, decim, ragged=1 % (128 // decim))
    x = _noise(n, cplx, seed=lead + 11 * n_blocks)
    xd = torch.from_numpy(x).cuda()
    r_d, y_d = _run(direct, xd, n_out)
    q = 2 if cplx else 4                                # items per 16 bytes
    H = NTAPS - 1 + (-(lead + NTAPS - 1)) % q           # lead + history: whole 16-byte units
    # the history placed `lead` items past a 16-byte boundary, in its own allocation; the slice starts on one
    hist_buf = torch.full((H + 16,), float("nan"), dtype=xd.dtype, device="cuda")
    hist = hist_buf[lead:lead + H]
    hist.copy_(xd[:H])
    buf = torch.full((n - H + 64,), float("nan"), dtype=xd.dtype, device="cuda")
    body = buf[:n - H]
    body.copy_(xd[H:])
    y = torch.full((n_out,), 7.0, dtype=xd.dtype, device="cuda")
    c, p, st = _exec_hist(tc, hist, body, y)
    assert (c, p, st) == r_d
    got = torch.view_as_real(y) if y.is_complex() else y
    assert bool(torch.isfinite(got).all())
    _close(taps, x, y, y_d)


def test_many_launches_of_one_plan():
    """more launches of one plan than it has tile counters, each one checked bit for bit against the first"""
    taps, tc, _ = _filters(True, 1)
    n, n_out = _n_in(_sm_count() * 64 + 8 * 5 + 1, True, 1, ragged=7)
    xd = torch.from_numpy(_noise(n, True, seed=3)).cuda()
    _, y0 = _run(tc, xd, n_out)
    for _ in range(150):
        _, y = _run(tc, xd, n_out)
        assert torch.equal(_bits(y), _bits(y0))
