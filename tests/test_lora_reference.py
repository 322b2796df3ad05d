"""The LoRa transmitter's CPU oracle (tests/lora_oracle.c) against an independent Python transcription, and the oracle's
frames back through a Python restatement of the reference's own hard-decision receive logic (gray_mapping.rs:60-72,
deinterleaver.rs:57-83, hamming_dec.rs:89-130, header_decoder.rs:83-250, decoder.rs:18-113) and of get_symbol_val
(utils.rs:1059-1078).  The reference's LoRa code has no tests, so this parity is unpinned.  No GPU needed."""
import itertools
import json
import os
import subprocess

import numpy as np
import pytest

from futuresdr_b200 import _lib, blocks, lora

import lora_oracle as lo

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = list(itertools.product(range(5, 13), range(1, 5), (False, True), (False, True), (False, True)))
SOME_LENGTHS = [0, 1, 2, 3, 5, 8, 13, 31, 64, 128, 254, 255]


def _pay(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def test_whitening_sequence_is_the_reference_table():
    with open(os.path.join(HERE, "golden", "lora_whitening_seq.json")) as f:
        golden = json.load(f)["bytes"]
    assert len(golden) == 255
    assert list(lo.whitening()) == golden == lo.py_whitening()


@pytest.mark.parametrize("sf", range(5, 13))
def test_encoder_oracle_matches_the_transcription(sf):
    for _, cr, crc, implicit, ldro in [c for c in CONFIGS if c[0] == sf]:
        for n in SOME_LENGTHS:
            p = _pay(n, sf * 1000 + n)
            a, b = lo.encode(p, sf, cr, crc, ldro, implicit), lo.py_encode(p, sf, cr, crc, ldro, implicit)
            assert (a is None) == (b is None) == (crc and n < 2)
            if a is not None:
                assert np.array_equal(a, b), (sf, cr, crc, implicit, ldro, n)
                assert a.size == lora.symbol_count(sf, cr, crc, ldro, implicit, n)
    _, cr, crc, implicit, ldro = CONFIGS[(sf - 5) * 32 + (sf * 7) % 32]
    for n in range(256):                              # every payload length on one configuration per SF
        p = _pay(n, n)
        a, b = lo.encode(p, sf, cr, crc, ldro, implicit), lo.py_encode(p, sf, cr, crc, ldro, implicit)
        assert (a is None and b is None) or np.array_equal(a, b), (sf, cr, crc, implicit, ldro, n)
    assert lo.encode(bytes(256), sf, 1, False, False, False) is None


@pytest.mark.parametrize("sf,os_,pad", [(sf, o, p) for sf in range(5, 13) for o in (1, 4, 8) for p in (0, 10000)])
def test_modulator_oracle_matches_the_transcription(sf, os_, pad):
    n = 16 if sf >= 11 else 40
    sym = lo.encode(_pay(n, sf), sf, 2, True, sf >= 11, False)
    sync = (8, 16) if sf > 5 else (8, 0)
    for k in range(3):                                # chirps: the three kinds, bit for bit
        args = [(0, True, None, False), (5, False, (1 << sf) * os_ // 4 - os_, False), (7, True, None, True)][k]
        a = lo.chirp(args[0], sf, os_, args[1], args[2], args[3])
        b = lo.py_chirp(args[0], sf, os_, args[1], args[2], args[3])
        assert np.array_equal(a.view(np.int32), b.view(np.int32))
    out, ph = lo.modulate(sym, sf, os_, sync, lora.preamble_len(sf), pad)
    assert out.size == lo.frame_len(sf, os_, lora.preamble_len(sf), pad, sym.size)
    assert np.array_equal(ph.view(np.int32), lo.py_phase(sym, sf, os_, sync, lora.preamble_len(sf), pad).view(np.int32))
    assert lo.ulp_diff(out, lo.f64_samples(ph)) <= 1
    if pad:                                           # the front pad: zero phase gives exactly (1, +0)
        assert out[0] == 1 + 0j and not np.signbit(out[0].imag)


# ---- the reference's hard-decision receive logic ---------------------------------------------------------------------
def _int2bool(v, n):
    return [bool((v >> (n - 1 - i)) & 1) for i in range(n)]


def _bool2int(b):
    return sum(int(x) << (len(b) - 1 - i) for i, x in enumerate(b))


def receive(symbols, sf, cr, has_crc, ldro, implicit, payload_len):
    """Symbols -> (payload, header ok, crc ok): FftDemod's hard value (bin - 1, / 4 in reduced-rate blocks), gray
    mapping, deinterleaving, Hamming decoding, the header parse and checksum, dewhitening and the CRC check.  The
    code rate and CRC flag of later blocks come from the header in explicit mode, from the arguments in implicit."""
    nibbles, pos, first = [], 0, True
    hdr_ok = True
    while pos < len(symbols):
        cw_len = 8 if first else 4 + cr
        reduced = (first and sf >= 7) or (not first and ldro)
        sf_app = sf - 2 if reduced else sf
        block = symbols[pos:pos + cw_len]
        pos += cw_len
        vals = []
        for s in block:
            v = (int(s) - 1) % (1 << sf)              # get_symbol_val's bin
            if reduced:
                v //= 4
            vals.append(v ^ (v >> 1))                 # gray_mapping.rs:60-72
        inter = [_int2bool(v, sf_app) for v in vals]
        deinter = [[False] * cw_len for _ in range(sf_app)]
        for i in range(cw_len):                       # deinterleaver.rs:57-83
            for j in range(sf_app):
                deinter[(i - j - 1) % sf_app][i] = inter[i][j]
        for k in range(sf_app):                       # hamming_dec.rs:89-130
            cr_app = cw_len - 4
            code = _int2bool(_bool2int(deinter[k]), cr_app + 4)
            data = code[0:4][::-1]
            if cr_app == 3:
                s0 = code[0] ^ code[1] ^ code[2] ^ code[4]
                s1 = code[1] ^ code[2] ^ code[3] ^ code[5]
                s2 = code[0] ^ code[1] ^ code[3] ^ code[6]
                syn = int(s0) + (int(s1) << 1) + (int(s2) << 2)
                flip = {5: 3, 7: 2, 3: 1, 6: 0}.get(syn)
                if flip is not None:
                    data[flip] = not data[flip]
            nibbles.append(_bool2int(data))
        if first and not implicit:                    # header_decoder.rs:184-250
            n = nibbles
            payload_len = (n[0] << 4) + n[1]
            has_crc = bool(n[2] & 1)
            cr = n[2] >> 1
            chk = ((n[3] & 1) << 4) + n[4]
            b = lambda x, k: (x >> k) & 1  # noqa: E731
            c4 = b(n[0], 3) ^ b(n[0], 2) ^ b(n[0], 1) ^ b(n[0], 0)
            c3 = b(n[0], 3) ^ b(n[1], 3) ^ b(n[1], 2) ^ b(n[1], 1) ^ b(n[2], 0)
            c2 = b(n[0], 2) ^ b(n[1], 3) ^ b(n[1], 0) ^ b(n[2], 3) ^ b(n[2], 1)
            c1 = b(n[0], 1) ^ b(n[1], 2) ^ b(n[1], 0) ^ b(n[2], 2) ^ b(n[2], 1) ^ b(n[2], 0)
            c0 = b(n[0], 0) ^ b(n[1], 1) ^ b(n[2], 3) ^ b(n[2], 2) ^ b(n[2], 1) ^ b(n[2], 0)
            hdr_ok = chk == (c4 << 4) + (c3 << 3) + (c2 << 2) + (c1 << 1) + c0 and payload_len != 0
        first = False
    start = 0 if implicit else 5
    total = start + 2 * payload_len + (4 if has_crc else 0)
    nib = nibbles[:total]                             # decoder.rs:18-113
    end = len(nib) - 4 if has_crc else len(nib)
    body = nib[start:end]
    out = [((body[2 * i + 1] ^ ((lo._WH[i] & 0xF0) >> 4)) << 4) | (body[2 * i] ^ (lo._WH[i] & 0x0F))
           for i in range(len(body) // 2)]
    crc_ok = True
    if has_crc:
        out_c = out + [(nib[-3] << 4) | nib[-4], (nib[-1] << 4) | nib[-2]]
        crc = 0
        for byte in out_c[:len(out_c) - 4]:
            for _ in range(8):
                crc = ((crc << 1) ^ 0x1021) if ((crc & 0x8000) >> 8) ^ (byte & 0x80) else (crc << 1)
                crc &= 0xFFFF
                byte = (byte << 1) & 0xFF
        crc ^= out_c[-3] ^ (out_c[-4] << 8)
        crc_ok = out_c[-2] + (out_c[-1] << 8) == crc
    return bytes(out), hdr_ok, crc_ok


@pytest.mark.parametrize("sf", range(5, 13))
def test_every_configuration_round_trips_through_the_reference_receiver(sf):
    for _, cr, crc, implicit, ldro in [c for c in CONFIGS if c[0] == sf]:
        for n in SOME_LENGTHS:
            if crc and n < 2:
                continue
            p = _pay(n, n + 17)
            got, hdr_ok, crc_ok = receive(lo.encode(p, sf, cr, crc, ldro, implicit), sf, cr, crc, ldro, implicit, n)
            if not implicit and n == 0:
                # header_decoder.rs:226 rejects a header announcing 0 bytes: the empty explicit frame does not decode
                assert not hdr_ok
                continue
            assert hdr_ok and crc_ok and got == p, (sf, cr, crc, implicit, ldro, n)


def _dechirp_bins(samples, sf, os_):
    """get_symbol_val (utils.rs:1059-1078) in float64 on every OS-th sample of each symbol: multiply by the conjugate
    of the id-0 upchirp (build_upchirp at OS 1), FFT, argmax of |.|^2."""
    n = 1 << sf
    t = np.arange(n, dtype=np.float64)
    ref = np.exp(-2j * np.pi * (t * t / (2 * n) - 0.5 * t))
    x = np.asarray(samples, np.complex128)[::os_].reshape(-1, n)
    return np.argmax(np.abs(np.fft.fft(x * ref, axis=1)) ** 2, axis=1)


# The running sum includes each sample's own increment (samples_from_phase_diff), which shifts every chirp by 1 / (2 OS)
# of a bin: at OS 1 that is half a bin and bins b and b + 1 tie, so the check runs at OS >= 2.
@pytest.mark.parametrize("sf,os_", [(5, 2), (6, 4), (7, 8), (9, 4), (12, 2)])
def test_chirps_demodulate_to_their_symbols(sf, os_):
    pre = lora.preamble_len(sf)
    sym = lo.encode(_pay(20, sf), sf, 1, True, False, False)
    sync = (8, 16)
    out, _ = lo.modulate(sym, sf, os_, sync, pre, 0)
    N = (1 << sf) * os_
    q = N // 4 - os_
    head = (pre + 2) * N
    assert list(_dechirp_bins(out[:pre * N], sf, os_)) == [0] * pre
    assert list(_dechirp_bins(out[pre * N:head], sf, os_)) == list(sync)
    data = out[head + 2 * N + q + (2 * N if sf < 7 else 0):]
    assert list(_dechirp_bins(data, sf, os_)) == [(int(s) - 1) % (1 << sf) for s in sym]


def test_burst_lengths_against_sample_count():
    """Explicit-header frames: the modulated length equals sample_count wherever sample_count's usize arithmetic does
    not underflow.  It underflows when header and payload fit the first interleaver block (short payloads at high SF);
    there the reference's own estimate would panic in a debug build, and the transmitter follows modulate()."""
    underflow = []
    for sf, cr, crc, _, ldro in [c for c in CONFIGS if not c[3]]:
        for n in range(0, 256, 3):
            if crc and n < 2:
                continue
            sym = lo.encode(bytes(n), sf, cr, crc, ldro, False)
            for os_, pad in ((1, 0), (4, 10000), (8, 0)):
                length = lo.frame_len(sf, os_, 8, pad, sym.size)
                sc = lo.sample_count(sf, 8, True, n, crc, cr, os_, pad, ldro)
                if sc is None:
                    underflow.append((sf, n))
                    with pytest.raises(ValueError):
                        lora.sample_count(sf, 8, True, n, crc, cr, os_, pad, ldro)
                    continue
                assert sc == length == lora.sample_count(sf, 8, True, n, crc, cr, os_, pad, ldro), (sf, cr, crc, ldro,
                                                                                                      n, os_, pad)
    assert underflow and all(n <= 3 for _, n in underflow)


def test_host_helpers():
    assert lora.SynchWord(value=0x34).verify_and_expand(7) == (24, 32)
    with pytest.raises(ValueError):
        lora.SynchWord(value=0x34).verify_and_expand(5)          # [24, 32] at SF5
    assert lora.SynchWord.from_pmt(bytes([8, 16])).expand() == (8, 16)
    assert lora.SynchWord.from_pmt(0x12).expand() == (8, 16)
    assert lora.preamble_len(5) == 12 and lora.preamble_len(6) == 8
    ldro = [lora.LdroMode.AUTO.resolve_if_auto(sf, bw) for sf in range(5, 13) for bw in lora.Bandwidth]
    assert [int(sf) for sf in range(5, 13) for bw in lora.Bandwidth
            if ldro[(sf - 5) * 4 + list(lora.Bandwidth).index(bw)] == lora.LdroMode.ENABLE] == [10, 11, 11, 12, 12, 12]
    for bad in ((4, 1), (13, 1), (7, 0), (7, 5)):
        with pytest.raises(_lib.B200SdrError):
            lora.symbol_count(bad[0], bad[1], False, False, False, 1)
    with pytest.raises(_lib.B200SdrError):
        lora.symbol_count(7, 1, False, False, False, 256)


def test_header_mirror_of_the_new_constants(tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sdr.h"\nint main(void) {\n'
                   '    printf("%d %zu %zu %zu\\n", B2S_LORA_MAX_PAYLOAD, sizeof(b2s_lora_burst),\n'
                   '           offsetof(b2s_lora_burst, index), offsetof(b2s_lora_burst, len));\n    return 0;\n}\n')
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(os.path.dirname(HERE), "include"), str(src), "-o",
                    str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = blocks.LORA_BURST
    assert got == [_lib.LORA_MAX_PAYLOAD, d.itemsize, d.fields["index"][1], d.fields["len"][1]]
