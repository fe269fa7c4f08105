"""Raster mixing handles (rxb200_fm_mix_create_raster) on the GPU: the raster kernels alone (rxb200_raster_device)
against the numpy model over every int16 value, over M, T, K, the stateless sample index n0, source offsets and short
calls; both exact anchors byte for byte against rxb200_ddc_device; every named shape through the handle against the port
and the golden hashes; the phase and filter history across reads, chunk calls and reset; a call longer than the
frame-group scratch; the device entry points with an unaligned capture; and refusals that leave no trace."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_handles as fh
import fm_raster as frs
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_raster_golden.json")


def _bins(K):
    return [0, 1, K // 2, K - 1, 1]


def _taps(n_taps, seed):
    """Random taps with sum |h| just under 2^22, and the shift that brings the largest sums near int16 full scale."""
    rng = np.random.default_rng(seed)
    h = rng.integers(-(1 << 22) // n_taps, (1 << 22) // n_taps, size=n_taps, endpoint=False)
    h[0] = h[0] or 1
    while frs.sum_abs(h) >= (1 << 22):
        h //= 2
    shift = 17 + int(np.ceil(np.log2(np.sqrt(n_taps) * (np.abs(h).mean() + 1))))    # typical |y| ~ 2^13
    return h.astype(np.int32), shift


CASES = sorted({(K, m, t) for K in (3, 4, 768, 4096) for m in (1, 7, 64, 4096)
                for t in (1, K - 1, K, 4 * K + 1, 8192) if 1 <= t <= 8192})


@pytest.mark.parametrize("K,decim,n_taps", CASES)
def test_raster_device_equals_model(K, decim, n_taps):
    torch = fh.torch()
    bins = _bins(K)
    taps, shift = _taps(n_taps, K + decim + n_taps)
    x = fh.every_int16(K * 7 + decim + n_taps)
    n_max = min(65536, max(decim + 3, (1 << 21) * decim // (n_taps * len(bins))))   # keeps the model's work bounded
    # the capture 0, 4 and 16 bytes past a 256-byte aligned allocation
    srcs = {off16: torch.from_numpy(np.concatenate([np.zeros(off16, np.int16), x])).cuda() for off16 in (0, 2, 8)}
    dst = torch.zeros(len(bins) * 2 * (65536 // decim) + 64, dtype=torch.int16, device="cuda")
    ddc = (decim, taps, shift)
    for n0 in ((1 << 64) - K + 1, (1 << 40) + 3):
        for n in sorted({n_max, decim - 1, 2 * decim + 1, 1}):
            for off16, src in (srcs.items() if n == n_max else [(0, srcs[0])]):
                if n < 1:
                    continue
                dst.fill_(0)
                fm.raster_device(K, bins, n0, ddc, src.data_ptr() + 2 * off16, n, dst.data_ptr())
                torch.cuda.synchronize()
                want, _ = frs.raster_model(x[:2 * n], K, bins, taps, decim, shift, phase=n0 % K)
                assert want.shape == (len(bins), 2 * (n // decim))
                got = dst[:want.size].cpu().numpy().reshape(want.shape)
                bad = np.argwhere(got != want)
                assert bad.size == 0, (K, decim, n_taps, n0, off16, n, bad[:4])
                assert not dst[want.size:].any().item(), (K, decim, n_taps, n0, n)   # nothing past n / M outputs


def test_raster_device_long_call_over_many_groups():
    """K = 4096, M = 1: 1024 frames per group of the 64 MiB scratch, so a call of 5000 outputs runs five groups."""
    torch = fh.torch()
    K, bins, taps = 4096, [3, 4095, 2048], np.array([7, -3, 11, 2, -9], np.int32)
    x = fh.every_int16(5)[:2 * 5000]
    src = torch.from_numpy(x).cuda()
    dst = torch.zeros(3 * 2 * 5000, dtype=torch.int16, device="cuda")
    fm.raster_device(K, bins, 77, (1, taps, 19), src.data_ptr(), 5000, dst.data_ptr())
    torch.cuda.synchronize()
    want, _ = frs.raster_model(x, K, bins, taps, 1, 19, phase=77)
    assert dst.cpu().numpy().tobytes() == want.tobytes()


@pytest.mark.parametrize("K", [4, 12, 768])
def test_anchors_against_ddc_device(K):
    torch = fh.torch()
    rate = 2_400_000
    x = fh.every_int16(K)[:2 * 30001]
    taps = fdd.lowpass(65, 0.02, gain_bits=20)
    src = torch.from_numpy(x).cuda()
    a = torch.zeros(2 * 30001, dtype=torch.int16, device="cuda")
    b = torch.zeros_like(a)
    for shift in (0, 9, 20, 47):
        fm.raster_device(K, [0], 5, (3, taps, shift + 15), src.data_ptr(), 30001, a.data_ptr())
        fm.ddc_device(rate, 0, 0, (3, taps, shift), src.data_ptr(), 30001, b.data_ptr())
        torch.cuda.synchronize()
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), (K, shift)
    xq = x.copy()
    xq[xq == -32768] = -32767
    src = torch.from_numpy(xq).cuda()
    for shift in (5, 20):
        for n0 in (0, 1, 2, 3, (1 << 40) + 3):
            fm.raster_device(K, [K // 4], n0, (3, taps, shift + 15), src.data_ptr(), 30001, a.data_ptr())
            fm.ddc_device(rate, rate // 4, n0, (3, taps, shift), src.data_ptr(), 30001, b.data_ptr())
            torch.cuda.synchronize()
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), (K, shift, n0)


def _levels_params(p):
    q = fm.FmParams.from_any(p)
    q.report_levels = 1 if q.squelch_level else 0
    return q


@pytest.mark.parametrize("name", sorted(frs.SHAPES))
def test_shapes_equal_the_port(name, port):
    p, K, bins, ddc, x, reads = frs.case_input(name, seed=5)
    p = _levels_params(p)
    mx = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    got, counts = fh.reads(mx, x, reads)
    assert mx.mix_ms() > 0
    q = fac.P(**p.reference_fields())
    for c, dec in enumerate(frs.decimated_reads(x, K, bins, ddc, reads)):
        y, lens = fdd.nonempty(dec)
        want, rl, wh = fac.port_run_seq(port, q, y, lens, return_chunks=True)
        fh.compare(p, got[c], want, (name, c))
        assert [n for n, d in zip(counts, dec) if d.size] == rl.tolist(), (name, c)
        assert mx.squelch_hits()[c] == wh[-1], (name, c)
        if p.report_levels:
            assert mx.levels()[c, -1] == fac.port_levels_seq(port, q, y, lens)[-1], (name, c)
    mx.close()


def test_golden():
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(frs.SHAPES)
    for name in sorted(frs.SHAPES):
        p, K, bins, ddc, x, reads = frs.case_input(name)
        g = gold[name]
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        mx = fm.FmMix(p, ddc=ddc, raster=(K, bins))
        got, counts = fh.reads(mx, x, g["lens_int16"])
        for c, gc in enumerate(g["channels"]):
            assert gc["bin"] == bins[c]
            assert [n for n, d in zip(counts, gc["dec_len"]) if d] == gc["result_len"], (name, c)
            assert hashlib.sha256(got[c].tobytes()).hexdigest() == gc["sha256"], (name, c)
        mx.close()


def _chain_lens(ops, M, pos=0):
    """The chain reads a sequence of ('read', n16) / ('chunk', n16, chunk16) calls hands the member, in order."""
    lens = []
    for op in ops:
        n16 = op[1]
        if op[0] == "read":
            d = fdd.decimated_len(pos, n16, M)
            if d:
                lens.append(d)
        else:
            for a in range(0, n16, op[2]):
                d = fdd.decimated_len(pos + a // 2, min(op[2], n16 - a), M)
                if d:
                    lens.append(d)
        pos += n16 // 2
    return lens


def _run_ops(mx, x, ops):
    out, at = [], 0
    for op in ops:
        part = x[at:at + op[1]]
        out.append(mx.process_read(part) if op[0] == "read" else mx.full_demod(part, op[2]))
        at += op[1]
    return np.concatenate(out, axis=1)


@pytest.mark.parametrize("name", ["am_k240_m100", "raw_k100_m100", "raw_sat_k3_m3"])
def test_carries_across_reads_chunks_and_reset(name, port):
    p, K, bins, ddc, x, _ = frs.case_input(name, seed=6)
    M = ddc[0]
    ops = [("chunk", 2 * M * 300 + 2 * 77, 2 * M * 100), ("read", 2 * 4099), ("read", 2 * 5),
           ("chunk", 2 * M * 200, 2 * M * 40), ("read", 2 * 30011), ("chunk", 2 * 333, 2 * M * 64)]
    x = x[:sum(op[1] for op in ops)]
    lens = _chain_lens(ops, M)
    mx = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    first = _run_ops(mx, x, ops)
    y, _ = frs.raster_model(x, K, bins, ddc[1], M, ddc[2])
    for c in range(len(bins)):
        assert y[c].size == sum(lens)
        fh.compare(p, first[c], fac.port_run_seq(port, p, y[c], lens), (name, c))
    mx.reset()
    assert _run_ops(mx, x, ops).tobytes() == first.tobytes()
    mx.close()


def test_long_call_equals_short_groups():
    """One read of 5000 outputs at K = 4096, M = 1 (five scratch groups) against the same capture in reads of at most
    1000 samples, each one group."""
    p = fac.with_(fac.RAW, downsample=1, offset_tuning=1)
    K, bins, ddc = 4096, [0, 5, 4091], (1, np.array([1, 2, 3, 2, 1], np.int32), 24)
    x = fh.every_int16(9)[:2 * 5000]
    one = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    many = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    a = one.process_read(x)
    b, _ = fh.reads(many, x, [2 * 1000, 2 * 999, 2 * 1])
    assert a.tobytes() == b.tobytes()
    one.close()
    many.close()


def test_device_entries_with_an_unaligned_capture():
    torch = fh.torch()
    p, K, bins, ddc, x, reads = frs.case_input("fm2b_f9_k64_m8", seed=8)
    host = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    want_reads, _ = fh.reads(host, x, reads)
    host.reset()
    M = ddc[0]
    chunk = 2 * M * 4096
    n = (x.size // chunk) * chunk
    want_call = host.full_demod(x[:n], chunk)
    host.close()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()
    cap = buf[2:]
    assert cap.data_ptr() % 16 == 4
    mx = fm.FmMix(p, ddc=ddc, raster=(K, bins))
    stride = want_reads.shape[1] + 8
    out = torch.zeros((len(bins), stride), dtype=torch.int16, device="cuda")
    parts = []
    for pos, n16 in fac.seq_bounds(x.size, reads):
        k = mx.process_read_device(cap.data_ptr() + 2 * pos, n16, out.data_ptr(), stride, sync=True)
        parts.append(out[:, :k].cpu().numpy())
    assert np.concatenate(parts, axis=1).tobytes() == want_reads.tobytes()
    mx.reset()
    k = mx.process_device(cap.data_ptr(), n, chunk, out.data_ptr(), stride)
    torch.cuda.synchronize()
    assert k == want_call.shape[1] and out[:, :k].cpu().numpy().tobytes() == want_call.tobytes()
    mx.close()


def test_refusals_leave_no_trace():
    p, K, bins, ddc, x, _ = frs.case_input("fm2b_f9_k64_m8", seed=9)
    for raster, dd in (((64, [64]), ddc), ((2, [0]), ddc), ((64, [0]), (8, np.full(4, 1 << 20, np.int32), 30))):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.FmMix(p, ddc=dd, raster=raster)
        assert e.value.code == _lib.EINVAL
    mx, fresh = fm.FmMix(p, ddc=ddc, raster=(K, bins)), fm.FmMix(p, ddc=ddc, raster=(K, bins))
    a = mx.full_demod(x[:2 * 8 * 4096], 2 * 8 * 1024)
    assert a.tobytes() == fresh.full_demod(x[:2 * 8 * 4096], 2 * 8 * 1024).tobytes()
    rest = x[2 * 8 * 4096:]
    for call in (lambda: mx.full_demod(rest[:2 * 8 * 1024], 2 * 8 * 1024 + 2),
                 lambda: mx.process_read(rest[:2 * 60]),                   # 7 or 8 outputs < 2^3 for the passes
                 lambda: mx.process_read(rest[:31])):
        with pytest.raises(_lib.Rxb200Error) as e:
            call()
        assert e.value.code == _lib.EUNSUPPORTED
    assert mx.decimated_len(2 * 60) == 2 * 7
    assert mx.process_read(rest[:2 * 20011]).tobytes() == fresh.process_read(rest[:2 * 20011]).tobytes()
    mx.close()
    fresh.close()
