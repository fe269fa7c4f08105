"""Decimating mixing handles (rxb200_fm_mix_create_ddc) on the GPU: fm_ddc_kernel alone (rxb200_ddc_device) against the
numpy model over every int16 value, on the int32 and int64 accumulators; the identity DDC against a plain mixing handle
on every kernel route; K channels against the port on the model's decimated streams; the phase and filter history
across ragged reads, chunk calls, mixed sequences and reset; the device entry points with an unaligned capture;
refusals that leave no trace; decimated_len and max_output; and the golden hashes of the reference."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_handles as fh
import fm_mix as fmx
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_ddc_golden.json")
IDENTITY = (1, np.ones(1, np.int32), 0)


def _tap_sets(decim, n_taps, seed):
    """(taps, shift) pairs: a Q15 low-pass (the int32 accumulator unless T is large) and large random taps at a small
    shift (the int64 accumulator, saturating outputs)."""
    rng = np.random.default_rng(seed)
    out = [(fdd.lowpass(n_taps, 0.45 / decim), 15),
           (rng.integers(-(1 << 20), 1 << 20, size=n_taps).astype(np.int32), 3)]
    if n_taps == 1:
        out.append((np.array([-(1 << 31)], np.int32), 62))                    # the largest |h| at the largest S
    return out


CASES = sorted({(m, t) for m in (1, 2, 7, 64, 4096) for t in (1, m, 4 * m + 1, 8192) if t <= 8192})


@pytest.mark.parametrize("decim,n_taps", CASES)
def test_ddc_device_equals_model(decim, n_taps):
    torch = fh.torch()
    rate, f = 2_400_000, 37500
    t = fm.mix_table(rate, f)
    L = t.shape[0]
    x = fh.every_int16(decim * 7 + n_taps)
    n_max = min(65536, max(decim + 3, (1 << 22) * decim // n_taps))     # keeps the model's work bounded
    # the capture 0, 4 and 16 bytes past a 256-byte aligned allocation
    srcs = {off16: torch.from_numpy(np.concatenate([np.zeros(off16, np.int16), x])).cuda() for off16 in (0, 2, 8)}
    dst = torch.zeros(2 * (65536 // decim) + 64, dtype=torch.int16, device="cuda")
    for taps, shift in _tap_sets(decim, n_taps, decim + n_taps):
        ddc = (decim, taps, shift)
        for phase in (0, (1 << 40) + 3):
            for off16, src in srcs.items():
                for n in sorted({n_max, n_max - 1, decim - 1, 2 * decim + 1, 1}):
                    if n < 1:
                        continue
                    dst.fill_(0)
                    fm.ddc_device(rate, f, phase, ddc, src.data_ptr() + 2 * off16, n, dst.data_ptr())
                    torch.cuda.synchronize()
                    want, _ = fdd.ddc_model(x[:2 * n], t, taps, decim, shift, table_phase=phase % L)
                    assert want.size == 2 * (n // decim)
                    got = dst[:want.size].cpu().numpy()
                    bad = np.flatnonzero(got != want)
                    assert bad.size == 0, (decim, n_taps, shift, phase, off16, n, bad[:4])
                    assert not dst[want.size:].any().item(), (decim, n_taps, phase, n)   # nothing past n / M outputs


def test_ddc_device_source_offsets():
    """The source at 4- and 16-byte offsets into a buffer reads the right samples."""
    torch = fh.torch()
    rate, f, ddc = 1_008_000, 24000, (3, fdd.lowpass(17, 0.1), 15)
    t = fm.mix_table(rate, f)
    x = fh.every_int16(3)[:2 * 10001]
    for pad in (2, 8):                                    # int16 of padding: 4 and 16 bytes
        buf = torch.from_numpy(np.concatenate([np.full(pad, 77, np.int16), x])).cuda()
        dst = torch.zeros(2 * (10001 // 3) + 8, dtype=torch.int16, device="cuda")
        fm.ddc_device(rate, f, 5, ddc, buf.data_ptr() + 2 * pad, 10001, dst.data_ptr())
        torch.cuda.synchronize()
        want, _ = fdd.ddc_model(x, t, ddc[1], 3, 15, table_phase=5)
        assert dst[:want.size].cpu().numpy().tobytes() == want.tobytes(), pad
        assert not dst[want.size:].any().item()


def test_ddc_device_refusals():
    torch = fh.torch()
    buf = torch.zeros(64, dtype=torch.int16, device="cuda")
    p = buf.data_ptr()
    good = (2, [1, 1], 1)
    for args, code in (((2_400_000, 0, 0, (0, [1], 0), p, 8, p), _lib.EINVAL),
                       ((2_400_000, 0, 0, (2, [1], 63), p, 8, p), _lib.EINVAL),
                       ((2_400_000, 0, 0, (2, [1] * 8193, 0), p, 8, p), _lib.EINVAL),
                       ((2_400_000, 1_200_000, 0, good, p, 8, p), _lib.EINVAL),
                       ((2_400_001, 1, 0, good, p, 8, p), _lib.EUNSUPPORTED),
                       ((2_400_000, 0, -1, good, p, 8, p), _lib.EINVAL),
                       ((2_400_000, 0, 0, good, p + 2, 8, p), _lib.EINVAL),
                       ((2_400_000, 0, 0, good, None, 8, p), _lib.EINVAL)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.ddc_device(*args)
        assert e.value.code == code, args


@pytest.mark.parametrize("name", sorted(fh.KERNEL_ROUTES))
def test_identity_is_a_plain_mixing_handle(name):
    """M = 1, h = {1}, S = 0 gives the bytes of a plain mixing handle, on the route the plain handle takes."""
    p, mode, chunk, lens, kind = fh.KERNEL_ROUTES[name]
    x = fac.signal(sum(lens) // 2, 41)
    offs = [0, 300_000]
    dd = fm.FmMix(p, 2_400_000, offs, ddc=IDENTITY)
    mx = fm.FmMix(p, 2_400_000, offs)
    pos = 0
    for c, n in enumerate(lens):
        part = x[pos:pos + n]
        if mode == "read":
            got, want = dd.process_read(part), mx.process_read(part)
        else:
            (got, gl), (want, wl) = dd.full_demod(part, chunk, True), mx.full_demod(part, chunk, True)
            assert gl.tolist() == wl.tolist(), (name, c)
        assert got.tobytes() == want.tobytes(), (name, c)
        assert dd.stats()["kernel_kind"] == kind == mx.stats()["kernel_kind"], (name, c, dd.stats())
        pos += n
    assert dd.squelch_hits().tolist() == mx.squelch_hits().tolist()
    dd.close()
    mx.close()


@pytest.mark.parametrize("k", [1, 3, 8, 33, 257])
def test_k_channels_equal_the_port(k, port):
    p, rate, _, ddc, _, reads = fdd.SHAPES["nbfm_m64_t257"]
    offs = [25000 * (j - k // 2) for j in range(k)]                    # a 25 kHz raster, up to +-3.2 MHz
    lens = [2 * 9001, 2 * 5003, 2 * 7919]
    x = fmx.capture(fdd.n_complex_for(lens), rate, offs[::7], 810 + k)
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    got, _ = fh.reads(mx, x, lens)
    for j, (want, _, wh) in enumerate(fh.port_channels(port, p, rate, offs, x, lens, ddc)):
        fh.compare(p, got[j], want, (k, offs[j]))
        assert mx.squelch_hits()[j] == wh[-1]
    mx.close()


@pytest.mark.parametrize("name", sorted(fdd.SHAPES))
def test_shapes_equal_the_port(name, port):
    p, rate, offs, ddc, x, reads = fdd.case_input(name, seed=5)
    p = fm.FmParams.from_any(p)
    p.report_levels = 1 if p.squelch_level else 0
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    got, counts = fh.reads(mx, x, reads)
    q = fac.P(**p.reference_fields())
    for j, (want, rl, wh) in enumerate(fh.port_channels(port, q, rate, offs, x, reads, ddc)):
        fh.compare(p, got[j], want, (name, offs[j]))
        dec = fdd.decimated_reads(x, fm.mix_table(rate, offs[j]), ddc, reads)
        assert [c for c, d in zip(counts, dec) if d.size] == rl.tolist(), (name, j)
        assert all(c == 0 for c, d in zip(counts, dec) if not d.size), (name, j)
        assert mx.squelch_hits()[j] == wh[-1], (name, j)
    if p.report_levels:
        lv = mx.levels()
        for j, f in enumerate(offs):
            y, lens = fdd.nonempty(fdd.decimated_reads(x, fm.mix_table(rate, f), ddc, reads))
            assert lv[j, -1] == fac.port_levels_seq(port, q, y, lens)[-1], (name, j)
    mx.close()


def test_empty_read_runs_no_chain_call():
    p, rate, offs, ddc, x, _ = fdd.case_input("fm_lut_squelch_m4", seed=3)
    p = fm.FmParams.from_any(p)
    p.report_levels = 1
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    mx.process_read(x[:2 * 4001])
    assert mx.levels().shape == (2, 1)
    hits = mx.squelch_hits().tolist()
    assert mx.decimated_len(2) == 0                       # 4001 samples in: the next emission is sample 4003
    r = mx.process_read(x[2 * 4001:2 * 4002])
    assert r.shape == (2, 0) and mx.levels().shape == (2, 0) and mx.squelch_hits().tolist() == hits
    assert mx.decimated_len(4) == 2                       # samples 4002, 4003: one output
    mx.close()


def _chain_lens(ops, M, pos=0):
    """The chain reads a sequence of ('read', n16) / ('chunk', n16, chunk16) calls hands the member, in order (empty
    reads skipped), and the capture samples it covers."""
    lens = []
    for op in ops:
        n16 = op[1]
        if op[0] == "read":
            d = fdd.decimated_len(pos, n16, M)
            if d:
                lens.append(d)
        else:
            c16 = op[2]
            for a in range(0, n16, c16):
                d = fdd.decimated_len(pos + a // 2, min(c16, n16 - a), M)
                if d:
                    lens.append(d)
        pos += n16 // 2
    return lens, pos


def _run_ops(mx, x, ops):
    out, at = [], 0
    for op in ops:
        part = x[at:at + op[1]]
        out.append(mx.process_read(part) if op[0] == "read" else mx.full_demod(part, op[2]))
        at += op[1]
    return np.concatenate(out, axis=1)


@pytest.mark.parametrize("name", ["am_m100", "raw_m100", "raw_wide_m3"])
def test_carries_across_reads_chunks_mixed_and_reset(name, port):
    p, rate, offs, ddc, x, _ = fdd.case_input(name, seed=6)
    M = ddc[0]
    ops = [("chunk", 2 * M * 300 + 2 * 77, 2 * M * 100), ("read", 2 * 4099), ("read", 2 * 5),
           ("chunk", 2 * M * 200, 2 * M * 40), ("read", 2 * 30011), ("chunk", 2 * 333, 2 * M * 64)]
    total = sum(op[1] for op in ops)
    x = x[:total]
    lens, _ = _chain_lens(ops, M)
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    first = _run_ops(mx, x, ops)
    for j, f in enumerate(offs):
        y, _ = fdd.ddc_model(x, fm.mix_table(rate, f), ddc[1], M, ddc[2])
        assert y.size == sum(lens)
        want = fac.port_run_seq(port, p, y, lens)
        fh.compare(p, first[j], want, (name, j))
    mx.reset()
    again = _run_ops(mx, x, ops)
    assert again.tobytes() == first.tobytes()
    mx.close()


def test_chunk_result_len_of_chunks_without_output():
    p, rate, offs, ddc, x, _ = fdd.case_input("am_m100", seed=7)
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    # 3 chunks of 200 samples and a last one of 50: at phase 0 the last chunk makes no output (emission at 99 mod 100)
    _, rl = mx.full_demod(x[:2 * 650], 2 * 200, True)
    assert rl.tolist() == [2, 2, 2, 0]
    _, rl = mx.full_demod(x[2 * 650:2 * 700], 2 * 200, True)      # samples 650..699: emission 699
    assert rl.tolist() == [1]
    mx.close()


@pytest.mark.parametrize("name", ["nbfm_m64_t257", "fm2b_f9_m8"])
def test_device_entries_with_an_unaligned_capture(name):
    torch = fh.torch()
    p, rate, offs, ddc, x, reads = fdd.case_input(name, seed=8)
    host = fm.FmMix(p, rate, offs, ddc=ddc)
    want_reads, _ = fh.reads(host, x, reads)
    host.reset()
    M = ddc[0]
    chunk = 2 * M * (4096 if p.downsample_passes else 1021)
    n = (x.size // chunk) * chunk
    want_call = host.full_demod(x[:n], chunk)
    host.close()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()
    cap = buf[2:]
    assert cap.data_ptr() % 16 == 4
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    stride = want_reads.shape[1] + 8
    out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
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
    # bad M, T, S and the sum bound at create: the extreme tap set (T = 8192 taps of -2^31, S = 62) is within it
    p, rate, offs, ddc, x, _ = fdd.case_input("fm2b_f9_m8", seed=9)
    for bad in ((0, ddc[1], 15), (4097, ddc[1], 15), (8, np.ones(8193, np.int32), 15), (8, ddc[1], -1),
                (8, ddc[1], 63)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.FmMix(p, rate, offs, ddc=bad)
        assert e.value.code == _lib.EINVAL
    fm.FmMix(p, rate, offs, ddc=(8, np.full(8192, -(1 << 31), np.int32), 62)).close()
    # a chunk that is not a multiple of 2M, a decimated read too short for the passes (2^3), a half sample
    mx, fresh = fm.FmMix(p, rate, offs, ddc=ddc), fm.FmMix(p, rate, offs, ddc=ddc)
    a = mx.full_demod(x[:2 * 8 * 4096], 2 * 8 * 1024)
    b = fresh.full_demod(x[:2 * 8 * 4096], 2 * 8 * 1024)
    assert a.tobytes() == b.tobytes()
    rest = x[2 * 8 * 4096:]
    for call in (lambda: mx.full_demod(rest[:2 * 8 * 1024], 2 * 8 * 1024 + 2),
                 lambda: mx.full_demod(rest[:2 * 8 * 1024], 2 * 1001),
                 lambda: mx.process_read(rest[:2 * 60]),                   # 60 samples: 7 or 8 outputs < 2^3
                 lambda: mx.process_read(rest[:2 * 40]),
                 lambda: mx.process_read(rest[:31])):
        with pytest.raises(_lib.Rxb200Error) as e:
            call()
        assert e.value.code == _lib.EUNSUPPORTED
    assert mx.decimated_len(2 * 60) == 2 * 7
    assert mx.process_read(rest[:2 * 20011]).tobytes() == fresh.process_read(rest[:2 * 20011]).tobytes()
    mx.close()
    fresh.close()


def test_decimated_len_and_max_output_follow_the_model():
    p, rate, offs, ddc, x, reads = fdd.case_input("am_m100", seed=10)
    M = ddc[0]
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    pos = 0
    for a, n in fac.seq_bounds(x.size, reads + [2 * 99, 2 * 1, 2 * 150]):
        d = mx.decimated_len(n)
        assert d == fdd.decimated_len(pos, n, M), (a, n)
        bound = mx.max_output(n, max(n, 1))
        r = mx.process_read(x[a:a + n])
        assert r.shape[1] <= bound and mx.max_output(n, 2 * M * 16) >= 0
        pos += n // 2
    # a plain mixing handle: decimated_len is the identity, max_output the member's
    pm = fm.FmMix(p, rate, offs)
    assert pm.decimated_len(1234) == 1234
    assert pm.max_output(4096, 512) == _lib.lib().rxb200_fm_max_output(pm.member(), 4096, 512)
    pm.close()
    mx.close()


def test_golden():
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fdd.SHAPES)
    for name in sorted(fdd.SHAPES):
        p, rate, offs, ddc, x, reads = fdd.case_input(name)
        g = gold[name]
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        mx = fm.FmMix(p, rate, offs, ddc=ddc)
        got, counts = fh.reads(mx, x, g["lens_int16"])
        for j, c in enumerate(g["channels"]):
            assert c["offset_hz"] == offs[j]
            assert [n for n, d in zip(counts, c["dec_len"]) if d] == c["result_len"], (name, j)
            assert hashlib.sha256(got[j].tobytes()).hexdigest() == c["sha256"], (name, j)
        mx.close()
