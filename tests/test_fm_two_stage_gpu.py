"""Two-stage mixing handles (rxb200_fm_mix_create_two_stage) on the GPU: both stages alone (rxb200_two_stage_device)
against the numpy model over every int16 value, over K, M1 M2, T, the stateless sample index n0, source offsets and short
calls; both exact anchors byte for byte against rxb200_power_ddc_device and the raster handle; every named shape
through the handle against the port and the golden hashes; the carried state across reads, chunk calls and reset; a
call longer than one scratch group against short calls; the device entry points with an unaligned capture; and
refusals that leave no trace."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_handles as fh
import fm_two_stage as fts
from rx_tools_b200 import _lib, fm, power

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_two_stage_golden.json")


def _offsets(rate, K, seed):
    """Channels in several bins, two in one bin, one on a bin centre and one on a bin edge."""
    rng = np.random.default_rng(seed)
    step = rate // K
    offs = [int(v) for v in rng.integers(-(rate // 2) + 1, rate // 2, size=5)]
    return offs + [offs[0] + 1, step if 2 * step < rate else 0, step // 2]


def _taps(n_taps, seed, bound):
    rng = np.random.default_rng(seed)
    h = rng.integers(-bound // n_taps, bound // n_taps, size=n_taps, endpoint=False)
    h[0] = h[0] or 1
    return h.astype(np.int32)


# (K, M1, T1, M2, T2): M1 M2 up to 4096, T up to 8192
CASES = [(3, 1, 1, 1, 1), (3, 3, 17, 2, 9), (4, 2, 49, 4, 129), (4, 64, 8192, 64, 3), (768, 16, 385, 4, 129),
         (768, 1, 5, 4096, 7), (4096, 64, 129, 2, 8192), (4096, 4096, 9, 1, 1)]


@pytest.mark.parametrize("K,M1,T1,M2,T2", CASES)
def test_two_stage_device_equals_model(K, M1, T1, M2, T2):
    torch = fh.torch()
    rate = 2_048_000 if K != 3 else 1_008_000
    offs = _offsets(rate, K, K + M1 + T2)
    coarse = (M1, _taps(T1, K + T1, 1 << 22), 30)
    fine = (M2, _taps(T2, M2 + T2, 1 << 20), 19)
    M = M1 * M2
    x = fh.every_int16(K * 7 + M1 + T2)
    n_max = min(x.size // 2, max(M + 3, 60 * M))
    srcs = {off16: torch.from_numpy(np.concatenate([np.zeros(off16, np.int16), x[:2 * n_max]])).cuda()
            for off16 in (0, 2, 8)}
    dst = torch.zeros(len(offs) * 2 * (n_max // M) + 64, dtype=torch.int16, device="cuda")
    for n0 in ((1 << 64) - K + 1, (1 << 40) + 3):
        for n in sorted({n_max, M - 1, 2 * M + 1, 1}):
            for off16, src in (srcs.items() if n == n_max else [(0, srcs[0])]):
                if n < 1:
                    continue
                dst.fill_(0)
                fm.two_stage_device(rate, K, offs, n0, coarse, fine, src.data_ptr() + 2 * off16, n, dst.data_ptr())
                torch.cuda.synchronize()
                want = fts.two_stage_model(x[:2 * n], rate, K, offs, coarse, fine, n0)
                assert want.shape == (len(offs), 2 * (n // M))
                got = dst[:want.size].cpu().numpy().reshape(want.shape)
                bad = np.argwhere(got != want)
                assert bad.size == 0, (K, M1, T1, M2, T2, n0, off16, n, bad[:4])
                assert not dst[want.size:].any().item(), (K, M1, M2, n0, n)   # nothing past n / M outputs


def test_anchors_byte_for_byte():
    torch = fh.torch()
    rate, K = 2_400_000, 16
    x = fh.every_int16(4)[:2 * 40001]
    src = torch.from_numpy(x).cuda()
    a = torch.zeros(8 * 2 * 40001, dtype=torch.int16, device="cuda")
    b = torch.zeros_like(a)
    offs = [0, 17, -74_999, 74_998]
    for M2, T2, S2 in ((1, 1, 0), (4, 129, 15), (5, 64, 20)):
        fine = (M2, power.ddc_lowpass(M2, T2 | 1, S2) if T2 > 1 else np.ones(1, np.int32), S2)
        n_out = 40001 // M2
        for n0 in (0, 12345, (1 << 40) + 3):
            fm.two_stage_device(rate, K, offs, n0, (1, np.ones(1, np.int32), 15), fine, src.data_ptr(), 40001,
                                a.data_ptr())
            for c, f in enumerate(offs):
                _lib.check(_lib.lib().rxb200_power_ddc_device(rate, f, n0, fm._ddc_c(fine)[0], src.data_ptr(), 40001,
                                                              b.data_ptr() + 4 * c * n_out, None))
            torch.cuda.synchronize()
            k = 2 * n_out * len(offs)
            assert a[:k].cpu().numpy().tobytes() == b[:k].cpu().numpy().tobytes(), (M2, n0)
    # the unit fine stage at bin centres is the raster handle
    rate, K = 2_400_000, 48
    bins = [0, 1, 23, 47, 25, 1]
    offs = [int(k * rate // K) if 2 * k <= K else int((k - K) * rate // K) for k in bins]
    coarse = (3, fdd.lowpass(65, 0.02, gain_bits=20), 35)
    p = fac.with_(fac.RAW, downsample=1, offset_tuning=1)
    ts = fm.FmMix(p, rate, offs, two_stage=(K, coarse, (1, np.ones(1, np.int32), 0)))
    ra = fm.FmMix(p, ddc=coarse, raster=(K, bins))
    got, _ = fh.reads(ts, x, fdd.READS)
    want, _ = fh.reads(ra, x, fdd.READS)
    assert got.tobytes() == want.tobytes()
    ts.close()
    ra.close()


def _levels_params(p):
    q = fm.FmParams.from_any(p)
    q.report_levels = 1 if q.squelch_level else 0
    return q


@pytest.mark.parametrize("name", sorted(fts.SHAPES))
def test_shapes_equal_the_port(name, port):
    p, rate, K, offs, coarse, fine, x, reads = fts.case_input(name, seed=5)
    p = _levels_params(p)
    mx = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    got, counts = fh.reads(mx, x, reads)
    assert mx.mix_ms() > 0
    q = fac.P(**p.reference_fields())
    for c, dec in enumerate(fts.decimated_reads(x, rate, K, offs, coarse, fine, reads)):
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
    assert sorted(gold) == sorted(fts.SHAPES)
    for name in sorted(fts.SHAPES):
        p, rate, K, offs, coarse, fine, x, reads = fts.case_input(name)
        g = gold[name]
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        mx = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
        got, counts = fh.reads(mx, x, g["lens_int16"])
        for c, gc in enumerate(g["channels"]):
            assert [n for n, d in zip(counts, gc["dec_len"]) if d] == gc["result_len"], (name, c)
            assert hashlib.sha256(got[c].tobytes()).hexdigest() == gc["sha256"], (name, c)
        mx.close()


def _chain_lens(ops, M, pos=0):
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


@pytest.mark.parametrize("name", ["am_m100", "raw_sat_k3", "raw_centres_edges"])
def test_carries_across_reads_chunks_and_reset(name, port):
    p, rate, K, offs, coarse, fine, x, _ = fts.case_input(name, seed=6)
    M = coarse[0] * fine[0]
    ops = [("chunk", 2 * M * 30 + 2 * 77, 2 * M * 10), ("read", 2 * 4099), ("read", 2 * 5), ("read", 2 * (M - 1)),
           ("chunk", 2 * M * 20, 2 * M * 4), ("read", 2 * 30011), ("chunk", 2 * 333, 2 * M * 64)]
    x = np.concatenate([x, x])[:sum(op[1] for op in ops)]
    lens = _chain_lens(ops, M)
    mx = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    first = _run_ops(mx, x, ops)
    y = fts.two_stage_model(x, rate, K, offs, coarse, fine)
    for c in range(len(offs)):
        assert y[c].size == sum(lens)
        fh.compare(p, first[c], fac.port_run_seq(port, p, y[c], lens), (name, c))
    mx.reset()
    assert _run_ops(mx, x, ops).tobytes() == first.tobytes()
    mx.close()


def test_long_call_equals_short_calls():
    """K = 4096 with 4000 distinct bins and T2 = 8192: a few hundred coarse frames per scratch group, so one read of
    6000 coarse frames runs many groups; against the same capture in reads of at most 1000 samples."""
    p = fac.with_(fac.RAW, downsample=1, offset_tuning=1)
    rate, K = 4_096_000, 4096
    offs = [1000 * k - 2_000_000 + 7 for k in range(4000)]
    coarse, fine = (1, np.array([7, -3, 11, 2, -9], np.int32), 19), (2, _taps(8192, 3, 1 << 18), 15)
    x = fh.every_int16(9)[:2 * 6000]
    one = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    many = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    a = one.process_read(x)
    b, _ = fh.reads(many, x, [2 * 1000, 2 * 999, 2 * 1])
    assert a.tobytes() == b.tobytes()
    one.close()
    many.close()


def test_device_entries_with_an_unaligned_capture():
    torch = fh.torch()
    p, rate, K, offs, coarse, fine, x, reads = fts.case_input("fm2b_f9", seed=8)
    host = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    want_reads, _ = fh.reads(host, x, reads)
    host.reset()
    M = coarse[0] * fine[0]
    chunk = 2 * M * 4096
    n = (x.size // chunk) * chunk
    want_call = host.full_demod(x[:n], chunk)
    host.close()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()
    cap = buf[2:]
    assert cap.data_ptr() % 16 == 4
    mx = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
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
    p, rate, K, offs, coarse, fine, x, _ = fts.case_input("fm2b_f9", seed=9)
    M = coarse[0] * fine[0]
    for ts in ((2, coarse, fine), (K, (coarse[0], np.full(4, 1 << 20, np.int32), 30), fine),
               (K, coarse, (4096, fine[1], 15))):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.FmMix(p, rate, offs, two_stage=ts)
        assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(p, rate, offs + [rate // 2], two_stage=(K, coarse, fine))
    assert e.value.code == _lib.EINVAL
    mx = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    fresh = fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    a = mx.full_demod(x[:2 * M * 4096], 2 * M * 1024)
    assert a.tobytes() == fresh.full_demod(x[:2 * M * 4096], 2 * M * 1024).tobytes()
    rest = x[2 * M * 4096:]
    for call in (lambda: mx.full_demod(rest[:2 * M * 1024], 2 * M * 1024 + 2),
                 lambda: mx.process_read(rest[:2 * M * 7 + 2]),               # 7 outputs < 2^3 for the passes
                 lambda: mx.process_read(rest[:31])):
        with pytest.raises(_lib.Rxb200Error) as e:
            call()
        assert e.value.code == _lib.EUNSUPPORTED
    assert mx.decimated_len(2 * M * 7 + 2) == 2 * 7
    assert mx.process_read(rest[:2 * 20011]).tobytes() == fresh.process_read(rest[:2 * 20011]).tobytes()
    mx.close()
    fresh.close()
