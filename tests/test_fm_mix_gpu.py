"""Several rx_fm channels of one capture (rxb200_fm_mix_*) on the GPU: the mixer kernel alone against the numpy model over
every int16 value, a zero offset against a plain handle on every kernel route, K channels against the port on the
model's mixed streams, the phase across calls, reads and reset, the device entry points with an unaligned capture,
refusals that leave the phases and the member alone, and the golden hashes of the reference."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_handles as fh
import fm_mix as fmx
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_mix_golden.json")


@pytest.mark.parametrize("rate,f", [(2_400_000, 12500), (2_400_000, -37500), (1_008_000, 24000), (48_000, 7),
                                    (2_400_000, 600_000), (2_400_000, 0), (1 << 20, 1)])
def test_mix_device_equals_model(rate, f):
    torch = fh.torch()
    x = fh.every_int16(rate % 1000 + f % 1000)
    t = fm.mix_table(rate, f)
    L = t.shape[0]
    src = torch.from_numpy(np.concatenate([np.zeros(8, np.int16), x])).cuda()
    dst = torch.zeros(x.size + 16, dtype=torch.int16, device="cuda")
    for phase in (0, L - 1, (1 << 40) + 3):
        for off16 in (0, 2, 8):                         # source at 0 / 4 / 16 bytes
            for n in (65536, 65535, 65533, 9, 1):       # odd complex counts, a partial last unit, a lone sample
                dst.fill_(0)
                s = src[8 - off16:]
                # destination at the source's alignment: 16-byte vectors when both are aligned, else 4-byte accesses
                d = dst[8 - off16:]
                fm.mix_device(rate, f, phase, s.data_ptr() + 2 * off16, n, d.data_ptr())
                torch.cuda.synchronize()
                got = d[:2 * n].cpu().numpy()
                want = fmx.mix_model(x[:2 * n], t, phase % L)
                bad = np.flatnonzero(got != want)
                assert bad.size == 0, (rate, f, phase, off16, n, bad[:4])
                assert not d[2 * n:2 * n + 8].any().item(), (rate, f, phase, off16, n)   # nothing past the end


def test_mix_device_refusals():
    torch = fh.torch()
    buf = torch.zeros(64, dtype=torch.int16, device="cuda")
    p = buf.data_ptr()
    for args, code in (((2_400_000, 1_200_000, 0, p, 8, p), _lib.EINVAL), ((2_400_001, 1, 0, p, 8, p), _lib.EUNSUPPORTED),
                       ((2_400_000, 0, -1, p, 8, p), _lib.EINVAL), ((2_400_000, 0, 0, p + 2, 8, p), _lib.EINVAL),
                       ((2_400_000, 0, 0, None, 8, p), _lib.EINVAL)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.mix_device(*args)
        assert e.value.code == code, args


@pytest.mark.parametrize("name", sorted(fh.KERNEL_ROUTES))
def test_zero_offset_is_a_plain_handle(name):
    """Channel f = 0 of a two-channel handle is byte for byte a plain one-channel handle on the capture, on the route
    the plain handle takes."""
    p, mode, chunk, lens, kind = fh.KERNEL_ROUTES[name]
    x = fac.signal(sum(lens) // 2, 40)
    mx = fm.FmMix(p, 2_400_000, [0, 300_000])
    d = fm.FmDemod(p)
    pos = 0
    for c, n in enumerate(lens):
        part = x[pos:pos + n]
        if mode == "read":
            got, want = mx.process_read(part), d.process_read(part)
        else:
            (got, gl), (want, wl) = mx.full_demod(part, chunk, True), d.full_demod(part, chunk, True)
            assert gl.tolist() == wl.tolist(), (name, c)
        assert got[0].tobytes() == want.tobytes(), (name, c)
        assert d.stats()["kernel_kind"] == kind and mx.stats()["kernel_kind"] == kind, (name, c, mx.stats())
        pos += n
    mx.close()
    d.close()


@pytest.mark.parametrize("k", [1, 3, 8, 33])
def test_k_channels_equal_the_port(k, port):
    p, rate, _, _ = fmx.case_input("fm5a_lut_d100")
    offs = [12500 * (j - k // 2) for j in range(k)]                       # a 12.5 kHz raster, up to +-200 kHz
    x = fmx.capture(fmx.n_complex_for(fmx.READS), rate, offs[::5], 800 + k)
    mx = fm.FmMix(p, rate, offs)
    got, _ = fh.reads(mx, x, fmx.READS)
    for j, (want, _, wh) in enumerate(fh.port_channels(port, p, rate, offs, x, fmx.READS)):
        fh.compare(p, got[j], want, (k, offs[j]))
        assert mx.squelch_hits()[j] == wh[-1]
    mx.close()


@pytest.mark.parametrize("name", sorted(fmx.SHAPES))
def test_shapes_equal_the_port(name, port):
    """Every shape of the CPU pins, read by read, with squelch hits and -L levels."""
    p, rate, offs, x = fmx.case_input(name, seed=5)
    p = fm.FmParams.from_any(p)
    p.report_levels = 1 if p.squelch_level else 0
    mx = fm.FmMix(p, rate, offs)
    got, _ = fh.reads(mx, x, fmx.READS)
    ref = fh.port_channels(port, fac.P(**fm.FmParams.from_any(p).reference_fields()), rate, offs, x, fmx.READS)
    for j, (want, _, wh) in enumerate(ref):
        fh.compare(p, got[j], want, (name, offs[j]))
        assert mx.squelch_hits()[j] == wh[-1], (name, j)
    if p.report_levels:
        # -L of the last read against the port's level of that read
        q = fac.P(**fm.FmParams.from_any(p).reference_fields())
        lv = mx.levels()
        for j, f in enumerate(offs):
            y = fmx.mix_model(x, fm.mix_table(rate, f))
            assert lv[j, -1] == fac.port_levels_seq(port, q, y, fmx.READS)[-1], (name, j)
    mx.close()


def test_phase_across_calls_reads_and_reset(port):
    p, rate, offs, x = fmx.case_input("fm5a_lut_d100", seed=6)
    c16 = 2 * 1021
    mx = fm.FmMix(p, rate, offs)
    one = mx.full_demod(x, c16)
    mx.reset()
    # several calls, each a whole number of chunks but the last
    cuts = [0, 3 * c16, 4 * c16, 11 * c16, x.size]
    several = np.concatenate([mx.full_demod(x[a:b], c16) for a, b in zip(cuts, cuts[1:])], axis=1)
    assert several.tobytes() == one.tobytes()
    mx.reset()
    reads, _ = fh.reads(mx, x, [c16])
    assert reads.tobytes() == one.tobytes()
    # ragged reads (1021:333:4093), twice with a reset between: the phases restart at 0
    mx.reset()
    first, counts = fh.reads(mx, x, fmx.READS)
    mx.reset()
    again, _ = fh.reads(mx, x, fmx.READS)
    assert again.tobytes() == first.tobytes()
    for j, (want, rl, _) in enumerate(fh.port_channels(port, p, rate, offs, x, fmx.READS)):
        assert first[j].tobytes() == want.tobytes() and counts == rl.tolist(), j
    mx.close()


@pytest.mark.parametrize("name", ["fm5a_lut_d100", "fm2b_f9"])
def test_device_entries_with_an_unaligned_capture(name):
    torch = fh.torch()
    p, rate, offs, x = fmx.case_input(name, seed=7)
    host = fm.FmMix(p, rate, offs)
    want_reads, counts = fh.reads(host, x, fmx.READS)
    host.reset()
    chunk = 2 * 4096 if p.downsample_passes else 2 * 1021
    n = (x.size // chunk) * chunk
    want_call = host.full_demod(x[:n], chunk)
    host.close()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()
    cap = buf[2:]                                        # 4 bytes past a 256-byte aligned allocation
    assert cap.data_ptr() % 16 == 4
    mx = fm.FmMix(p, rate, offs)
    stride = want_reads.shape[1] + 8
    out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
    parts = []
    for pos, n16 in fac.seq_bounds(x.size, fmx.READS):
        k = mx.process_read_device(cap.data_ptr() + 2 * pos, n16, out.data_ptr(), stride, sync=True)
        parts.append(out[:, :k].cpu().numpy())
    assert np.concatenate(parts, axis=1).tobytes() == want_reads.tobytes()
    mx.reset()
    k = mx.process_device(cap.data_ptr(), n, chunk, out.data_ptr(), stride)
    torch.cuda.synchronize()
    assert k == want_call.shape[1] and out[:, :k].cpu().numpy().tobytes() == want_call.tobytes()
    mx.close()


def test_refusals_leave_state_alone(port):
    torch = fh.torch()
    p, rate, offs, kw = fmx.SHAPES["fm2b_f9"]
    chunk = 8 * 2048
    x = fmx.capture(3 * chunk // 2, rate, offs, 8, **kw)
    mx = fm.FmMix(p, rate, offs)
    a = mx.full_demod(x[:chunk], chunk)
    rest = np.ascontiguousarray(x[chunk:chunk + 2 * chunk])
    for call, code in ((lambda: mx.full_demod(rest[:2 * 1001], 2 * 1001), _lib.EUNSUPPORTED),   # off the granule
                       (lambda: mx.process_read(rest[:31]), _lib.EUNSUPPORTED)):               # half a sample
        with pytest.raises(_lib.Rxb200Error) as e:
            call()
        assert e.value.code == code
    assert fh.raw_process(mx, rest, chunk, 1) == _lib.ECAPACITY
    assert fh.raw_process(mx, rest, chunk, 1 << 16, pcm=False) == _lib.EINVAL
    assert _lib.lib().rxb200_fm_mix_process(mx._h, None, rest.size, chunk, rest.ctypes.data, 1 << 16, None,
                                            None) == _lib.EINVAL
    d_in = torch.from_numpy(np.concatenate([np.zeros(1, np.int16), rest])).cuda()
    d_out = torch.zeros(1 << 16, dtype=torch.int16, device="cuda")
    with pytest.raises(_lib.Rxb200Error) as e:                  # a capture at a 2-byte offset
        mx.process_device(d_in.data_ptr() + 2, rest.size, chunk, d_out.data_ptr(), 1 << 14)
    assert e.value.code == _lib.EINVAL
    b = mx.full_demod(rest, chunk)
    want = fh.port_channels(port, p, rate, offs, x[:3 * chunk], [chunk])
    for j in range(len(offs)):
        assert np.concatenate([a[j], b[j]]).tobytes() == want[j][0].tobytes(), j
    mx.close()
    # per-chunk reduction stages: a last chunk of 4 complex samples makes no decimated sample, so the call is refused
    # before the mixer runs; levels and the phases stay
    q = fm.FmParams.from_any(fmx.SHAPES["fm_lut_d42_squelch"][0])
    q.report_levels = 1
    rate, offs = 1_008_000, [-20000, 20000]
    x = fmx.capture(6000, rate, offs, 9, quiet_half=True)
    mx = fm.FmMix(q, rate, offs)
    a = mx.full_demod(x[:2 * 3000], 2 * 1000)
    lv = mx.levels()
    with pytest.raises(_lib.Rxb200Error) as e:
        mx.full_demod(x[2 * 3000:2 * 3000 + 2 * 1004], 2 * 1000)
    assert e.value.code == _lib.EUNSUPPORTED
    assert mx.levels().tolist() == lv.tolist()
    b = mx.full_demod(x[2 * 3000:], 2 * 1000)
    qr = fac.P(**q.reference_fields())
    for j, f in enumerate(offs):
        y = fmx.mix_model(x, fm.mix_table(rate, f))
        assert np.concatenate([a[j], b[j]]).tobytes() == port.fm_run(qr, y, 2 * 1000).tobytes(), j
    mx.close()


def test_golden():
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fmx.SHAPES)
    for name in sorted(fmx.SHAPES):
        p, rate, offs, x = fmx.case_input(name)
        g = gold[name]
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        mx = fm.FmMix(p, rate, offs)
        got, counts = fh.reads(mx, x, g["lens_int16"])
        for j, c in enumerate(g["channels"]):
            assert c["offset_hz"] == offs[j]
            if fac.INTEGER(p):
                assert counts == c["result_len"], (name, j)
                assert hashlib.sha256(got[j].tobytes()).hexdigest() == c["sha256"], (name, j)
            else:
                assert counts == c["result_len"], (name, j)      # fp64 atan2: the port pins the bytes (above)
        mx.close()
