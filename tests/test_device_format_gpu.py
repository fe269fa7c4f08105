"""Capture handles in a device's own format, on the GPU.  The widening kinds of rxb200_sdr_convert_device equal the numpy
rule (tests/device_format.py) over every byte value at every source offset; and every capture handle kind (rx_fm plain,
single stage, raster and two stages; rx_sdr's three kinds in CS16 and CF32; rx_power's stream calls and bursts), fed a
CS8, CU8 or CS12 stream, gives byte for byte what the same handle gives on the stream's CS16 widening, with and without
a resampler, over ragged host and device calls, device captures at byte offsets 0-3 and a host call of several
staging groups.  Reset keeps the format; setting it after a call is refused and changes nothing."""
import numpy as np
import pytest

import device_format as df
import fm_handles as fh
import power_mix as pm
from rx_tools_b200 import _lib, fm, power, sdr
from rx_tools_b200 import resample as rs

pytestmark = pytest.mark.gpu

R = 2_016_000
OFFS = [-300_000, 0, 252_000, 504_000]
BINS = [0, 1, 3, 7]
P = fm.derive_params(rate_s=170_000).params
RATE = (21, 25, 24)                      # a device-rate plan: L/N = 21/25, J = 24
FMTS = list(df.FORMATS)


def _cuts(n_complex, seed):
    """Ragged call lengths (complex elements) covering n_complex: 1, 3 and odd lengths, then random ones."""
    rng = np.random.default_rng(seed)
    out, at = [], 0
    for c in [1, 3, 4093]:
        out.append(min(c, n_complex - at))
        at += out[-1]
    while at < n_complex:
        out.append(min(int(rng.integers(1000, 7778)), n_complex - at))
        at += out[-1]
    return [c for c in out if c]


def _parts(b, fmt, cuts):
    """The narrow bytes of each call, and the CS16 widening of the same calls."""
    e, out, wide, at = df.ELEM[fmt], [], [], 0
    for c in cuts:
        out.append(b[e * at:e * (at + c)])
        wide.append(df.widen(out[-1], fmt))
        at += c
    return out, wide


def _dev(torch, a, off):
    """a's bytes in device memory at byte offset off of a fresh buffer; (buffer, pointer)."""
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    d = torch.zeros(raw.size + 8, dtype=torch.uint8, device="cuda")
    if raw.size:
        d[off:off + raw.size] = torch.from_numpy(raw).cuda()
    return d, d.data_ptr() + off


def _resampler(h):
    L, N, J = RATE
    h.set_device_rate(L, N, rs.lowpass(L, N, J), 15)


# ---- the kernel
@pytest.mark.parametrize("fmt", FMTS)
def test_convert_kinds_every_byte_every_offset(fmt):
    torch = fh.torch()
    kind = {"CS8": 5, "CU8": 6, "CS12": fm.CVT_CS12_CS16}[fmt]
    e = df.ELEM[fmt]
    rng = np.random.default_rng(3)
    every = np.tile(np.arange(256, dtype=np.uint8), 3 * 64)                        # every byte at every position
    for n in (1, 7, 8, 15, 16, 17, 4095, (every.size // e), 1_000_003):
        b = np.concatenate([every, rng.integers(0, 256, e * n, dtype=np.uint8)])[:e * n] if n > every.size // e \
            else every[:e * n]
        want = df.widen(b, fmt)
        for off in range(4):
            d_in, p = _dev(torch, b, off)
            d_out = torch.zeros(2 * n + 8, dtype=torch.int16, device="cuda")
            _lib.check(_lib.lib().rxb200_sdr_convert_device(kind, p, n, d_out.data_ptr(), None))
            torch.cuda.synchronize()
            assert np.array_equal(d_out[:2 * n].cpu().numpy(), want), (fmt, n, off)
            assert not d_out[2 * n:].any()
        # the host entry
        out = np.zeros(2 * n, np.int16)
        _lib.check(_lib.lib().rxb200_sdr_convert(kind, b.ctypes.data, n, out.ctypes.data, 0))
        assert np.array_equal(out, want), (fmt, n)
    # a destination that is not 4-byte aligned is refused; 4 and 7 are not widening kinds
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    assert _lib.lib().rxb200_sdr_convert_device(kind, d.data_ptr(), 4, d.data_ptr() + 2, None) == _lib.EINVAL
    for bad in (4, 7, -1):
        assert _lib.lib().rxb200_sdr_convert_device(bad, d.data_ptr(), 4, d.data_ptr(), None) == _lib.EINVAL


# ---- rx_fm
def _fm_mix(kind):
    M = 8
    if kind == "plain":
        return fm.FmMix(P, R, OFFS[:2])
    if kind == "single":
        return fm.FmMix(P, R, OFFS, ddc=(M, power.ddc_lowpass(M, 257, 15), 15))
    if kind == "raster":
        return fm.FmMix(P, ddc=(M, power.ddc_lowpass(M, 257, 15), 30), raster=(8, BINS))
    coarse = (2, power.ddc_lowpass(2, 49, 15), 30)
    fine = (4, power.ddc_lowpass(4, 129, 15), 15)
    return fm.FmMix(P, R, OFFS, two_stage=(4, coarse, fine))


def _fm_reads(mx, parts, device, off=0):
    torch = fh.torch()
    outs = []
    for x in parts:
        if not device:
            outs.append(mx.process_read(x))
            continue
        _a, n16 = _lib.in_array(x, getattr(mx, "_in_fmt", _lib.IN_CS16))
        cap = mx.max_output(n16, max(mx._capture_int16(n16), 1)) + 8
        d_in, p = _dev(torch, x, off)
        d_out = torch.zeros((mx.n_channels, cap), dtype=torch.int16, device="cuda")
        n = mx.process_read_device(p, n16, d_out.data_ptr(), cap, sync=True)
        outs.append(d_out[:, :n].cpu().numpy())
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("rate", [False, True], ids=["capture", "device_rate"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["plain", "single", "raster", "two_stage"])
def test_fm_mix_equals_widened(kind, fmt, rate):
    b = df.narrow_stream(60_000, fmt, 1)
    xs, ws = _parts(b, fmt, _cuts(60_000, 2))
    ref = _fm_mix(kind)
    if rate:
        _resampler(ref)
    want = _fm_reads(ref, ws, False)
    ref.close()
    for device, off in ((False, 0), (True, 0), (True, 1), (True, 2), (True, 3)):
        if kind == "plain" and off in (1, 2):
            continue                                         # the other kinds cover them; keeps the run short
        mx = _fm_mix(kind)
        mx.set_input_format(fmt)
        if rate:
            _resampler(mx)                                   # after the format: either order
        got = _fm_reads(mx, xs, device, off)
        assert np.array_equal(got, want), (kind, fmt, rate, device, off)
        mx.close()


def test_fm_mix_chunked_calls_equal_widened():
    b = df.narrow_stream(200_000, "CU8", 2)
    mx, ref = _fm_mix("single"), _fm_mix("single")
    mx.set_input_format("CU8")
    for c0, c1 in ((0, 65_536), (65_536, 145_536), (145_536, 200_000)):
        part = b[2 * c0:2 * c1]
        assert np.array_equal(mx.full_demod(part, 4096), ref.full_demod(df.widen(part, "CU8"), 4096))
    mx.close()
    ref.close()


# ---- rx_sdr
def _sdr_mix(kind):
    M = 8
    if kind == "single":
        return sdr.SdrMix(R, OFFS, ddc=(M, power.ddc_lowpass(M, 257, 15), 15))
    if kind == "raster":
        return sdr.SdrMix(ddc=(M, power.ddc_lowpass(M, 257, 15), 30), raster=(8, BINS))
    coarse = (2, power.ddc_lowpass(2, 49, 15), 30)
    fine = (4, power.ddc_lowpass(4, 129, 15), 15)
    return sdr.SdrMix(R, OFFS, two_stage=(4, coarse, fine))


def _sdr_calls(mx, parts, fmt, device, off=0):
    torch = fh.torch()
    outs = []
    for x in parts:
        if not device:
            outs.append(mx.process(x, fmt))
            continue
        _a, n16 = _lib.in_array(x, getattr(mx, "_in_fmt", _lib.IN_CS16))
        n = mx.decimated_len(n16)
        E = sdr.ELEM_BYTES[fmt]
        stride = max(n, 1)
        d_in, p = _dev(torch, x, off)
        d_out = torch.zeros(mx.n_channels * stride * E, dtype=torch.uint8, device="cuda")
        got = mx.process_device(p, n16, fmt, d_out.data_ptr(), mx.n_channels * stride, stride)
        assert got == n
        o = d_out.cpu().numpy().view(sdr.DTYPES[fmt]).reshape(mx.n_channels, -1)
        outs.append(o[:, :2 * n])
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("rate", [False, True], ids=["capture", "device_rate"])
@pytest.mark.parametrize("out", [sdr.OUT_CS16, fm.CVT_CS16_CF32], ids=["CS16", "CF32"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["single", "raster", "two_stage"])
def test_sdr_mix_equals_widened(kind, fmt, out, rate):
    b = df.narrow_stream(60_000, fmt, 3)
    xs, ws = _parts(b, fmt, _cuts(60_000, 4))
    ref = _sdr_mix(kind)
    if rate:
        _resampler(ref)
    want = _sdr_calls(ref, ws, out, False)
    ref.close()
    for device, off in ((False, 0), (True, 0), (True, 1), (True, 2), (True, 3)):
        mx = _sdr_mix(kind)
        if rate:
            _resampler(mx)                                   # before the format: either order
        mx.set_input_format(fmt)
        got = _sdr_calls(mx, xs, out, device, off)
        assert np.array_equal(got, want), (kind, fmt, out, rate, device, off)
        mx.close()


@pytest.mark.parametrize("rate", [False, True], ids=["capture", "device_rate"])
@pytest.mark.parametrize("fmt", ["CU8", "CS12"])
def test_sdr_mix_host_call_over_several_groups(fmt, rate):
    """One host call of 24 M elements crosses RXB200_SDR_MIX_SCRATCH_BYTES (the upload, its widening and the rows
    counted) and equals the widened stream in one call of a CS16 handle."""
    rng = np.random.default_rng(8)
    b = rng.integers(0, 256, size=df.ELEM[fmt] * 24_000_000, dtype=np.uint8)
    ref, mx = _sdr_mix("single"), _sdr_mix("single")
    if rate:
        _resampler(ref)
        _resampler(mx)
    mx.set_input_format(fmt)
    assert np.array_equal(mx.process(b), ref.process(df.widen(b, fmt)))
    ref.close()
    mx.close()


# ---- rx_power
def _power_call(mx, x, device, off, burst=None):
    torch = fh.torch()
    _a, n16 = _lib.in_array(x, getattr(mx, "_in_fmt", _lib.IN_CS16))
    if not device:
        return mx.accumulate(x) if burst is None else mx.accumulate_burst(*burst, x)
    d, p = _dev(torch, x, off)
    if burst is None:
        mx.accumulate_device(p, n16, sync=True)
    else:
        mx.accumulate_burst_device(*burst, p, n16, sync=True)


@pytest.mark.parametrize("rate", [False, True], ids=["capture", "device_rate"])
@pytest.mark.parametrize("fmt", FMTS)
def test_power_mix_stream_equals_widened(fmt, rate):
    L, N, J = RATE
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    pas = dd[0] * pl.buf_len // 2                       # capture samples per pass
    cuts, n0 = [], 0
    for k in (1, 3, 2):
        c = rs.in_len(L, N, n0, k * pas) if rate else k * pas
        cuts.append(c)
        n0 += c
    b = df.narrow_stream(n0, fmt, 5)
    xs, ws = _parts(b, fmt, cuts)
    ref = power.PowerMix(pl, Rp, offs, dd, win)
    if rate:
        _resampler(ref)
    for w in ws:
        ref.accumulate(w)
    want = ref.read()
    ref.close()
    for device, off in ((False, 0), (True, 0), (True, 1), (True, 3)):
        mx = power.PowerMix(pl, Rp, offs, dd, win)
        mx.set_input_format(fmt)
        if rate:
            _resampler(mx)
        for x in xs:
            _power_call(mx, x, device, off)
        got = mx.read()
        assert all(np.array_equal(u, v) for u, v in zip(got, want)), (fmt, rate, device, off)
        assert mx.kernel_ms() >= 0
        mx.close()


@pytest.mark.parametrize("rate", [False, True], ids=["capture", "burst_rate"])
@pytest.mark.parametrize("fmt", FMTS)
def test_power_mix_bursts_equal_widened(fmt, rate):
    L, N, J = RATE
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    nh = len(offs)
    ranges = [(0, nh), (1, max(2, nh // 2)), (nh - 1, nh)]

    def make(f):
        h = power.PowerMix(pl, Rp, offs, dd, win)
        if f:
            h.set_input_format(f)
        if rate:
            h.set_burst_device_rate(L, N, rs.lowpass(L, N, J), 15)
        return h

    ref = make(None)
    n_el = [ref.burst_in_len(p) // 2 for p in (1, 2, 1)]
    bursts = [df.narrow_stream(n, fmt, 20 + k) for k, n in enumerate(n_el)]
    for (hb, he), bb in zip(ranges, bursts):
        ref.accumulate_burst(hb, he, df.widen(bb, fmt))
    want = ref.read()
    ref.close()
    for device, off in ((False, 0), (True, 0), (True, 2)):
        mx = make(fmt)
        for (hb, he), bb in zip(ranges, bursts):
            _power_call(mx, bb, device, off, burst=(hb, he))
        got = mx.read()
        assert all(np.array_equal(u, v) for u, v in zip(got, want)), (fmt, rate, device, off)
        mx.close()


# ---- when the format can be set, reset, refusals
def test_set_after_samples_is_refused_and_reset_keeps_the_format():
    b = df.narrow_stream(40_000, "CS8", 6)
    w = df.widen(b, "CS8")
    for make in (lambda: _fm_mix("single"), lambda: _sdr_mix("raster")):
        h, ref = make(), make()
        call = (lambda a, x: a.process_read(x)) if isinstance(h, fm.FmMix) else (lambda a, x: a.process(x))
        for bad in (-1, 4, 99):
            with pytest.raises(_lib.Rxb200Error) as e:
                h.set_input_format(bad)
            assert e.value.code == _lib.EINVAL
        h.set_input_format("CS8")
        first = call(h, b)
        assert np.array_equal(first, call(ref, w))
        setter = "rxb200_fm_mix_set_input_format" if isinstance(h, fm.FmMix) else "rxb200_sdr_mix_set_input_format"
        with pytest.raises(_lib.Rxb200Error) as e:
            _lib.check(getattr(_lib.lib(), setter)(h._h, _lib.IN_CS16))
        assert e.value.code == _lib.EINVAL
        # the refused setter changed nothing: the stream continues in CS8
        b2 = df.narrow_stream(10_000, "CS8", 7)
        assert np.array_equal(call(h, b2), call(ref, df.widen(b2, "CS8")))
        # reset keeps CS8
        h.reset()
        assert np.array_equal(call(h, b), first)
        h.close()
        ref.close()
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    p = power.PowerMix(pl, Rp, offs, dd, win)
    p.set_input_format("CU8")
    p.accumulate_burst(0, 1, np.zeros(2 * (p.burst_int16(1) // 2), np.uint8))   # a burst takes samples too
    with pytest.raises(_lib.Rxb200Error) as e:
        _lib.check(_lib.lib().rxb200_power_mix_set_input_format(p._m, _lib.IN_CS16))
    assert e.value.code == _lib.EINVAL
    # a narrow stream of an odd n_int16 is refused
    assert _lib.lib().rxb200_power_mix_accumulate(p._m, np.zeros(8, np.uint8).ctypes.data, 7) == _lib.EUNSUPPORTED
    p.reset()
    x = df.narrow_stream(dd[0] * pl.buf_len // 2, "CU8", 9)
    p.accumulate(x)                                            # still CU8 after reset
    q = power.PowerMix(pl, Rp, offs, dd, win)
    q.accumulate(df.widen(x, "CU8"))
    assert all(np.array_equal(u, v) for u, v in zip(p.read(), q.read()))
    p.close()
    q.close()
