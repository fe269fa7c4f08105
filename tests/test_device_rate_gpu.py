"""Capture handles with a resampler attached, on the GPU: every handle kind (rx_fm single stage, raster and two stages;
rx_sdr's three kinds in CS16 and CF32; rx_power) equals the composition byte for byte: the resampler's numpy model
(tests/resample.py) over the device stream, then the same handle without a resampler on its output, cut into the
calls the device calls emit.  The plans are 21/25 at J = 24 (int32, taps in shared memory), 187/256 at J = 136 (int64,
taps through the caches) and 25/21 (L > N).  Ragged device calls go through the host and device entries; attach after
a call is refused, reset keeps the resampler, refused calls change nothing, and the identity resampler gives the
unattached handle's bytes."""
import numpy as np
import pytest

import fm_handles as fh
import power_mix as pm
import resample as rsm
from rx_tools_b200 import _lib, fm, power, sdr
from rx_tools_b200 import resample as rs

pytestmark = pytest.mark.gpu

PLANS = {"21/25": (21, 25, 24), "187/256": (187, 256, 136), "25/21": (25, 21, 24)}
RAGGED = {"1": [1], "3": [3], "4093": [4093], "131072": [131072], "1000:7777": "rand"}
R = 2_016_000
OFFS = [-300_000, 0, 252_000, 504_000]
BINS = [0, 1, 3, 7]
P = fm.derive_params(rate_s=170_000).params


def _plan(name):
    L, N, J = PLANS[name]
    taps = rs.lowpass(L, N, J)
    if name != "25/21":
        assert rsm.wide(taps, L, 15) == (name == "187/256")
    return L, N, taps


def _stream(n_complex, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 6000, size=2 * n_complex).round().clip(-32768, 32767).astype(np.int16)
    x[:64] = rng.integers(-32768, 32768, 64)            # full-scale samples early: saturation paths
    return x


def _cuts(n_complex, pattern, seed):
    """Device-call lengths (complex samples) covering n_complex."""
    rng = np.random.default_rng(seed)
    out, at = [], 0
    while at < n_complex:
        c = int(rng.integers(1000, 7778)) if pattern == "rand" else pattern[len(out) % len(pattern)]
        c = min(c, n_complex - at)
        out.append(c)
        at += c
    return out


def _capture_cuts(cuts, L, N):
    """The capture samples each device call emits."""
    out, n0 = [], 0
    for c in cuts:
        out.append(rsm.out_count(n0, c, L, N))
        n0 += c
    return out


def _split(a16, lens):
    out, at = [], 0
    for n in lens:
        out.append(a16[2 * at:2 * (at + n)])
        at += n
    return out


# ---- rx_fm
def _fm_mix(kind):
    M = 8
    if kind == "single":
        return fm.FmMix(P, R, OFFS, ddc=(M, power.ddc_lowpass(M, 257, 15), 15))
    if kind == "raster":
        return fm.FmMix(P, ddc=(M, power.ddc_lowpass(M, 257, 15), 30), raster=(8, BINS))
    coarse = (2, power.ddc_lowpass(2, 49, 15), 30)
    fine = (4, power.ddc_lowpass(4, 129, 15), 15)
    return fm.FmMix(P, R, OFFS, two_stage=(4, coarse, fine))


def _fm_reads(mx, parts, device):
    torch = fh.torch()
    outs = []
    for x in parts:
        if not device:
            outs.append(mx.process_read(x))
            continue
        cap = mx.max_output(x.size, max(mx._capture_int16(x.size), 1)) + 8
        d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        d_out = torch.zeros((mx.n_channels, cap), dtype=torch.int16, device="cuda")
        n = mx.process_read_device(d_in.data_ptr(), x.size, d_out.data_ptr(), cap, sync=True)
        outs.append(d_out[:, :n].cpu().numpy())
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("kind", ["single", "raster", "two_stage"])
def test_fm_mix_equals_composition(kind, plan):
    L, N, taps = _plan(plan)
    x = _stream(60_000, 1)
    y = rsm.resample_model(x, L, N, taps, 15)[0]
    for name, pattern in RAGGED.items():
        if name in ("1", "3") and plan == "187/256":
            continue                                     # covered by the other plans; keeps the run short
        cuts = _cuts(x.size // 2 if name not in ("1", "3") else 3000, pattern, 7)
        xs = _split(x, cuts)
        ys = [v for v in _split(y, _capture_cuts(cuts, L, N)) if v.size]
        ref = _fm_mix(kind)
        want = _fm_reads(ref, ys, False)
        for device in (False, True):
            mx = _fm_mix(kind)
            mx.set_device_rate(L, N, taps, 15)
            got = _fm_reads(mx, xs, device)
            assert np.array_equal(got, want), (kind, plan, name, device)
            mx.close()
        ref.close()


def test_fm_mix_chunked_calls_equal_composition():
    L, N, taps = _plan("21/25")
    x = _stream(200_000, 2)
    y = rsm.resample_model(x, L, N, taps, 15)[0]
    cuts = [65_536, 80_000, 54_464]
    mx, ref = _fm_mix("single"), _fm_mix("single")
    mx.set_device_rate(L, N, taps, 15)
    for xa, ya in zip(_split(x, cuts), _split(y, _capture_cuts(cuts, L, N))):
        assert np.array_equal(mx.full_demod(xa, 4096), ref.full_demod(ya, 4096))
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


def _sdr_calls(mx, parts, fmt, device):
    torch = fh.torch()
    outs = []
    for x in parts:
        if not device:
            outs.append(mx.process(x, fmt))
            continue
        n = mx.decimated_len(x.size)
        E = sdr.ELEM_BYTES[fmt]
        stride = max(n, 1)
        d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        d_out = torch.zeros(mx.n_channels * stride * E, dtype=torch.uint8, device="cuda")
        got = mx.process_device(d_in.data_ptr(), x.size, fmt, d_out.data_ptr(), mx.n_channels * stride, stride)
        assert got == n
        o = d_out.cpu().numpy().view(sdr.DTYPES[fmt]).reshape(mx.n_channels, -1)
        outs.append(o[:, :2 * n])
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("fmt", [sdr.OUT_CS16, fm.CVT_CS16_CF32], ids=["CS16", "CF32"])
@pytest.mark.parametrize("kind", ["single", "raster", "two_stage"])
def test_sdr_mix_equals_composition(kind, fmt, plan):
    L, N, taps = _plan(plan)
    x = _stream(60_000, 3)
    y = rsm.resample_model(x, L, N, taps, 15)[0]
    ref = _sdr_mix(kind)
    want = ref.process(y, fmt)
    ref.close()
    for name, pattern in RAGGED.items():
        cuts = _cuts(x.size // 2 if name not in ("1", "3") else 3000, pattern, 9)
        n_cap = sum(_capture_cuts(cuts, L, N))
        for device in (False, True):
            mx = _sdr_mix(kind)
            mx.set_device_rate(L, N, taps, 15)
            got = _sdr_calls(mx, _split(x, cuts), fmt, device)
            w = want[:, :2 * (n_cap // 8)] if sum(cuts) < x.size // 2 else want
            assert np.array_equal(got, w), (kind, plan, name, device)
            mx.close()


def test_sdr_mix_host_call_over_several_groups():
    """A host call long enough for several staging groups (the device-rate upload, the resampled capture and the rows
    counted) equals the resampler handle followed by the unattached handle."""
    L, N, taps = _plan("21/25")
    x = np.random.default_rng(8).integers(-9000, 9000, size=2 * 16_000_000, dtype=np.int16)
    r = rs.Resampler(L, N, taps, 15)
    y = r.process(x)
    r.close()
    ref, mx = _sdr_mix("single"), _sdr_mix("single")
    mx.set_device_rate(L, N, taps, 15)
    assert np.array_equal(mx.process(x), ref.process(y))
    ref.close()
    mx.close()


# ---- rx_power
@pytest.mark.parametrize("plan", ["21/25", "187/256"])
def test_power_mix_equals_composition(plan):
    L, N, taps = _plan(plan)
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    pas = dd[0] * pl.buf_len // 2                       # capture samples per pass
    # device calls that resample to 1, 3 and 2 passes (L <= N: rxb200_resample_in_len is exact)
    cuts, n0 = [], 0
    for k in (1, 3, 2):
        c = rs.in_len(L, N, n0, k * pas)
        assert rsm.out_count(n0, c, L, N) == k * pas
        cuts.append(c)
        n0 += c
    x = _stream(n0, 4)
    y = rsm.resample_model(x, L, N, taps, 15)[0]
    ref = power.PowerMix(pl, Rp, offs, dd, win)
    ref.accumulate(y)
    want = ref.read()
    for device in (False, True):
        mx = power.PowerMix(pl, Rp, offs, dd, win)
        mx.set_device_rate(L, N, taps, 15)
        torch = fh.torch()

        def call(xa):
            if device:
                d = torch.from_numpy(np.ascontiguousarray(xa)).cuda()
                mx.accumulate_device(d.data_ptr(), xa.size, sync=True)
            else:
                mx.accumulate(xa)

        at = 0
        for k, c in enumerate(cuts):
            if k == 1:
                # between two calls, refused calls change nothing: one whose device samples resample to between 1 and
                # pas - 1 capture samples (in_len is the fewest that reach a whole pass), and an odd one
                short = rs.in_len(L, N, at, pas) - 1
                assert 0 < rsm.out_count(at, short, L, N) < pas
                for bad in (x[2 * at:2 * (at + short)], x[2 * at:2 * (at + c) - 1]):
                    with pytest.raises(_lib.Rxb200Error) as e:
                        call(bad)
                    assert e.value.code == _lib.EUNSUPPORTED
                with pytest.raises(_lib.Rxb200Error) as e:
                    mx.accumulate_burst(0, 1, np.zeros(mx.burst_int16(1), np.int16))
                assert e.value.code == _lib.EUNSUPPORTED
            call(x[2 * at:2 * (at + c)])
            at += c
        got = mx.read()
        assert all(np.array_equal(u, v) for u, v in zip(got, want)), (plan, device)
        assert mx.kernel_ms() >= 0
        mx.close()
    ref.close()


# ---- attach, reset, refusals, identity
def test_attach_rules_reset_and_refusals():
    L, N, taps = _plan("21/25")
    x = _stream(40_000, 5)
    for make in (lambda: _fm_mix("single"), lambda: _sdr_mix("single")):
        h = make()
        bad = np.zeros(L * 24, np.int32)
        with pytest.raises(_lib.Rxb200Error) as e:
            h.set_device_rate(0, N, bad, 15)                     # rxb200_resample_create's refusal
        assert e.value.code == _lib.EINVAL
        h.set_device_rate(L, N, taps, 15)
        with pytest.raises(_lib.Rxb200Error):
            h.set_device_rate(L, N, taps, 15)                    # once only
        first = h.process_read(x) if isinstance(h, fm.FmMix) else h.process(x)
        with pytest.raises(_lib.Rxb200Error) as e:
            h.set_device_rate(L, N, taps, 15)                    # after a call
        assert e.value.code == _lib.EINVAL
        # a refused call (odd length, the handle's own code) changes nothing: reset, then the same stream gives the
        # same bytes
        h.reset()
        with pytest.raises(_lib.Rxb200Error) as e:
            if isinstance(h, fm.FmMix):
                h.process_read(x[:-1])
            else:
                h.process(x[:-1])
        assert e.value.code == (_lib.EUNSUPPORTED if isinstance(h, fm.FmMix) else _lib.EINVAL)
        again = h.process_read(x) if isinstance(h, fm.FmMix) else h.process(x)
        assert np.array_equal(first, again)
        h.close()
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    p = power.PowerMix(pl, Rp, offs, dd, win)
    p.accumulate(np.zeros(dd[0] * pl.buf_len, np.int16))
    with pytest.raises(_lib.Rxb200Error) as e:
        p.set_device_rate(L, N, taps, 15)
    assert e.value.code == _lib.EINVAL
    p.reset()
    p.set_device_rate(L, N, taps, 15)
    p.close()


def test_identity_resampler_is_the_unattached_handle():
    one = np.array([1 << 15], np.int32)
    x = _stream(50_000, 6)
    for kind in ("single", "raster", "two_stage"):
        a, b = _fm_mix(kind), _fm_mix(kind)
        a.set_device_rate(1, 1, one, 15)
        assert np.array_equal(a.process_read(x), b.process_read(x)), kind
        a.close()
        b.close()
        for fmt in (sdr.OUT_CS16, fm.CVT_CS16_CF32):
            a, b = _sdr_mix(kind), _sdr_mix(kind)
            a.set_device_rate(1, 1, one, 15)
            assert np.array_equal(a.process(x, fmt), b.process(x, fmt)), (kind, fmt)
            a.close()
            b.close()
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    xp = pm.capture(2 * dd[0] * pl.buf_len // 2, Rp, offs, 77)
    a, b = power.PowerMix(pl, Rp, offs, dd, win), power.PowerMix(pl, Rp, offs, dd, win)
    a.set_device_rate(1, 1, one, 15)
    a.accumulate(xp)
    b.accumulate(xp)
    assert all(np.array_equal(u, v) for u, v in zip(a.read(), b.read()))
    a.close()
    b.close()
