"""The rational resampler on the GPU: rxb200_resample_device against the numpy model over every int16 value in I and Q
for many up/down ratios, taps per phase and both accumulators, at device counts near 0, 2^40 and 2^64, from sources at
0-, 4- and 16-byte offsets, with guard words past the outputs and calls too short to emit one; both anchors byte for
byte (the identity, and L = 1 against rxb200_ddc_device with M - 1 leading zeros); and the handle: read patterns through
the host and device entries against one call, a host call over several scratch groups, reset, and refused calls that
leave the count and the history as they were."""
import numpy as np
import pytest

import fm_handles as fh
import resample as rm
from rx_tools_b200 import _lib, fm, resample

pytestmark = pytest.mark.gpu

RATIOS = [(1, 1), (1, 7), (7, 1), (5, 8), (21, 25), (504, 625), (187, 256), (2125, 3072)]
JS = [1, 8, 24, 192, 1024]
N0S = [0, (1 << 40) + 3, (1 << 64) - (1 << 20)]
GUARD = 0x7A7A


def _taps(rng, L, J, wide):
    """Random taps whose accumulator is int64 (wide) or int32, with the shift that keeps outputs mostly unsaturated."""
    if wide:
        h = rng.integers(-(1 << 20), (1 << 20) + 1, size=L * J).astype(np.int32)
        h[:L] = 1 << 20                                     # tap 0 of every phase: each phase's sum reaches 2^20
        S = 24
    else:
        lim = max(1, 65535 // J - 1)
        h = rng.integers(-lim, lim + 1, size=L * J).astype(np.int32)
        S = 15
    assert rm.wide(h, L, S) == wide
    return h, S


def _device(L, N, h, S, n0, x, offset_bytes=0, extra=16):
    """rxb200_resample_device over x (int16 [2c]) from a source offset_bytes into its buffer: (outputs, guard tail)."""
    torch = fh.torch()
    c = x.size // 2
    n = rm.out_count(n0, c, L, N)
    pad = offset_bytes // 2
    buf = torch.zeros(x.size + pad + 8, dtype=torch.int16, device="cuda")
    buf[pad:pad + x.size] = torch.from_numpy(x).cuda()
    dst = torch.full((2 * (n + extra),), GUARD, dtype=torch.int16, device="cuda")
    resample.resample_device(L, N, h, S, n0, buf.data_ptr() + offset_bytes, c, dst.data_ptr())
    torch.cuda.synchronize()
    d = dst.cpu().numpy()
    return d[:2 * n], d[2 * n:]


def _cases():
    out, k = [], 0
    for L, N in RATIOS:
        for J in JS:
            if J * L > (1 << 22):
                continue
            for wide in (False, True):
                out.append((L, N, J, wide, N0S[k % 3], (0, 4, 16)[(k // 3) % 3]))
                k += 1
    return out


@pytest.mark.parametrize("L,N,J,wide,n0,off", _cases())
def test_device_entry_equals_model_over_every_int16(L, N, J, wide, n0, off):
    rng = np.random.default_rng(L * 7 + N * 3 + J + wide)
    h, S = _taps(rng, L, J, wide)
    x = fh.every_int16(L + N + J)
    got, tail = _device(L, N, h, S, n0, x, off)
    want, _ = rm.resample_model(x, L, N, h, S, n0)
    assert np.array_equal(got, want)
    assert np.all(tail == GUARD)


@pytest.mark.parametrize("L,N,n0,c", [(1, 7, 1, 5), (1, 7, 0, 0), (2, 9, 1, 3), (1, 1000, 5, 990), (3, 4, 0, 1)])
def test_device_calls_too_short_to_emit(L, N, n0, c):
    h = np.arange(1, 4 * L + 1, dtype=np.int32)
    x = np.arange(2 * max(c, 1), dtype=np.int16)[:2 * c]
    got, tail = _device(L, N, h, 15, n0, x if c else np.zeros(2, np.int16)[:0])
    assert got.size == 2 * rm.out_count(n0, c, L, N)
    want, _ = rm.resample_model(x, L, N, h, 15, n0)
    assert np.array_equal(got, want)
    assert np.all(tail == GUARD)


def test_identity_anchor_on_device():
    x = fh.every_int16(3)
    got, tail = _device(1, 1, np.array([1 << 15], np.int32), 15, 12345, x)
    assert np.array_equal(got, x) and np.all(tail == GUARD)


@pytest.mark.parametrize("M,T,S", [(2, 65, 15), (7, 225, 15), (25, 9, 13), (4, 1, 0)])
def test_decimation_anchor_against_ddc_device(M, T, S):
    torch = fh.torch()
    rng = np.random.default_rng(M + T)
    h = rng.integers(-3000, 3001, size=T).astype(np.int32)
    x = fh.every_int16(M)
    got, _ = _device(1, M, h, S, 0, x)
    z = np.concatenate([np.zeros(2 * (M - 1), np.int16), x])
    src = torch.from_numpy(z).cuda()
    n = (z.size // 2) // M
    d = torch.zeros(2 * n + 2, dtype=torch.int16, device="cuda")
    fm.ddc_device(1_000_000, 0, 0, (M, h, S), src.data_ptr(), z.size // 2, d.data_ptr())
    torch.cuda.synchronize()
    assert n == got.size // 2
    assert np.array_equal(got, d.cpu().numpy()[:2 * n])


# (L, N, J): the 2.4 Msps NOAA plan (int32 accumulator, taps in shared memory) and the 30.72 Msps FM-band plan (int64
# accumulator, 25 432 taps read through the caches)
PLAN = (21, 25, 24)
WIDE_PLAN = (187, 256, 136)


def _plan_handle(plan=PLAN):
    L, N, J = plan
    h = resample.lowpass(L, N, J)
    return resample.Resampler(L, N, h, 15), h


def _stream(n, seed=7):
    return np.random.default_rng(seed).integers(-32768, 32768, size=2 * n).astype(np.int16)


def _host_calls(r, x, lens16):
    parts, at, i = [], 0, 0
    while at < x.size:
        n = min(lens16[i % len(lens16)], x.size - at)
        parts.append(r.process(x[at:at + n]))
        at += n
        i += 1
    return np.concatenate(parts)


def _device_calls(r, x, lens16):
    torch = fh.torch()
    src = torch.from_numpy(x).cuda()
    total = rm.out_count(0, x.size // 2, r.up, r.down)
    dst = torch.full((2 * total + 32,), GUARD, dtype=torch.int16, device="cuda")
    at, i, done = 0, 0, 0
    while at < x.size:
        n = min(lens16[i % len(lens16)], x.size - at)
        got = r.process_device(src.data_ptr() + 2 * at, n, dst.data_ptr() + 4 * done, total - done, sync=0)
        done += got
        at += n
        i += 1
    torch.cuda.synchronize()
    d = dst.cpu().numpy()
    assert done == total and np.all(d[2 * total:] == GUARD)
    return d[:2 * total]


@pytest.mark.parametrize("lens16", [[2], [6], [2 * 4093], [2 * 131072], [2 * 1000, 2 * 7777]],
                         ids=["1", "3", "4093", "131072", "1000:7777"])
@pytest.mark.parametrize("plan", [PLAN, WIDE_PLAN], ids=["21_25_J24", "187_256_J136"])
def test_handle_read_patterns_equal_one_call(lens16, plan):
    L, N, J = plan
    n = 20_000 if lens16[0] <= 6 else 400_000
    x = _stream(n)
    r, h = _plan_handle(plan)
    assert rm.wide(h, L, 15) == (plan == WIDE_PLAN) and (L * J > 12288) == (plan == WIDE_PLAN)
    want, _ = rm.resample_model(x, L, N, h, 15)
    assert np.array_equal(_host_calls(r, x, lens16), want)
    r.reset()
    assert np.array_equal(_device_calls(r, x, lens16), want)
    r.close()


def test_host_call_over_several_scratch_groups_equals_one_group():
    """(1, 7) groups hold about 14.7 M device samples: 40 M samples cross two group boundaries."""
    torch = fh.torch()
    h = np.array([3, -7, 11, 2000, 11, -7, 3, 1], np.int32)
    r = resample.Resampler(1, 7, h, 11)
    x = _stream(40_000_000, seed=11)
    got = r.process(x)
    src = torch.from_numpy(x).cuda()
    n = rm.out_count(0, x.size // 2, 1, 7)
    d = torch.zeros(2 * n, dtype=torch.int16, device="cuda")
    resample.resample_device(1, 7, h, 11, 0, src.data_ptr(), x.size // 2, d.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(got, d.cpu().numpy())
    r.close()


def test_reset_and_refused_calls_leave_the_state():
    L, N, J = PLAN
    x = _stream(50_000, seed=3)
    r, h = _plan_handle()
    want, _ = rm.resample_model(x, L, N, h, 15)
    a = r.process(x[:2 * 777])
    L_ = _lib.lib()
    small = np.zeros(2, np.int16)
    piece = x[2 * 777:2 * 5777]
    assert L_.rxb200_resample_process(r._h, piece.ctypes.data, piece.size, small.ctypes.data, 1, None) == _lib.ECAPACITY
    assert L_.rxb200_resample_process(r._h, piece.ctypes.data, 3, small.ctypes.data, 100, None) == _lib.EINVAL
    b = r.process(x[2 * 777:])
    assert np.array_equal(np.concatenate([a, b]), want)
    r.reset()
    assert np.array_equal(r.process(x), want)
    assert r.kernel_ms() > 0.0
    r.close()
