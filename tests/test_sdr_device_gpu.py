"""rxb200_sdr_convert_device on torch buffers against the port's orx_sdr_*: every kind, on a non-default stream, from
pointers inside larger buffers (CS12 sources at every byte offset), at lengths that make several grid-stride trips and a
tail, with nothing written past the last output."""
import ctypes as C

import numpy as np
import pytest

import fm_handles as fh
import mix_scale as ms
import oracle
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu

PORT = {fm.CVT_CS16_CS8: "orx_sdr_cs16_to_cs8", fm.CVT_CS16_CU8: "orx_sdr_cs16_to_cu8",
        fm.CVT_CS16_CF32: "orx_sdr_cs16_to_cf32", fm.CVT_CS12_CS16: "orx_sdr_cs12_to_cs16"}
OUT_BYTES = {fm.CVT_CS16_CS8: 2, fm.CVT_CS16_CU8: 2, fm.CVT_CS16_CF32: 8, fm.CVT_CS12_CS16: 4}   # per element
GUARD = 64              # bytes checked past the last output
PAD = 0xa5


def _lengths():
    # the CS16 kinds move 4 elements per thread and trip over n_sm * 8 CTAs of 256 threads: k trips and a tail of 3
    sms = ms.device_sms()
    return [1, 3, 4, 5] + [k * sms * 8 * 1024 + 3 for k in (2, 3)]


def _port(kind, src, n):
    f = getattr(oracle.port().L, PORT[kind])
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    f.restype = None
    out = np.empty(n * OUT_BYTES[kind], np.uint8)
    f(src.ctypes.data, n if kind == fm.CVT_CS12_CS16 else 2 * n, out.ctypes.data)     # the CS16 ones count int16
    return out


def _input(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == fm.CVT_CS12_CS16:
        return rng.integers(0, 256, size=3 * n, dtype=np.int32).astype(np.uint8)
    # every int16 value first, then random ones
    v = np.arange(-32768, 32768, dtype=np.int32)
    x = np.concatenate([v, rng.integers(-32768, 32768, size=max(0, 2 * n - v.size), dtype=np.int32)])[:2 * n]
    return x.astype(np.int16).view(np.uint8)


@pytest.mark.parametrize("kind", [fm.CVT_CS16_CS8, fm.CVT_CS16_CU8, fm.CVT_CS16_CF32, fm.CVT_CS12_CS16])
def test_device_entry_equals_the_port(kind):
    torch = fh.torch()
    s = torch.cuda.Stream()
    src_offs = range(4) if kind == fm.CVT_CS12_CS16 else (0,)
    for n in _lengths():
        x = _input(kind, n, n + kind)
        want = _port(kind, x, n)
        host = torch.from_numpy(x).pin_memory()
        for so in src_offs:
            # each pointer 256 bytes into its buffer (plus so for a CS12 source)
            src = torch.zeros(256 + so + x.size, dtype=torch.uint8, device="cuda")
            dst = torch.full((256 + want.size + GUARD,), PAD, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                # the source arrives on s behind a wait: a conversion that ignored s would read zeros
                torch.cuda._sleep(20_000_000)
                src[256 + so:].copy_(host, non_blocking=True)
                _lib.check(_lib.lib().rxb200_sdr_convert_device(kind, src.data_ptr() + 256 + so, n,
                                                                dst.data_ptr() + 256, s.cuda_stream))
            s.synchronize()
            got = dst.cpu().numpy()
            bad = np.flatnonzero(got[256:256 + want.size] != want)
            assert bad.size == 0, (kind, n, so, bad[:4])             # CF32 compared as bytes: bit for bit
            assert (got[:256] == PAD).all() and (got[256 + want.size:] == PAD).all(), (kind, n, so)
