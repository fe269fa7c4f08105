"""rxb200_sdr_convert_device's refusals, which come before any CUDA call: a CS12 destination that is not 4-byte aligned
(the unpack stores one 32-bit word per element), CS16 pointers off 16 bytes, an unknown kind and null pointers.

The pointers are plain integers.  With n_elems = 0 a refusal that went missing returns RXB200_OK without launching
anything, so that form runs everywhere; with n_elems > 0 it would launch on those integers, so that form runs only where
there is no device to launch on."""
import ctypes as C

import pytest

from rx_tools_b200 import _lib, fm

BASE = 1 << 20          # an integer address, 256-byte aligned; never dereferenced


def _sizes():
    return (0,) if _lib.lib().rxb200_device_count() > 0 else (0, 8)


def _convert(kind, src, n, dst):
    return _lib.lib().rxb200_sdr_convert_device(kind, C.c_void_p(src) if src else None, n,
                                                C.c_void_p(dst) if dst else None, None)


@pytest.mark.parametrize("dst_off", [1, 2, 3, 6])
def test_cs12_destination_off_four_bytes(dst_off):
    for n in _sizes():
        assert _convert(fm.CVT_CS12_CS16, BASE, n, BASE + 4096 + dst_off) == _lib.EINVAL, (dst_off, n)


@pytest.mark.parametrize("kind", [fm.CVT_CS16_CS8, fm.CVT_CS16_CU8, fm.CVT_CS16_CF32])
@pytest.mark.parametrize("src_off,dst_off", [(4, 0), (0, 4), (8, 8), (2, 0), (0, 12)])
def test_cs16_pointers_off_sixteen_bytes(kind, src_off, dst_off):
    for n in _sizes():
        assert _convert(kind, BASE + src_off, n, BASE + 4096 + dst_off) == _lib.EINVAL, (kind, src_off, dst_off, n)


@pytest.mark.parametrize("kind", [-1, 4])
def test_unknown_kind(kind):
    for n in _sizes():
        assert _convert(kind, BASE, n, BASE + 4096) == _lib.EINVAL, (kind, n)


@pytest.mark.parametrize("kind", [fm.CVT_CS16_CS8, fm.CVT_CS16_CU8, fm.CVT_CS16_CF32, fm.CVT_CS12_CS16])
def test_null_pointers(kind):
    for n in _sizes():
        assert _convert(kind, None, n, BASE) == _lib.EINVAL, (kind, n)
        assert _convert(kind, BASE, n, None) == _lib.EINVAL, (kind, n)


def test_cs12_source_may_take_any_byte_offset():
    """The refusal is the destination's alone: a CS12 source at any byte offset and a 4-byte aligned destination pass
    the checks (n_elems = 0: nothing to convert, nothing launched)."""
    for src_off in range(4):
        assert _convert(fm.CVT_CS12_CS16, BASE + src_off, 0, BASE + 4096 + 4) == _lib.OK, src_off
