"""The rx_fm group entry points without a GPU: bad arguments are refused before any device is touched, and creating a
group fails like creating a handle (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from rx_tools_b200 import _lib, fm


def test_bad_arguments_and_null_group():
    L = _lib.lib()
    pc = fm.FmParams().to_c()
    g = C.c_void_p()
    for n_ch, n_dev in ((0, 1), (4, 0), (-1, 2)):
        assert L.rxb200_fm_group_create(C.byref(pc), n_ch, n_dev, None, C.byref(g)) == _lib.EINVAL
    assert L.rxb200_fm_group_create(None, 4, 2, None, C.byref(g)) == _lib.EINVAL
    assert L.rxb200_fm_group_create(C.byref(pc), 4, 2, None, None) == _lib.EINVAL
    buf = np.zeros(64, dtype=np.int16)
    n = C.c_size_t(0)
    assert L.rxb200_fm_group_process(None, buf.ctypes.data, 32, 32, buf.ctypes.data, 64, C.byref(n), None) == _lib.EINVAL
    assert L.rxb200_fm_group_process_read(None, buf.ctypes.data, 32, buf.ctypes.data, 64, C.byref(n)) == _lib.EINVAL
    hits = np.zeros(4, dtype=np.int32)
    assert L.rxb200_fm_group_squelch_hits(None, hits.ctypes.data_as(C.POINTER(C.c_int))) == _lib.EINVAL
    assert L.rxb200_fm_group_levels(None, hits.ctypes.data_as(C.POINTER(C.c_int)), 4, C.byref(n)) == _lib.EINVAL
    assert L.rxb200_fm_group_reset(None) == _lib.EINVAL
    assert L.rxb200_fm_group_size(None) == 0
    assert L.rxb200_fm_group_member(None, 0) is None
    L.rxb200_fm_group_destroy(None)


def test_no_cpu_fallback_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmGroup(fm.FmParams(), 5, [0, 0])
    assert e.value.code == _lib.ENODEV

