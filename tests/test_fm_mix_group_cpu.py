"""The mixing group entry points without a GPU: bad arguments and bad offsets are refused before any device is touched,
with the codes a single mixing handle returns, and creating a group fails like creating a handle (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

import fm_mix as fmx
from rx_tools_b200 import _lib, fm

P = fmx.SHAPES["fm5a_lut_d100"][0]


def _create(offs, rate=2_400_000, n_dev=2, n_channels=None, params=True, out=True):
    L = _lib.lib()
    pc = fm.FmParams.from_any(P).to_c()
    o = np.ascontiguousarray([] if offs is None else offs, dtype=np.int32)
    g = C.c_void_p()
    return L.rxb200_fm_mix_group_create(C.byref(pc) if params else None, rate,
                                        o.ctypes.data_as(C.POINTER(C.c_int)) if offs is not None else None,
                                        len(o) if n_channels is None else n_channels, n_dev, None,
                                        C.byref(g) if out else None)


def test_bad_arguments():
    assert _create([0, 12500], n_channels=0) == _lib.EINVAL
    assert _create([0, 12500], n_channels=-1) == _lib.EINVAL
    assert _create([0, 12500], n_dev=0) == _lib.EINVAL
    assert _create([0, 12500], params=False) == _lib.EINVAL
    assert _create(None, n_channels=2) == _lib.EINVAL
    assert _create([0, 12500], out=False) == _lib.EINVAL


@pytest.mark.parametrize("n_dev", [1, 2, 3])
def test_a_bad_offset_on_the_last_channel(n_dev):
    """Every channel's table is checked before any member is created, so the last member's bad offset gives the code
    rxb200_fm_mix_create gives, with or without a device."""
    ok = [-25000, 0, 12500, 37500]
    for f in (1_200_000, -1_200_000, 2_000_000):               # |f| >= R/2
        assert _create(ok + [f], n_dev=n_dev) == _lib.EINVAL, f
    assert _create(ok + [12500], rate=0, n_dev=n_dev) == _lib.EINVAL
    # at 2 400 001 Hz the period of 12 500 Hz is the whole rate, above 2^20
    assert _create([0, 0, 0, 12500], rate=2_400_001, n_dev=n_dev) == _lib.EUNSUPPORTED
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMixGroup(P, 2_400_000, ok + [1_200_000], n_dev=n_dev)
    assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(P, 2_400_000, ok + [1_200_000])
    assert e.value.code == _lib.EINVAL


def test_null_group():
    L = _lib.lib()
    buf = np.zeros(64, dtype=np.int16)
    n = C.c_size_t(0)
    assert L.rxb200_fm_mix_group_process(None, buf.ctypes.data, 32, 32, buf.ctypes.data, 64, C.byref(n),
                                         None) == _lib.EINVAL
    assert L.rxb200_fm_mix_group_process_read(None, buf.ctypes.data, 32, buf.ctypes.data, 64, C.byref(n)) == _lib.EINVAL
    hits = np.zeros(4, dtype=np.int32)
    assert L.rxb200_fm_mix_group_squelch_hits(None, hits.ctypes.data_as(C.POINTER(C.c_int))) == _lib.EINVAL
    assert L.rxb200_fm_mix_group_levels(None, hits.ctypes.data_as(C.POINTER(C.c_int)), 4, C.byref(n)) == _lib.EINVAL
    assert L.rxb200_fm_mix_group_reset(None) == _lib.EINVAL
    assert L.rxb200_fm_mix_group_size(None) == 0
    assert L.rxb200_fm_mix_group_member(None, 0) is None
    L.rxb200_fm_mix_group_destroy(None)


def test_no_cpu_fallback_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMixGroup(P, 2_400_000, [-25000, 0, 12500], [0, 0])
    assert e.value.code == _lib.ENODEV
