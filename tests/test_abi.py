"""The C-ABI library loads and exports every symbol include/rxb200.h declares; without a GPU every
create call fails loudly (no CPU fallback).  No compute calls here."""
import ctypes as C
import os
import re

import pytest

from rx_tools_b200 import _lib, fm, power

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "rxb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rxb200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    syms = header_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(L, s), f"librxb200.so does not export {s}"
    assert sorted(_lib.SYMBOLS) == syms
    assert L.rxb200_abi_version() == 3


def test_no_cpu_fallback_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmDemod(fm.FmParams())
    assert e.value.code == _lib.ENODEV
    with pytest.raises(_lib.Rxb200Error) as e:
        power.PowerScanner(power.plan_range("100M:101M:1k"), "hamming")
    assert e.value.code == _lib.ENODEV


def test_disc_device_refuses_before_any_device_work():
    """rxb200_fm_disc_device checks its form and pointers before it touches a device (also where there is none)."""
    L = _lib.lib()
    for form in (-1, 9):
        assert L.rxb200_fm_disc_device(form, None, 1, None, None) == _lib.EINVAL
    assert L.rxb200_fm_disc_device(0, None, 1, None, None) == _lib.EINVAL
    assert L.rxb200_fm_disc_device(0, 16, 1, None, None) == _lib.EINVAL
    assert L.rxb200_fm_disc_device(0, 4, 1, 16, None) == _lib.EINVAL         # quads not 16-byte aligned
    assert _lib.lib().rxb200_last_error()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "rx_tools_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".c")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in text and "from oracle" not in text, f
                assert "rx_oracle" not in text and "libref_" not in text, f
