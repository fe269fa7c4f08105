"""Capture handles in a device's own format, without a GPU: the widening rule (tests/device_format.py) over every byte
value and against the reference port's CS12 unpack; the setters' refusals; RXB200_DEVICE_FORMAT's refusals in each
shell before the device opens; rx_sdr's capture-mode -I refusal as it was without the variable; and the replay device
opening CS8 and CU8 files."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import device_format as df
from rx_tools_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
HOST = os.path.join(os.path.dirname(HERE), "host")


# ---- the rule
def test_cs8_and_cu8_over_every_byte():
    b = np.arange(256, dtype=np.uint8)
    s8 = df.widen(b, "CS8")
    assert s8.dtype == np.int16 and s8.size == 256
    assert np.array_equal(s8, b.view(np.int8).astype(np.int16) * 256)
    u8 = df.widen(b, "CU8")
    assert np.array_equal(u8, (b.astype(np.int16) - 128) * 256)
    # CU8 b is CS8 b ^ 0x80: the kernel's flip of each byte's top bit
    assert np.array_equal(u8, df.widen(b ^ 0x80, "CS8"))
    assert s8.min() == -32768 and s8.max() == 127 * 256


def test_cs12_equals_the_reference_unpack():
    import oracle
    f = oracle.port().L.orx_sdr_cs12_to_cs16
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    f.restype = None
    rng = np.random.default_rng(12)
    for n in (1, 2, 3, 1000, 65_537):
        y = rng.integers(0, 256, 3 * n, dtype=np.uint8)
        out = np.empty(2 * n, np.int16)
        f(y.ctypes.data, n, out.ctypes.data)
        assert np.array_equal(out, df.widen(y, "CS12")), n


def test_in_array_counts_two_int16_per_element():
    for fmt, e in (("CS8", 2), ("CU8", 2), ("CS12", 3)):
        a, n16 = _lib.in_array(np.zeros(5 * e, np.uint8), df.FORMATS[fmt])
        assert a.dtype == np.uint8 and n16 == 10
        with pytest.raises(ValueError):
            _lib.in_array(np.zeros(5 * e + 1, np.uint8), df.FORMATS[fmt])
    a, n16 = _lib.in_array(np.zeros(10, np.int16), _lib.IN_CS16)
    assert a.dtype == np.int16 and n16 == 10


def test_setters_refuse_a_null_handle():
    """A NULL handle is refused before anything touches a device (an unknown format needs a handle, which needs a GPU:
    that case is in tests/test_device_format_gpu.py)."""
    L = _lib.lib()
    for name in ("rxb200_fm_mix_set_input_format", "rxb200_sdr_mix_set_input_format",
                 "rxb200_power_mix_set_input_format"):
        for fmt in (_lib.IN_CS16, _lib.IN_CU8, 99, -1):
            assert getattr(L, name)(None, fmt) == _lib.EINVAL, (name, fmt)
    assert (_lib.IN_CS16, _lib.IN_CS8, _lib.IN_CU8, _lib.IN_CS12) == (0, 1, 2, 3)


# ---- the shells
@pytest.fixture(scope="module")
def shells():
    subprocess.run(["make", "-C", HOST, "-s"], check=True)


def _shell(tmp_path, exe, args, env):
    e = {k: v for k, v in os.environ.items() if not k.startswith("RXB200_")}
    e.update(env)
    missing = tmp_path / "no_such_capture.cs16"        # opening the device fails: a refusal must come first
    return subprocess.run([os.path.join(HOST, exe)] + args[:-1] + ["-d", f"driver=file,path={missing}", args[-1]],
                          capture_output=True, env=e, timeout=60)


SHELL_CASES = {
    "rx_fm": ("rx_fm_b200", ["-M", "fm", "-s", "24k", "-l", "50", "-f", "162.4M", "-f", "162.55M"]),
    "rx_sdr": ("rx_sdr_b200", ["-s", "250k", "-F", "CS16", "-f", "100M", "-f", "100.95M"]),
    "rx_power": ("rx_power_b200", ["-f", "88M:108M:10k", "-1"]),
}


def _refused(r, tmp_path, needle):
    err = r.stderr.decode()
    assert r.returncode == 1 and needle in err, err
    assert "Failed to open" not in err and not list(tmp_path.glob("out*")), err


@pytest.mark.parametrize("shell", sorted(SHELL_CASES))
def test_shell_refusals_before_the_device(tmp_path, shells, shell):
    exe, args = SHELL_CASES[shell]
    out = str(tmp_path / "out")
    # without a capture (or tile) variable
    _refused(_shell(tmp_path, exe, args + [out], {"RXB200_DEVICE_FORMAT": "CU8"}), tmp_path, "RXB200_DEVICE_FORMAT needs")
    # an unknown format, in capture mode and (rx_power) tile mode
    modes = [{"RXB200_CAPTURE_RATE": "100000000"}] + ([{"RXB200_TILE_RATE": "10000000"}] if shell == "rx_power" else [])
    for mode in modes:
        for bad in ("CF32", "cu8", "U8", ""):
            r = _shell(tmp_path, exe, args + [out], dict(mode, RXB200_DEVICE_FORMAT=bad))
            _refused(r, tmp_path, f"RXB200_DEVICE_FORMAT={bad} is not one of")


def test_rx_sdr_input_format_against_the_variable(tmp_path, shells):
    exe, args = SHELL_CASES["rx_sdr"]
    out = str(tmp_path / "out")
    cap = {"RXB200_CAPTURE_RATE": "100000000"}
    # -I that names another format than the variable: both named
    for var, i in (("CU8", "CS8"), ("CS8", "CS16"), ("CS12", "CU8"), ("CS16", "CS8")):
        r = _shell(tmp_path, exe, ["-I", i] + args + [out], dict(cap, RXB200_DEVICE_FORMAT=var))
        _refused(r, tmp_path, f"RXB200_DEVICE_FORMAT={var}, not -I {i}")
    # -I equal to the variable, or left out, passes the check: the run gets as far as opening the (missing) device
    for var, extra in (("CU8", ["-I", "CU8"]), ("CS12", []), ("CS16", ["-I", "CS16"])):
        r = _shell(tmp_path, exe, extra + args + [out], dict(cap, RXB200_DEVICE_FORMAT=var))
        err = r.stderr.decode()
        assert r.returncode == 1 and "Failed to open" in err and "-I" not in err, err
        assert not list(tmp_path.glob("out*"))


def test_rx_sdr_refusal_without_the_variable_unchanged(tmp_path, shells):
    """Without RXB200_DEVICE_FORMAT, capture mode still reads CS16 only, with the same message."""
    r = _shell(tmp_path, "rx_sdr_b200", ["-f", "100M", "-I", "CS8", "-F", "CS8", str(tmp_path / "out")],
               {"RXB200_CAPTURE_RATE": "100000000"})
    assert r.returncode == 1 and r.stderr.decode().endswith(
        "Capture mode (RXB200_CAPTURE_RATE) reads CS16, not CS8.\n"), r.stderr.decode()
    assert not list(tmp_path.glob("out*"))


@pytest.mark.parametrize("fmt", ["CS8", "CU8"])
def test_replay_device_opens_8_bit_files(tmp_path, shells, fmt):
    """The replay device takes CS8 and CU8 as 2-byte elements, raw: plain rx_sdr written as read gives the file back."""
    b = df.narrow_stream(10_000, fmt, 4)
    cap = tmp_path / f"cap.{fmt.lower()}"
    b.tofile(cap)
    out = tmp_path / "out.bin"
    e = {k: v for k, v in os.environ.items() if not k.startswith("RXB200_")}
    r = subprocess.run([os.path.join(HOST, "rx_sdr_b200"), "-d", f"driver=file,path={cap},reads=999:1", "-I", fmt,
                        "-F", fmt, str(out)], capture_output=True, env=e, timeout=60)
    assert r.returncode == 0, r.stderr.decode()
    assert out.read_bytes() == b.tobytes()
