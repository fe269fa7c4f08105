"""The capture handles' input formats (include/rxb200.h, "capture handles in a device's own format"; DESIGN.md section
4.8): the widening rule in numpy, narrow streams, and replay files in each format beside their CS16 widening."""
import os

import numpy as np

from rx_tools_b200 import _lib

FORMATS = {"CS8": _lib.IN_CS8, "CU8": _lib.IN_CU8, "CS12": _lib.IN_CS12}
ELEM = {"CS16": 4, "CS8": 2, "CU8": 2, "CS12": 3}


def widen(b, fmt: str) -> np.ndarray:
    """The rule: bytes b of format fmt (whole elements) to interleaved CS16, int16[2 n]."""
    b = np.ascontiguousarray(b, dtype=np.uint8).reshape(-1)
    if fmt == "CS8":
        return (b.astype(np.int32) << 8).astype(np.uint16).view(np.int16)
    if fmt == "CU8":
        return ((b.astype(np.int32) - 128) << 8).astype(np.int16)
    assert fmt == "CS12" and b.size % 3 == 0
    b0, b1, b2 = (b[k::3].astype(np.uint32) for k in range(3))
    out = np.empty(2 * b0.size, np.uint16)
    out[0::2] = ((b1 << 12) | (b0 << 4)) & 0xffff
    out[1::2] = ((b2 << 8) | (b1 & 0xf0)) & 0xffff
    return out.view(np.int16)


def narrow_stream(n_complex: int, fmt: str, seed: int) -> np.ndarray:
    """n_complex elements of fmt as bytes: a strong tone and noise, with full-scale bytes early (every byte value
    appears in a long stream)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_complex)
    if fmt == "CS12":
        # 12-bit I and Q packed as the rule unpacks them: I = b1 << 12 | b0 << 4 takes I's 12 bits as b1[3:0] b0
        i = (1500 * np.cos(0.0137 * t) + rng.normal(0, 300, n_complex)).round().clip(-2048, 2047).astype(np.int64) & 0xfff
        q = (1500 * np.sin(0.0137 * t) + rng.normal(0, 300, n_complex)).round().clip(-2048, 2047).astype(np.int64) & 0xfff
        b = np.empty(3 * n_complex, np.uint8)
        b[0::3] = i & 0xff
        b[1::3] = (i >> 8) | ((q & 0xf) << 4)
        b[2::3] = q >> 4
        b[:48] = rng.integers(0, 256, 48)
        return b
    i = 60 * np.cos(0.0137 * t) + rng.normal(0, 20, n_complex)
    q = 60 * np.sin(0.0137 * t) + rng.normal(0, 20, n_complex)
    s = np.empty(2 * n_complex)
    s[0::2], s[1::2] = i, q
    s = s.round().clip(-128, 127).astype(np.int64)
    b = (s & 0xff).astype(np.uint8) if fmt == "CS8" else (s + 128).astype(np.uint8)
    b[:64] = rng.integers(0, 256, 64)
    return b


def write_replay(directory: str, fmt: str, b) -> tuple:
    """The replay files of one stream: bytes b as <fmt>.bin and their widening as widened.cs16; (narrow, cs16) paths."""
    narrow = os.path.join(directory, f"cap.{fmt.lower()}")
    cs16 = os.path.join(directory, "widened.cs16")
    np.ascontiguousarray(b, dtype=np.uint8).tofile(narrow)
    widen(b, fmt).tofile(cs16)
    return narrow, cs16
