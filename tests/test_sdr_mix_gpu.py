"""rx_sdr I/Q down-converter handles (rxb200_sdr_mix_*) on the GPU: each kind against its stateless rule
(rxb200_power_ddc_device, rxb200_two_stage_device) over every int16 value in every format; every named shape against the
numpy model; seeded ragged call sequences (calls shorter than M, ending at every phase of M and M1, crossing a host
call's scratch groups, reset then a replay) against one call; every format against CS16 through rxb200_sdr_convert;
device entries at 4- and 16-byte offsets with guard words past every row; and refusals that leave the handle as it was."""
import numpy as np
import pytest

import fm_handles as fh
import sdr_mix as sm
from rx_tools_b200 import _lib, fm, power, sdr

pytestmark = pytest.mark.gpu

FMTS = (sdr.OUT_CS16, sdr.CVT_CS16_CS8, sdr.CVT_CS16_CU8, sdr.CVT_CS16_CF32)
NAMES = {sdr.OUT_CS16: "CS16", sdr.CVT_CS16_CS8: "CS8", sdr.CVT_CS16_CU8: "CU8", sdr.CVT_CS16_CF32: "CF32"}
SINGLE = (1_000_000, [0, 123_457, -499_999, 250_000], (5, np.array([3, -7, 11, 2000, 11, -7, 3], np.int32), 11))
TWO = (1_000_000, 10, [0, 123_457, -499_999, 250_000, 50_001],
       (5, np.array([9, 300, 3000, 300, 9], np.int32), 27), (3, np.array([1, 4000, 9000, 4000, 1], np.int32), 15))


def _single():
    R, offs, dd = SINGLE
    return sdr.SdrMix(R, offs, ddc=dd)


def _two():
    R, K, offs, c1, c2 = TWO
    return sdr.SdrMix(R, offs, two_stage=(K, c1, c2))


def _stateless(kind, x):
    """Per channel, the stateless entry's CS16 outputs over the whole capture x."""
    torch = fh.torch()
    src = torch.from_numpy(x).cuda()
    if kind == "single":
        R, offs, dd = SINGLE
        n = x.size // 2 // dd[0]
        out = []
        for f in offs:
            d = torch.zeros(2 * n + 2, dtype=torch.int16, device="cuda")
            power.power_ddc_device(R, f, 0, dd, src.data_ptr(), x.size // 2, d.data_ptr())
            torch.cuda.synchronize()
            out.append(d.cpu().numpy()[:2 * n])
        return np.stack(out)
    R, K, offs, c1, c2 = TWO
    n = x.size // 2 // (c1[0] * c2[0])
    d = torch.zeros(len(offs) * 2 * n + 2, dtype=torch.int16, device="cuda")
    fm.two_stage_device(R, K, offs, 0, c1, c2, src.data_ptr(), x.size // 2, d.data_ptr())
    torch.cuda.synchronize()
    return d.cpu().numpy()[:len(offs) * 2 * n].reshape(len(offs), 2 * n)


def _calls(h, x, lens16, fmt):
    """The concatenation of the host calls over x cut at lens16 (cycled), per channel."""
    parts, at, i = [], 0, 0
    while at < x.size:
        n = min(lens16[i % len(lens16)], x.size - at)
        parts.append(h.process(x[at:at + n], fmt))
        at += n
        i += 1
    return np.concatenate(parts, axis=1)


@pytest.mark.parametrize("kind", ["single", "two"])
def test_handle_equals_stateless_rule_every_int16_every_format(kind):
    x = fh.every_int16(41 if kind == "single" else 42)
    want16 = _stateless(kind, x)
    h = _single() if kind == "single" else _two()
    for fmt in FMTS:
        h.reset()
        got = h.process(x, fmt)
        assert np.array_equal(got.view(np.uint8), sm.convert(want16, NAMES[fmt]).view(np.uint8)), NAMES[fmt]
        if fmt != sdr.OUT_CS16:
            conv = fm.sdr_convert(fmt, want16.reshape(-1)).reshape(got.shape)
            assert np.array_equal(got.view(np.uint8), conv.view(np.uint8)), NAMES[fmt]
    h.close()


@pytest.mark.parametrize("name", list(sm.SHAPES))
def test_shapes_equal_model(name):
    x = sm.case_capture(name)
    want, M = sm.model(name, x)
    h = sm.handle(name)
    for fmt in (sdr.OUT_CS16, sdr.CVT_CS16_CF32):
        h.reset()
        got = _calls(h, x, [2 * 7 * M + 6, 2 * M * 3, 10, 2 * 1000 * M + 2], fmt)
        assert np.array_equal(got.view(np.uint8), sm.convert(want, NAMES[fmt]).view(np.uint8)), (name, NAMES[fmt])
    h.close()


@pytest.mark.parametrize("kind", ["single", "two"])
def test_ragged_calls_equal_one_call(kind):
    rng = np.random.default_rng(7 if kind == "single" else 8)
    x = rng.integers(-32768, 32768, size=2 * 40_000, dtype=np.int32).astype(np.int16)
    h = _single() if kind == "single" else _two()
    M = SINGLE[2][0] if kind == "single" else TWO[3][0] * TWO[4][0]
    M1 = M if kind == "single" else TWO[3][0]
    one = h.process(x, sdr.CVT_CS16_CU8)
    # calls shorter than M; calls of k M + 1 and k M1 + 1 samples, whose ends step through every phase of M and of M1 in
    # turn; long ones
    seqs = [[2], [2 * (M - 1)], [2 * (M + 1)], [2 * (3 * M + 1)], [2 * (M1 + 1)], [2 * (7 * M1 + 1)],
            [int(v) * 2 for v in rng.integers(1, 3000, size=40)]]
    for lens in seqs:
        h.reset()
        got = _calls(h, x, lens, sdr.CVT_CS16_CU8)
        assert np.array_equal(got, one), lens
    # reset, then a replay
    h.reset()
    assert np.array_equal(h.process(x, sdr.CVT_CS16_CU8), one)
    h.close()


@pytest.mark.parametrize("kind", ["single", "two"])
def test_host_call_across_scratch_groups(kind):
    """A host call longer than one group of RXB200_SDR_MIX_SCRATCH_BYTES equals short calls."""
    h = _single() if kind == "single" else _two()
    M = SINGLE[2][0] if kind == "single" else TWO[3][0] * TWO[4][0]
    n = (64 << 20) // (4 * M + 8 * h.n_channels) * M * 2 + 12_345        # complex samples: beyond two groups
    rng = np.random.default_rng(3)
    x = rng.integers(-32768, 32768, size=2 * n, dtype=np.int32).astype(np.int16)
    one = h.process(x, sdr.CVT_CS16_CF32)
    h.reset()
    got = _calls(h, x, [2 * 1_000_003], sdr.CVT_CS16_CF32)
    assert np.array_equal(got.view(np.uint8), one.view(np.uint8))
    h.close()


@pytest.mark.parametrize("kind", ["single", "two"])
@pytest.mark.parametrize("fmt", FMTS)
def test_device_entry_offsets_and_guards(kind, fmt):
    torch = fh.torch()
    rng = np.random.default_rng(fmt + 10)
    x = rng.integers(-32768, 32768, size=2 * 30_000, dtype=np.int32).astype(np.int16)
    h = _single() if kind == "single" else _two()
    want = h.process(x, fmt)
    E = sdr.ELEM_BYTES[fmt]
    lens = [2 * 4999, 2 * 17, 2 * 10_000, 2 * 14_984]
    for off in (4, 16):
        h.reset()
        src = torch.from_numpy(np.concatenate([np.zeros(off // 2, np.int16), x])).cuda()
        parts = []
        at = 0
        for n16 in lens:
            n = h.decimated_len(n16)
            stride = n + 3                                     # 3 guard elements after every row
            cap = (h.n_channels - 1) * stride + n
            buf = torch.full((off + cap * E + 64,), 0xA5, dtype=torch.uint8, device="cuda")
            got = h.process_device(src.data_ptr() + off + 2 * at, n16, fmt, buf.data_ptr() + off, cap, stride)
            assert got == n
            b = buf.cpu().numpy()
            assert (b[:off] == 0xA5).all() and (b[off + cap * E:] == 0xA5).all()
            rows = b[off:off + cap * E]
            for c in range(h.n_channels):
                if c < h.n_channels - 1:
                    assert (rows[(c * stride + n) * E:(c + 1) * stride * E] == 0xA5).all()
            parts.append(np.stack([rows[c * stride * E:(c * stride + n) * E] for c in range(h.n_channels)]))
            at += n16
        assert np.array_equal(np.concatenate(parts, axis=1), want.view(np.uint8).reshape(h.n_channels, -1))
    h.close()


@pytest.mark.parametrize("kind", ["single", "two"])
def test_refusals_leave_the_handle_unchanged(kind):
    torch = fh.torch()
    rng = np.random.default_rng(99)
    x = rng.integers(-32768, 32768, size=2 * 9_000, dtype=np.int32).astype(np.int16)
    h = _single() if kind == "single" else _two()
    want = h.process(x, sdr.OUT_CS16)
    h.reset()
    first = h.process(x[:2 * 4001], sdr.OUT_CS16)
    src = torch.from_numpy(x).cuda()
    n = h.decimated_len(2 * 3000)
    out = torch.zeros(4 * h.n_channels * (n + 8), dtype=torch.uint8, device="cuda")
    bad = [
        (src.data_ptr() + 2, 6000, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n, n, _lib.EINVAL),    # capture align
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr() + 2, h.n_channels * n, n, _lib.EINVAL),    # output align
        (src.data_ptr(), 6001, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n, n, _lib.EINVAL),        # odd n_int16
        (src.data_ptr(), 6000, 3, out.data_ptr(), h.n_channels * n, n, _lib.EINVAL),                   # bad format
        (src.data_ptr(), 6000, 7, out.data_ptr(), h.n_channels * n, n, _lib.EINVAL),
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n, n - 1, _lib.ECAPACITY),  # stride
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n - 1, n, _lib.ECAPACITY),  # capacity
        (0, 6000, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n, n, _lib.EINVAL),
    ]
    for s, n16, fmt, o, cap, stride, code in bad:
        with pytest.raises(_lib.Rxb200Error) as e:
            h.process_device(s, n16, fmt, o, cap, stride)
        assert e.value.code == code
    with pytest.raises(_lib.Rxb200Error):
        h.process(x[:5], sdr.OUT_CS16)
    rest = h.process(x[2 * 4001:], sdr.OUT_CS16)
    assert np.array_equal(np.concatenate([first, rest], axis=1), want)
    h.close()
