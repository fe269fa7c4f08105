"""rx_sdr raster I/Q handles (rxb200_sdr_mix_create_raster) on the GPU: the handle against rxb200_raster_device and
rx_sdr's conversion over every int16 value in every format for K = 3, 405, 768 and 4096; the anchor to the single-stage
handle (bin 0 at shift S + 15 is that handle at offset 0 with shift S) in every format; every named shape against the
model and the golden hashes; ragged call sequences ending at every phase of M and several residues of K against one
call; a host call spanning several scratch groups and raster frame groups against short calls; device entries at 4- and
16-byte offsets with guard bytes past every row; refusals that change neither the outputs nor the next call's bytes; and
reset."""
import json
import os

import numpy as np
import pytest

import fm_handles as fh
import sdr_raster as sr
from rx_tools_b200 import _lib, fm, power, sdr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "sdr_raster_golden.json")))
FMTS = (sdr.OUT_CS16, sdr.CVT_CS16_CS8, sdr.CVT_CS16_CU8, sdr.CVT_CS16_CF32)
NAMES = {sdr.OUT_CS16: "CS16", sdr.CVT_CS16_CS8: "CS8", sdr.CVT_CS16_CU8: "CU8", sdr.CVT_CS16_CF32: "CF32"}
# K -> (bins, (M, taps, S)): K = 405 is the FM broadcast plan, K = 768 tools/fm_raster_time.py's
RASTERS = {
    3: ([0, 1, 2, 1], (3, np.array([5, -40, 900, 4000, 900, -40, 5], np.int32), 20)),
    405: sr.SHAPES["broadcast_k405_c100"][1:3],
    768: ([0, 1, 383, 384, 385, 767, 100, 100], (64, power.ddc_lowpass(64, 2049, 15), 30)),
    4096: ([0, 1, 2048, 4095, 7], (16, power.ddc_lowpass(16, 257, 15), 30)),
}
SMALL = (48, [0, 24, 5, 47, 5], (6, power.ddc_lowpass(6, 97, 15), 30))


def _handle(K, bins, dd):
    return sdr.SdrMix(ddc=dd, raster=(K, bins))


def _stateless(K, bins, dd, x):
    """rxb200_raster_device's CS16 outputs over the whole capture x, per channel."""
    torch = fh.torch()
    src = torch.from_numpy(x).cuda()
    n = x.size // 2 // dd[0]
    d = torch.zeros(len(bins) * 2 * n + 2, dtype=torch.int16, device="cuda")
    fm.raster_device(K, bins, 0, dd, src.data_ptr(), x.size // 2, d.data_ptr())
    torch.cuda.synchronize()
    return d.cpu().numpy()[:len(bins) * 2 * n].reshape(len(bins), 2 * n)


def _calls(h, x, lens16, fmt):
    """The concatenation of the host calls over x cut at lens16 (cycled), per channel."""
    parts, at, i = [], 0, 0
    while at < x.size:
        n = min(lens16[i % len(lens16)], x.size - at)
        parts.append(h.process(x[at:at + n], fmt))
        at += n
        i += 1
    return np.concatenate(parts, axis=1)


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


@pytest.mark.parametrize("K", list(RASTERS))
def test_handle_equals_raster_device_every_int16_every_format(K):
    bins, dd = RASTERS[K]
    x = fh.every_int16(K)
    want16 = _stateless(K, bins, dd, x)
    h = _handle(K, bins, dd)
    for fmt in FMTS:
        h.reset()
        got = h.process(x, fmt)
        assert _same(got, sr.convert(want16, NAMES[fmt])), NAMES[fmt]
        if fmt != sdr.OUT_CS16:
            assert _same(got, fm.sdr_convert(fmt, want16.reshape(-1)).reshape(got.shape)), NAMES[fmt]
    h.close()


@pytest.mark.parametrize("fmt", FMTS)
def test_bin0_anchor_is_the_single_stage_handle(fmt):
    """Bin 0 at shift S + 15 is byte for byte the single-stage handle at offset 0 with shift S."""
    M, T = 8, 257
    taps = power.ddc_lowpass(M, T, 15)
    x = np.concatenate([fh.every_int16(5), np.full(2 * 4000, -32768, np.int16), fh.every_int16(6)])
    ras = sdr.SdrMix(ddc=(M, taps, 30), raster=(40, [0, 0, 3]))
    one = sdr.SdrMix(2_000_000, [0], ddc=(M, taps, 15))
    lens = [2 * 7 * M + 6, 2 * 5000, 2 * 3]
    a = _calls(ras, x, lens, fmt)
    b = _calls(one, x, lens, fmt)
    assert _same(a[0], b[0]) and _same(a[1], b[0])
    ras.close()
    one.close()


@pytest.mark.parametrize("name", list(sr.SHAPES))
def test_shapes_equal_model_and_golden(name):
    x = sr.case_capture(name)
    want, M = sr.model(name, x)
    h = sr.handle(name)
    for fmt in FMTS:
        h.reset()
        got = _calls(h, x, [2 * 7 * M + 6, 2 * M * 3, 10, 2 * 1000 * M + 2], fmt)
        assert _same(got, sr.convert(want, NAMES[fmt])), (name, NAMES[fmt])
        assert sr.digest(got) == GOLDEN[name][NAMES[fmt]], (name, NAMES[fmt])
    h.close()


@pytest.mark.parametrize("K", [48, 405])
def test_ragged_calls_equal_one_call(K):
    bins, dd = (SMALL[1], SMALL[2]) if K == 48 else RASTERS[405]
    M = dd[0]
    rng = np.random.default_rng(K)
    x = rng.integers(-32768, 32768, size=2 * 60_000, dtype=np.int32).astype(np.int16)
    h = _handle(K, bins, dd)
    one = h.process(x, sdr.CVT_CS16_CU8)
    # calls shorter than M; calls of k M + 1 samples, whose ends step through every phase of M; calls of K + 1 and
    # 2 K + 3 samples, whose ends step through residues of K; long ones
    seqs = [[2], [2 * (M - 1)], [2 * (M + 1)], [2 * (3 * M + 1)], [2 * (K + 1)], [2 * (2 * K + 3)],
            [int(v) * 2 for v in rng.integers(1, 3000, size=40)]]
    for lens in seqs:
        h.reset()
        assert np.array_equal(_calls(h, x, lens, sdr.CVT_CS16_CU8), one), lens
    h.close()


def test_host_call_across_scratch_and_frame_groups():
    """One host call over more than two RXB200_SDR_MIX_SCRATCH_BYTES groups, each over several raster frame groups
    (K = 4096: 1024 frames per group), equals short calls."""
    K, bins, dd = 4096, [0, 1, 2048, 4095], (4, power.ddc_lowpass(4, 33, 15), 30)
    h = _handle(K, bins, dd)
    M = dd[0]
    n = (64 << 20) // (4 * M + 8 * h.n_channels) * M * 2 + 12_345         # complex samples: beyond two groups
    x = np.random.default_rng(3).integers(-32768, 32768, size=2 * n, dtype=np.int32).astype(np.int16)
    one = h.process(x, sdr.CVT_CS16_CF32)
    h.reset()
    got = _calls(h, x, [2 * 1_000_003], sdr.CVT_CS16_CF32)
    assert _same(got, one)
    h.close()


@pytest.mark.parametrize("fmt", FMTS)
def test_device_entry_offsets_and_guards(fmt):
    torch = fh.torch()
    K, bins, dd = SMALL
    x = np.random.default_rng(fmt + 10).integers(-32768, 32768, size=2 * 30_000, dtype=np.int32).astype(np.int16)
    h = _handle(K, bins, dd)
    want = h.process(x, fmt)
    E = sdr.ELEM_BYTES[fmt]
    lens = [2 * 4999, 2 * 17, 2 * 10_000, 2 * 14_984]
    for off in (4, 16):
        h.reset()
        src = torch.from_numpy(np.concatenate([np.zeros(off // 2, np.int16), x])).cuda()
        parts, at = [], 0
        for n16 in lens:
            n = h.decimated_len(n16)
            stride = n + 3                                     # 3 guard elements after every row
            cap = (h.n_channels - 1) * stride + n
            buf = torch.full((off + cap * E + 64,), 0xA5, dtype=torch.uint8, device="cuda")
            assert h.process_device(src.data_ptr() + off + 2 * at, n16, fmt, buf.data_ptr() + off, cap, stride) == n
            b = buf.cpu().numpy()
            assert (b[:off] == 0xA5).all() and (b[off + cap * E:] == 0xA5).all()
            rows = b[off:off + cap * E]
            for c in range(h.n_channels - 1):
                assert (rows[(c * stride + n) * E:(c + 1) * stride * E] == 0xA5).all()
            parts.append(np.stack([rows[c * stride * E:(c * stride + n) * E] for c in range(h.n_channels)]))
            at += n16
        assert np.array_equal(np.concatenate(parts, axis=1), want.view(np.uint8).reshape(h.n_channels, -1))
    h.close()


def test_refusals_leave_the_handle_unchanged():
    torch = fh.torch()
    K, bins, dd = SMALL
    x = np.random.default_rng(99).integers(-32768, 32768, size=2 * 9_000, dtype=np.int32).astype(np.int16)
    h = _handle(K, bins, dd)
    want = h.process(x, sdr.OUT_CS16)
    h.reset()
    first = h.process(x[:2 * 4001], sdr.OUT_CS16)
    src = torch.from_numpy(x).cuda()
    n = h.decimated_len(2 * 3000)
    C = h.n_channels
    out = torch.zeros(8 * C * (n + 8), dtype=torch.uint8, device="cuda")
    bad = [
        (src.data_ptr() + 2, 6000, sdr.OUT_CS16, out.data_ptr(), C * n, n, _lib.EINVAL),        # capture alignment
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr() + 2, C * n, n, _lib.EINVAL),        # output alignment
        (src.data_ptr(), 6000, sdr.CVT_CS16_CS8, out.data_ptr() + 1, C * n, n, _lib.EINVAL),
        (src.data_ptr(), 6001, sdr.OUT_CS16, out.data_ptr(), C * n, n, _lib.EINVAL),            # odd n_int16
        (src.data_ptr(), 6000, 3, out.data_ptr(), C * n, n, _lib.EINVAL),                       # bad format
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr(), C * n, n - 1, _lib.ECAPACITY),     # stride
        (src.data_ptr(), 6000, sdr.OUT_CS16, out.data_ptr(), C * n - 1, n, _lib.ECAPACITY),     # capacity
        (0, 6000, sdr.OUT_CS16, out.data_ptr(), C * n, n, _lib.EINVAL),
    ]
    before = out.cpu().numpy().copy()
    for s, n16, fmt, o, cap, stride, code in bad:
        with pytest.raises(_lib.Rxb200Error) as e:
            h.process_device(s, n16, fmt, o, cap, stride)
        assert e.value.code == code
    with pytest.raises(_lib.Rxb200Error):
        h.process(x[:5], sdr.OUT_CS16)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), before)
    rest = h.process(x[2 * 4001:], sdr.OUT_CS16)
    assert np.array_equal(np.concatenate([first, rest], axis=1), want)
    h.close()


def test_reset_starts_over():
    K, bins, dd = SMALL
    x = np.random.default_rng(5).integers(-32768, 32768, size=2 * 20_000, dtype=np.int32).astype(np.int16)
    h = _handle(K, bins, dd)
    one = h.process(x, sdr.CVT_CS16_CS8)
    h.process(x[:2 * 1234], sdr.CVT_CS16_CS8)          # leaves a history and a phase of M and of K behind
    h.reset()
    assert h.decimated_len(2 * 5) == 5 // dd[0]
    assert np.array_equal(h.process(x, sdr.CVT_CS16_CS8), one)
    h.close()
