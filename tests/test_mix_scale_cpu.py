"""The restated launch rules of fm_mix.cu (tests/mix_scale.py) at the points the GPU tests lean on, and the sparse DDC
model against fm_ddc.ddc_model: every shape, one call at a far table phase, and a ragged read sequence that carries the
history from read to read, on the CPU."""
import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import mix_scale as ms
from rx_tools_b200 import fm

H100_SMS = 132


def test_mix_trips_bound():
    # a full grid row is 1056 CTAs: its last CTA makes a second trip once the call has more than (2 * 1056 - 1) * 256
    # units of 8 samples
    edge = (2 * 1056 - 1) * 256 * 8
    assert ms.mix_trips_at_least(edge, 1, H100_SMS) == 1
    assert ms.mix_trips_at_least(edge + 1, 1, H100_SMS) == 2
    assert ms.mix_trips_at_least(2 * H100_SMS * 8 * 2048 + 5, 1, H100_SMS) == 2
    assert ms.mix_trips_at_least(98304, 1, H100_SMS) == 1          # the longest call of the short tests
    # a grid row of a 3-row call has a third of the CTAs
    assert ms.mix_trips_at_least(2 * H100_SMS * 8 * 2048 // 3 + 8, 3, H100_SMS) == 2
    assert ms.mix_trips_at_least(1, 1, H100_SMS) == 1


def test_mix_smem_rule():
    assert ms.mix_uses_smem([48] * 256)                               # 96 KiB exactly
    assert not ms.mix_uses_smem([48] * 255 + [49])
    assert ms.mix_uses_smem([48] * 600)                               # every grid row within the limit
    assert not ms.mix_uses_smem([1] * 512 + [12289])                  # the last grid row alone beyond it
    assert ms.mix_uses_smem([12288]) and not ms.mix_uses_smem([1 << 20])
    assert ms.groups(256) == 1 and ms.groups(257) == 2 and ms.groups(600) == 3


def test_ddc_regimes():
    # the tool's operating point: M = 64, T = 257, 300 k outputs are span-bound at 124 outputs (8 129 staged samples)
    assert ms.ddc_regime(300_000, 64, 257, 1, H100_SMS) == (124, "span")
    assert (124 - 1) * 64 + 257 == 8129
    # M = 4096, T <= 16: 2^28 samples (65 536 outputs) share out at 249; 2 n_sm 256 + 64 outputs reach 256
    assert ms.ddc_regime(65536, 4096, 16, 1, H100_SMS) == (249, "n_out")
    assert ms.ddc_regime(2 * H100_SMS * 256 + 64, 4096, 16, 1, H100_SMS) == (256, "reach")
    assert ms.ddc_regime(2 * H100_SMS * 256 + 64, 4096, 1, 1, H100_SMS) == (256, "reach")
    # T < M stages T samples per output; T = 8192 leaves room for one output
    assert ms.ddc_regime(10 ** 6, 100, 31, 1, H100_SMS) == ((8192 - 31) // 31 + 1, "span")
    assert ms.ddc_regime(500, 8, 8192, 1, H100_SMS) == (1, "span")
    assert ms.ddc_regime(1, 1, 1, 1, H100_SMS) == (1, "n_out")
    assert [ms.ddc_lanes(T) for T in (1, 2, 3, 7, 16, 29, 257)] == [1, 2, 4, 8, 16, 32, 32]
    # two grid rows share out over half the CTAs
    assert ms.ddc_ctas(257, H100_SMS) == H100_SMS and ms.ddc_ctas(1, H100_SMS) == 2 * H100_SMS
    assert ms.ddc_regime(2 * H100_SMS * 100, 64, 257, 257, H100_SMS) == (124, "span")
    assert ms.ddc_regime(2 * H100_SMS * 100, 64, 257, 1, H100_SMS) == (100, "n_out")


@pytest.mark.parametrize("name", sorted(fdd.SHAPES))
def test_sparse_model_equals_the_model(name):
    """Every shape's first channel over its read sequence, read by read with the history carried, and the whole capture
    at once split by reads."""
    _, rate, offs, ddc, x, reads = fdd.case_input(name, seed=4)
    M, taps, S = ddc
    for f in (offs[0], offs[-1]):
        t = fm.mix_table(rate, f)
        want = fdd.decimated_reads(x, t, ddc, reads)
        pos, hist = 0, None
        for (a, n), w in zip(fac.seq_bounds(x.size, reads), want):
            y, h2 = ms.ddc_sparse(x[a:a + n], t, taps, M, S, pos, hist)
            _, hw = fdd.ddc_model(x[a:a + n], t, taps, M, S, pos, hist)
            assert np.array_equal(y, w) and np.array_equal(h2, hw), (name, f, a)
            pos, hist = pos + n // 2, h2
        whole = ms.sparse_reads(x, t, ddc, reads)
        assert all(np.array_equal(a, b) for a, b in zip(whole, want)), (name, f)


@pytest.mark.parametrize("decim,n_taps,shift", [(1, 1, 0), (7, 29, 3), (100, 31, 15), (16, 7, 2), (4096, 16, 3)])
def test_sparse_model_far_phase_random_taps(decim, n_taps, shift):
    """One call at table phase 2^40 + 3 with large random taps (saturating outputs) and a random history."""
    rng = np.random.default_rng(decim + n_taps)
    taps = rng.integers(-(1 << 20), 1 << 20, size=n_taps).astype(np.int32)
    t = fm.mix_table(2_400_000, 37500)
    n = max(3 * decim + 5, 4001)
    x = rng.integers(-32768, 32768, size=2 * n).astype(np.int16)
    hist = rng.integers(-32768, 32768, size=2 * (n_taps - 1)).astype(np.int16)
    for pos in (0, 5, decim - 1):
        phase = (1 << 40) + 3
        want, wh = fdd.ddc_model(x, t, taps, decim, shift, pos, hist, table_phase=phase)
        got, gh = ms.ddc_sparse(x, t, taps, decim, shift, pos, hist, table_phase=phase)
        assert want.size and np.array_equal(got, want) and np.array_equal(gh, wh), pos


def test_sparse_model_is_the_mixer_at_identity():
    x = fmx.capture(3001, 2_400_000, [12500], 21)
    t = fm.mix_table(2_400_000, 12500)
    y, h = ms.ddc_sparse(x, t, np.ones(1, np.int32), 1, 0, 0, None, table_phase=17)
    assert np.array_equal(y, fmx.mix_model(x, t, 17)) and h.size == 0
