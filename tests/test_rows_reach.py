"""The row front end (rx_tools_b200/csrc/fm_rows.cuh, row_start_state) rebuilds the filter state in front of a warp's
first row from the last 128 input samples of the row before it.  That is exact only if the chain scale -> rotate ->
P half-band passes -> droop FIR -> discriminator forgets everything older than 128 input samples.  Pinned here on the
port oracle: the PCM after a row-aligned point S must not change when everything more than 128 samples before S is
replaced by silence."""
import numpy as np
import pytest

import oracle
from rx_tools_b200 import synth

ROW = 1024          # input samples per row


@pytest.mark.parametrize("fir", [0, 9])
@pytest.mark.parametrize("P", [1, 2, 3])
def test_state_at_a_row_start_depends_on_the_last_128_samples_only(P, fir, port):
    p = oracle.FmParams(downsample=1 << P, downsample_passes=P, comp_fir_size=fir, custom_atan=oracle.ATAN_FAST,
                        rate_out=2_400_000 >> P)
    n_pre, n_row, n_s = ROW, ROW, 2 * ROW          # noise, the row R before S, then S; S starts on a row boundary
    n = n_pre + n_row + n_s
    for seed in range(24):
        x = synth.uniform_iq(n, -32768, 32767, 1000 + seed)
        y = x.copy()
        y[: 2 * (n_pre + n_row - 128)] = 0             # zeros + R[-128:] + S
        chunk = 2 * n                                  # one chunk: no chunk start inside
        a = port.fm_run(p, x, chunk)
        b = port.fm_run(p, y, chunk)
        s0 = (n_pre + n_row) >> P                      # first PCM sample of S
        assert a.size == b.size == n >> P
        assert np.array_equal(a[s0:], b[s0:]), (seed, np.flatnonzero(a[s0:] != b[s0:])[:5])
        # the comparison can see a difference: with three passes and the FIR (the longest reach) 64 samples are too few
        if seed == 0 and P == 3 and fir:
            z = x.copy()
            z[: 2 * (n_pre + n_row - 64)] = 0
            assert not np.array_equal(a[s0:], port.fm_run(p, z, chunk)[s0:])
