"""The port against the unmodified reference (oracle/_ref) on every draw of tests/fm_paths.py: the GPU sweeps compare
with the port, so the port must give the reference's bytes wherever the sweeps go."""
import numpy as np
import pytest

import fm_paths

pytestmark = pytest.mark.ref


@pytest.mark.parametrize("family", sorted(fm_paths.N_DRAWS))
def test_port_is_reference_on_every_draw(family, port, ref_fm):
    for seed in range(fm_paths.N_DRAWS[family]):
        d = fm_paths.draw(family, seed)
        for c in range(d.n_channels):
            want, lw, _ = ref_fm.run(d.params, d.x[c], d.chunk, return_chunks=True)
            got, lg, _ = port.fm_run(d.params, d.x[c], d.chunk, return_chunks=True)
            assert np.array_equal(lg, lw), (family, seed, c)
            assert got.size == want.size and np.array_equal(got, want), (family, seed, c, np.flatnonzero(got != want)[:5])
