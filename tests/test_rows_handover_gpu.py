"""The split kernel with the row front end (kernel_kind 1): every front-end warp rebuilds its start state from the last
128 samples of the row before its stretch, and an item's back end takes the margin rows before the item from the
previous items of the channel through global memory (rx_tools_b200/csrc/fm_rows.cuh).  Item lengths of 1, 3 and 16
rows make the margin span four, two and one older items and leave front-end warps without rows; the output must be
the port's, byte for byte."""
import numpy as np
import pytest

from cases import fm_cases
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

SHAPES = ["cfg2B", "wbfm_P1_fir", "wbfm_P2_fir", "wbfm_P2_nofir", "F0_P1", "burst_then_silence", "zeros_P3_deemph"]
SEGS = [1024, 3072, 16384]


def _case(name):
    if name == "zeros_P3_deemph":       # silence on the cfg2B shape: the de-emphasis brackets never close
        c = next(c for c in fm_cases() if c.name == "cfg2B")
        return c.params, (lambda: np.zeros(1 << 20, dtype=np.int16)), c.chunk_int16
    c = next(c for c in fm_cases() if c.name == name)
    return c.params, c.make_input, c.chunk_int16


@pytest.mark.parametrize("seg", SEGS)
@pytest.mark.parametrize("name", SHAPES)
def test_rows_item_lengths(name, seg, port):
    params, make, chunk = _case(name)
    x = make()
    want = port.fm_run(params, x, chunk)
    d = fm.FmDemod(params)
    d.tune(segment_len=seg)
    got = d.full_demod(x, chunk)
    assert d.stats()["kernel_kind"] == 1
    assert d.stats()["segment_len"] <= seg
    assert got.size == want.size and np.array_equal(got, want), np.flatnonzero(got != want)[:5]
    d.close()


@pytest.mark.parametrize("seg", [0, 3072])
@pytest.mark.parametrize("name", ["cfg2B", "wbfm_P1_fir", "wbfm_P2_nofir"])
def test_rows_split_streaming_calls(name, seg, port):
    """Calls of 2, 5 and 1 chunk and the rest: every call's first warp starts from the carry, the others from the
    row before them, and items never reach into the previous call."""
    params, make, _ = _case(name)
    x = make()
    chunk = 65536                       # 32 rows; the input is 16 chunks
    want = port.fm_run(params, x, chunk)
    d = fm.FmDemod(params)
    if seg:
        d.tune(segment_len=seg)
    cuts = [0, 2 * chunk, 7 * chunk, 8 * chunk, x.size]
    parts = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        parts.append(d.full_demod(x[a:b], chunk))
        assert d.stats()["kernel_kind"] == 1
    got = np.concatenate(parts)
    assert got.size == want.size and np.array_equal(got, want), np.flatnonzero(got != want)[:5]
    d.close()


@pytest.mark.parametrize("seg", [0, 1024])
def test_rows_three_channels(seg, port):
    """Margins are handed over within a channel only: channel c's first item starts from its own carry."""
    params, make, chunk = _case("cfg2B")
    x = make()
    n = x.size // 2
    xs = np.stack([x[:n], x[x.size - n:], np.zeros(n, dtype=np.int16)])
    d = fm.FmDemod(params, n_channels=3)
    if seg:
        d.tune(segment_len=seg)
    got = d.full_demod(xs, chunk)
    assert d.stats()["kernel_kind"] == 1
    for ch in range(3):
        assert np.array_equal(got[ch], port.fm_run(params, xs[ch], chunk)), ch
    d.close()
