"""Seeded sweeps of the specialised rx_fm paths (tests/fm_paths.py) against the port, byte for byte: the split kernel with
the row front end (kernel_kind 1), the stream path (kernel_kind 3) and the fused kernel's specialisations (kernel_kind
0).  Every draw runs as a sequence of calls on chunk boundaries -- calls of one stream may take different kernels -- then
once more as a single call after reset().  The named edge cases of tests/golden/fm_paths_golden.json are checked
against the reference's own sha256."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_paths
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fm_paths_golden.json")
_FIXUPS: dict = {}                   # family -> largest fixup_segments any call reported


def _want(port, d):
    outs, lens = [], None
    for c in range(d.n_channels):
        w, lens, _ = port.fm_run(d.params, d.x[c], d.chunk, return_chunks=True)
        outs.append(w)
    return np.stack(outs), lens


@pytest.mark.parametrize("family,seed", fm_paths.all_ids(), ids=[f"{f}-{s}" for f, s in fm_paths.all_ids()])
def test_fm_path_draw(family, seed, port, monkeypatch):
    d = fm_paths.draw(family, seed)
    assert -1 not in d.kinds + [d.single_kind], d.tags
    for k, v in d.env.items():                          # read once, at create
        monkeypatch.setenv(k, v)
    want, want_lens = _want(port, d)
    dm = fm.FmDemod(d.params, n_channels=d.n_channels)
    try:
        dm.tune(*d.tune)
        parts, lens = [], []
        for i, (a, b) in enumerate(d.calls()):
            got, lg = dm.full_demod(d.x[:, a:b], d.chunk, return_chunks=True)
            st = dm.stats()
            assert st["kernel_kind"] == d.kinds[i], (i, d.kinds, d.tags)
            _FIXUPS[family] = max(_FIXUPS.get(family, 0), st["fixup_segments"])
            parts.append(got)
            lens.append(lg)
        got = np.concatenate(parts, axis=1)
        assert np.array_equal(np.concatenate(lens), want_lens), d.tags
        assert got.shape == want.shape, (got.shape, want.shape, d.tags)
        bad = np.argwhere(got != want)
        assert bad.size == 0, (bad[:5].tolist(), d.kinds, d.tags)
        dm.reset()
        one = dm.full_demod(d.x, d.chunk)
        assert dm.stats()["kernel_kind"] == d.single_kind, d.tags
        assert np.array_equal(one, want), (np.argwhere(one != want)[:5].tolist(), d.tags)
    finally:
        dm.close()


@pytest.mark.parametrize("family", ["rows", "stream", "fused"])
def test_fm_path_fixup_ran(family):
    """Some call of every family left a de-emphasis bracket open after its replay, so the serial fix-up pass ran and was
    checked above."""
    if family not in _FIXUPS:
        pytest.skip("no draw of this family ran in this session")
    assert _FIXUPS[family] > 0


def test_fm_paths_golden_cases():
    """The named edge cases against the reference's own bytes (no reference on the GPU machine: its hashes travel)."""
    gold = json.load(open(GOLDEN))
    cases = fm_paths.golden_cases()
    assert sorted(gold) == sorted(cases)
    for name, (p, chunk, x) in cases.items():
        dm = fm.FmDemod(p)
        got, lens = dm.full_demod(x, chunk, return_chunks=True)
        kind = dm.stats()["kernel_kind"]
        dm.close()
        assert kind == fm_paths.expected_kind(p, 1, x.size, chunk, {}, 0), name
        assert lens.tolist() == gold[name]["result_len"], name
        assert hashlib.sha256(got.tobytes()).hexdigest() == gold[name]["sha256"], name


@pytest.mark.parametrize("P", [1, 2, 3])
def test_fm_rows_margin_boundary(P, port):
    """The de-emphasis replay at the largest that the split kernel holds runs there; one sample more moves the call to
    the fused kernel (same bytes), and past the fused kernel's own limit the call is refused."""
    p = fm_paths.FmParams(downsample=1 << P, downsample_passes=P, comp_fir_size=9, custom_atan=fm_paths.ATAN_FAST,
                          deemph=1, deemph_a=23, rate_out=fm_paths.RATE_OUT[P], rate_out2=48_000)
    w_rows, w_fused = fm_paths.replay_limits(p)
    x = fm_paths.channel_input(np.random.default_rng(P), "loud", 300 * fm_paths.ROW_LEN, True)   # longer than the replays
    chunk = 16 * fm_paths.ROW_I16
    want = port.fm_run(p, x, chunk)
    for warm, kind in ((w_rows, 1), (w_rows + 1, 0), (w_fused, 0)):
        assert fm_paths.expected_kind(p, 1, x.size, chunk, {}, warm) == kind
        dm = fm.FmDemod(p)
        dm.tune(0, warm)
        got = dm.full_demod(x, chunk)
        assert dm.stats()["kernel_kind"] == kind, warm
        assert np.array_equal(got, want), warm
        dm.close()
    dm = fm.FmDemod(p)
    dm.tune(0, w_fused + 1)
    with pytest.raises(fm._lib.Rxb200Error) as e:
        dm.full_demod(x, chunk)
    assert e.value.code == fm._lib.EUNSUPPORTED
    dm.close()
