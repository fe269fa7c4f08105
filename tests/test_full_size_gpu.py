"""BASELINE.json's full sizes, pinned to the UNMODIFIED reference: tests/golden/full_golden.json holds the sha256 of what
oracle/_ref produced for the exact inputs of tests/full_inputs.py (minted in the authoring container by
tests/golden/make_full_golden.py; the reference needs ~50 s for all of it).  The CUDA path runs the same inputs
through the C-ABI and must reproduce the hashes: 1 GiB rx_fm streams (2 048 chunks, every per-chunk result_len),
cfg1 at 2^20 samples (24 576 PCM), 256 channels x 2.4 M (cfg5A), 871 hops x 36 sweeps (every row + the CSV), 610
hop buffers (cfg3).  The fp64 atan2 outputs are compared with the reference's vectors byte for byte, unless the port, run
over the same input, meets an atan2 value within 2^-30 of an integer (where CUDA's libm and glibc's may truncate
differently): then <= 1 LSB on <= 1e-5 of the samples."""
import json
import os

import numpy as np
import pytest

import fm_disc as fd
import full_inputs as FI
import oracle
from cases import fm_cases
from rx_tools_b200 import fm, power
from rx_tools_b200.synth import digest

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = json.load(open(os.path.join(G, "full_golden.json")))
VEC = np.load(os.path.join(G, "full_std_vectors.npz"))


def _close_to_reference(got, want, params, x, chunk16):
    assert got.size == want.size
    oracle.port().fm_run(params, x, chunk16)
    if not fd.port_met_near_integer():
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (bad.size, bad[:5], got[bad[:5]], want[bad[:5]])
        return
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max() <= 1, d.max()
    assert np.count_nonzero(d) <= max(1, int(1e-5 * d.size)), np.count_nonzero(d)


@pytest.fixture(scope="module")
def one_gib():
    period = FI.fm_one_gib_period()
    assert digest(period) == GOLD["fm2b"]["period_sha256"]
    return np.tile(period, FI.FM_TILES)


@pytest.mark.parametrize("name,cli", [("fm2b", dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9)),
                                      ("fm2a", dict(wbfm=1, rate_s=2400000, rate_r=48000))])
def test_fm_one_gib_equals_reference(one_gib, name, cli):
    g = GOLD[name]
    p = fm.derive_params(**cli).params
    assert p.reference_fields() == {k: v for k, v in g["params"].items()}       # the reference's own optimal_settings()
    assert one_gib.size == g["n_in_int16"] and one_gib.size * 2 == 1 << 30
    dem = fm.FmDemod(p)
    got, lens = dem.full_demod(one_gib, FI.CHUNK16, return_chunks=True)
    assert got.size == g["n_out"] == 5368709
    assert [int(v) for v in got[:8]] == g["head"] and [int(v) for v in got[-8:]] == g["tail"]
    assert digest(lens.astype(np.int32)) == g["chunk_result_len_sha256"]
    assert digest(got) == g["output_sha256"], "1 GiB stream differs from the reference"
    # size-independent property on top: two calls split on a chunk boundary == one call (device-side carry)
    dem.reset()
    cut = (one_gib.size // 3 // FI.CHUNK16) * FI.CHUNK16
    a = dem.full_demod(one_gib[:cut], FI.CHUNK16)
    b = dem.full_demod(one_gib[cut:], FI.CHUNK16)
    assert digest(np.concatenate([a, b])) == g["output_sha256"]
    dem.close()


@pytest.mark.parametrize("nm,atan", [("std", 0), ("fast", 1), ("lut", 2)])
def test_cfg1_at_two_to_the_twenty(nm, atan):
    g = GOLD[f"cfg1_{nm}"]
    x = FI.cfg1_input()
    assert digest(x) == g["input_sha256"]
    p = fm.derive_params(rate_s=1024000, rate_r=24000, custom_atan=atan).params
    assert p.reference_fields() == g["params"]
    dem = fm.FmDemod(p)
    got = dem.full_demod(x, FI.CHUNK16)
    assert got.size == g["n_out"] == 24576                   # BASELINE.md §2: 2^20 samples -> exactly 24 576 PCM
    if atan == 0:
        _close_to_reference(got, VEC["cfg1_std_full"], oracle.FmParams(**p.reference_fields()), x, FI.CHUNK16)
    else:
        assert digest(got) == g["output_sha256"]
    dem.close()


@pytest.mark.parametrize("case", [c for c in fm_cases() if not c.exact], ids=lambda c: c.name)
def test_atan2_cases_against_reference_vectors(case):
    """The float path against what the reference itself produced (not only the port)."""
    dem = fm.FmDemod(case.params)
    x = case.make_input()
    got = dem.full_demod(x, case.chunk_int16)
    _close_to_reference(got, VEC["case_" + case.name], case.params, x, case.chunk_int16)
    dem.close()


def test_cfg5a_256_channels():
    g = GOLD["cfg5A"]
    xs = np.stack([FI.cfg5_channel(ch) for ch in range(FI.CFG5_CHANNELS)])
    assert xs.shape == (256, 2 * 2_400_000)
    p = fm.FmParams.from_any(oracle.FmParams(**g["params"]))
    dem = fm.FmDemod(p, n_channels=FI.CFG5_CHANNELS)
    got = dem.full_demod(xs, FI.CHUNK16)
    assert got.shape == (256, g["n_out_per_channel"]) and g["n_out_per_channel"] == 24000
    for ch, sha in g["channel_sha256"].items():
        assert digest(got[int(ch)]) == sha, f"channel {ch}"
    assert digest(got) == g["all_channels_sha256"]
    dem.close()


def test_cfg4_871_hops_36_sweeps():
    g = GOLD["cfg4"]
    plan = power.plan_range("24M:1766M:1k", 0.285)
    assert (plan.n_hops, plan.bin_e) == (g["tune_count"], g["bin_e"]) == (871, 12)
    hb = FI.cfg4_hops(plan.n_hops, plan.buf_len)
    assert digest(hb) == g["input_sha256"]
    sc = power.PowerScanner(plan, "hamming")
    sc.scanner(hb, FI.CFG4_PASSES)
    avg, smp = sc.read()
    assert int(smp[0]) == g["samples"] and np.all(smp == smp[0])
    for i, sha in g["row_sha256"].items():
        assert digest(avg[int(i)]) == sha, f"hop {i}"
    assert digest(avg) == g["avg_sha256"], "spectrum rows differ from the reference"
    # the report: csv_dbm()'s text for all 871 rows, dB values computed on the device
    csv = sc.csv_rows_device()
    assert digest(np.frombuffer(csv.encode(), dtype=np.uint8)) == g["csv_sha256"]
    # exact additivity over passes (int64 sums): the same sweeps in two batches
    sc.reset()
    sc.scanner(hb[:10], 10)
    sc.scanner(hb[10:], FI.CFG4_PASSES - 10)
    avg2, _ = sc.read()
    assert digest(avg2) == g["avg_sha256"]
    sc.close()


def test_cfg3_610_hop_buffers():
    g = GOLD["cfg3"]
    plan = power.plan_range("100M:101M:1k")
    hb = FI.cfg3_hops(plan.buf_len)
    assert digest(hb) == g["input_sha256"]
    sc = power.PowerScanner(plan, "hann")
    sc.scanner(hb, FI.CFG3_BUFFERS)
    avg, smp = sc.read()
    assert int(smp[0]) == g["samples"] == 4880
    assert [int(v) for v in avg.reshape(-1)[:8]] == g["avg_head"]
    assert digest(avg) == g["avg_sha256"]
    sc.close()
