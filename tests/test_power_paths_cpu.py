"""CPU side of the rx_power path sweeps (tests/power_paths.py): the draws reach every path of
``rxb200_power_accumulate_device`` on both sides of each boundary, the planner equals the reference's
``frequency_range`` on every cli draw and the port equals the reference there, and the port reproduces the reference
hashes of tests/golden/power_paths_golden.json."""
import json
import os

import numpy as np
import pytest

import power_paths
from rx_tools_b200.synth import digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "power_paths_golden.json")


@pytest.fixture(scope="module")
def draws():
    return {fam: [power_paths.draw(fam, s) for s in range(n)] for fam, n in power_paths.N_DRAWS.items()}


def _run(draws):
    return [d for ds in draws.values() for d in ds if not d.dropped]


def test_every_path_row_is_reached(draws):
    ds = _run(draws)
    keys = set().union(*(d.tags["paths"] for d in ds))
    # power_fft8_kernel<E, T>: every E at 512 (E <= 12) and 1024, E 13 at 1024 only, whatever the knob says
    assert {k for k in keys if k[0] == "fft8"} == {("fft8", e, 512) for e in range(3, 13)} | \
        {("fft8", e, 1024) for e in range(3, 14)}
    t512_at_13 = [d for d in ds if d.env.get("RXB200_POWER_THREADS") == "512" and d.plan.bin_e == 13]
    assert t512_at_13 and all(d.paths[-1]["threads"] == 1024 for d in t512_at_13)
    # the generic kernel under RXB200_POWER_V1 on the fast path's shapes, every NB, both table placements
    v1 = [d for d in ds if "RXB200_POWER_V1" in d.env]
    assert {d.plan.bin_e for d in v1 if d.paths[-1]["kernel"] == "generic"} == set(range(1, 14))
    assert {k[1] for k in keys if k[0] == "generic"} == set(power_paths.NB_LADDER)
    assert {k[2] for k in keys if k[0] == "generic"} == {0, 1}
    assert {("rms",), ("big_load",), ("big_decim",)} <= keys
    # every NB with boxcar and with -F, the FIR on and off
    gen = [d for d in ds if d.tags["kernel"] == "generic"]
    for nb in power_paths.NB_LADDER:
        assert any(d.tags["boxcar"] for d in gen if d.paths[-1]["nb"] == nb), nb
        assert any(d.tags["F"] for d in gen if d.paths[-1]["nb"] == nb), nb
    assert {(d.tags["F"], d.tags["fir"]) for d in gen if d.tags["F"]} == {(1, 0), (1, 1)}
    assert {d.plan.downsample_passes for d in gen if d.tags["F"]} >= set(range(1, 7))
    # peak hold on the fast, generic, rms and big paths
    assert {d.tags["kernel"] for d in ds if d.plan.peak_hold} >= {"fft8", "generic", "rms", "big_load", "big_decim"}


def test_boundaries_are_met_from_both_sides(draws):
    geo = draws["geometry"]
    sides = {(d.tags["what"], d.tags.get("side"), d.tags["kernel"]) for d in geo}
    assert ("smem_limit", "below", "generic") in sides or ("smem_limit", "below", "fft8") in sides
    assert {("smem_limit", "above", "big_load"), ("smem_limit", "above", "big_decim")} <= sides
    for d in geo:
        if d.tags["what"] == "smem_limit":
            big = power_paths.is_big(d.plan)
            assert big == (d.tags["side"] == "above"), d.tags
            # the pair is adjacent: the buffer 8 int16 shorter (or longer) than it is valid on the other side, or not
            assert (16 + 256 + 2 * d.plan.buf_len > power_paths.SMEM_LIMIT) == big
    flip = [(d.tags["side"], d.paths[-1]["tables_in_smem"]) for d in geo if d.tags["what"] == "tables_flip"]
    assert sorted(set(flip)) == [("in", 1), ("out", 0)]
    assert any(d.tags["partial_slot"] for d in geo) and any(d.tags["partial_block"] for d in geo)
    assert any(d.tags["partial_slot"] and d.tags["partial_block"] for d in geo)


def test_launch_and_tables_coverage(draws):
    ds = _run(draws)
    slices = set().union(*(d.tags["slices"] for d in ds))
    assert 1 in slices and max(slices) >= 2
    assert any(max(d.tags["slices"]) >= 2 for d in ds if d.tags["kernel"] == "fft8")
    assert any(max(d.tags["slices"]) >= 2 for d in ds if d.tags["kernel"] == "generic")
    launch = draws["launch"]
    assert sorted(d.tags["ranks"] for d in launch if d.tags["what"] == "shard") == list(power_paths.SHARD_RANKS)
    assert {d.plan.n_hops for d in launch if d.tags["what"] == "many_hops"} == {131, 264, 600}
    assert any(d.n_pass == 700 for d in launch)
    assert {d.tags["kernel"] for d in launch if d.device} >= {"fft8", "generic", "rms"}
    tab = draws["tables"]
    assert {(d.tags["kernel"], d.tags["triv"]) for d in tab if d.sine is not None} >= \
        {("fft8", 0), ("fft8", 1), ("generic", 0), ("generic", 1)}
    assert any(d.sine is not None and (d.sine == -32768).any() for d in tab)
    w = np.concatenate([d.window for d in tab if d.tags["window"] == "int32"])
    assert (w >= 1 << 16).any() and (w < 0).any()
    inputs = {d.tags["input"] for d in ds}
    assert inputs == set(power_paths.INPUTS)
    assert any(d.tags["silent"] for d in ds)
    assert {d.tags.get("split") for d in ds} >= {"whole", "passes", "hops", "both", "shard"}


def test_cli_family(draws):
    cli = draws["cli"]
    run = [d for d in cli if not d.dropped]
    dropped = [d for d in cli if d.dropped]
    assert len(run) >= 120 and all(d.dropped == "size cap" for d in dropped), [d.dropped for d in dropped]
    assert {d.tags["mode"] for d in run} == {"boxcar", "F0", "F9"}
    assert {d.tags["window"] for d in run} == set(power_paths.WINDOWS)
    assert {d.tags["crop"] for d in run} == {0.0, 0.1, 0.285, 0.5}
    assert {d.tags["kernel"] for d in run} >= {"fft8", "generic", "big_load", "big_decim"}
    assert min(d.plan.bin_e for d in run) == 1 and max(d.plan.downsample for d in run if d.plan.boxcar) > 500
    assert max(d.plan.downsample_passes for d in run) >= 8


@pytest.mark.ref
@pytest.mark.parametrize("seed", range(power_paths.N_DRAWS["cli"]))
def test_cli_draw_port_equals_reference(seed, port, ref_power):
    """rxb200_power_plan_range equals the reference's frequency_range, and the port the reference's scanner."""
    d = power_paths.draw("cli", seed)
    c = d.cli
    custom = None
    if c["window"] == "hann" and d.plan:                 # plain Hann is a host-built table, not a reference -w shape
        custom = power_paths.power.window_table("hann", 1 << d.plan.bin_e)
    try:
        rp = ref_power.setup(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"], c["window"], custom)
    except RuntimeError:
        assert d.dropped and d.dropped.startswith("planner"), d.dropped
        return
    assert d.plan is not None
    assert (rp.tune_count, rp.bin_e, rp.buf_len, rp.downsample, rp.downsample_passes, rp.rate) == \
        (d.plan.n_hops, d.plan.bin_e, d.plan.buf_len, d.plan.downsample, d.plan.downsample_passes, d.plan.rate)
    assert rp.crop == d.plan.crop
    if d.dropped:
        return
    win, sine = ref_power.tables()
    assert np.array_equal(win, d.window) or d.plan.bin_e == 0
    avg_r, smp_r = ref_power.scan(d.x, d.n_pass)
    avg_p, smp_p = power_paths.port_result(port, d)
    assert np.array_equal(smp_p, smp_r)
    assert np.array_equal(avg_p, avg_r)


def test_port_reproduces_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(power_paths.GOLDEN_CASES)
    for name, c in power_paths.GOLDEN_CASES.items():
        plan = power_paths.golden_plan(c)
        e = gold[name]
        assert [plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes] == e["plan"], name
        win = power_paths.power.window_table(c["window"], 1 << plan.bin_e)
        avg, smp = port.power_scan(power_paths.oracle_params(plan), win, power_paths.golden_input(c, plan),
                                   c["n_pass"], plan.n_hops)
        assert digest(avg) == e["avg_sha256"], name
        assert smp.tolist() == e["samples"], name


def test_golden_covers_the_edges():
    want = {"box1400_bin_e1": (1, 1400, 0), "box311_bin_e7": (7, 311, 0), "F9_P8_bin_e1": (1, 256, 8),
            "F9_P10_bin_e1": (1, 1024, 10), "bin_e15_global_tables": (15, None, 0), "rms_bin_e0": (0, 1, 0)}
    for name, (e, ds, P) in want.items():
        plan = power_paths.golden_plan(power_paths.GOLDEN_CASES[name])
        assert (plan.bin_e, plan.downsample_passes) == (e, P), name
        assert ds is None or plan.downsample == ds, name
    paths = {name: power_paths.expected_path(power_paths.golden_plan(c), {}, c["n_pass"], 1)
             for name, c in power_paths.GOLDEN_CASES.items()}
    assert paths["bin_e15_global_tables"]["tables_in_smem"] == 0
    lim = power_paths.golden_plan(power_paths.GOLDEN_CASES["smem_limit_box7_bin_e13"])
    assert not power_paths.is_big(lim) and 16 + 256 + 2 * (lim.buf_len + 2 * (2 << lim.bin_e)) > power_paths.SMEM_LIMIT
    assert {p["kernel"] for p in paths.values()} >= {"rms", "fft8", "generic"}
