"""CPU side of the rx_fm path sweeps (tests/fm_paths.py): the draws reach every region they are meant to reach, the
planner figures the expectations restate match the build, and the port gives the reference's bytes on the named edge
cases of tests/golden/fm_paths_golden.json."""
import hashlib
import json
import os
import re
from collections import defaultdict

import pytest

import fm_paths

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_paths_golden.json")
PTXAS_LOG = os.path.join(os.path.dirname(HERE), "rx_tools_b200", "csrc", "fm_kernels.ptxas.log")


@pytest.fixture(scope="module")
def draws():
    return {fam: [fm_paths.draw(fam, s) for s in range(n)] for fam, n in fm_paths.N_DRAWS.items()}


def _seen(ds, key):
    out = set()
    for d in ds:
        v = d.tags[key]
        out.update(v if isinstance(v, list) else [v])
    return out


def test_rows_family_coverage(draws):
    ds = draws["rows"]
    assert {(d.tags["P"], d.tags["fir"], d.tags["serial"]) for d in ds} == \
        {(P, f, s) for P in (1, 2, 3) for f in (0, 9) for s in fm_paths.SERIAL}
    assert _seen([d for d in ds if d.params.deemph], "a") == set(fm_paths.ROWS_A)
    assert _seen([d for d in ds if d.params.rate_out2 > 0], "rate_out2") == set(fm_paths.RATE_OUT2)
    assert _seen(ds, "chunk_rows") == set(fm_paths.ROWS_CHUNK_ROWS)
    assert _seen([d for d in ds if d.params.deemph], "warm_is") == {"0", "1", "7", "a", "4a"}
    assert _seen(ds, "n_ch") == {1, 2, 3, 4, 5}
    assert set(fm_paths.INPUTS) | {"silent"} <= _seen(ds, "inputs")
    assert {0} | set(range(1, 21)) <= _seen(ds, "seg_rows")
    assert any(d.tags["seg_ragged"] for d in ds)
    assert any(d.tags["rows"] == 16 or d.tags["rows"] < 20 for d in ds) and max(d.tags["rows"] for d in ds) > 300
    # a ragged last chunk, a one-row chunk, margins handed over from 2 and 4 older items
    assert sum(d.tags["rows"] % d.tags["chunk_rows"] != 0 for d in ds) > 50
    assert any(d.tags["chunk_rows"] == 1 and 1 in d.kinds for d in ds)
    assert {2, 4} <= {d.tags["margin_items"] for d in ds if 1 in d.kinds}
    # calls of one stream on the row kernel and on the fused kernel, and row shapes whose margin needs the fused kernel
    assert sum(0 in d.kinds and 1 in d.kinds for d in ds) >= 20
    assert sum(not d.tags["margin_fits"] for d in ds) >= 5
    assert all(d.single_kind == 0 for d in ds if not d.tags["margin_fits"])


def test_stream_family_coverage(draws):
    ds = draws["stream"]
    a = _seen(ds, "a")
    assert any(v % 2 for v in a) and any(v % 2 == 0 for v in a) and {1, 2} <= a and max(a) > 300
    assert _seen(ds, "resample") == {"off", "ratio1", "ratio"}
    assert {0, 64} <= _seen(ds, "piece") and any(p > 64 for p in _seen(ds, "piece"))
    assert _seen(ds, "win") == {128, 256} and _seen(ds, "t") == {32, 64, 128}
    assert sum(3 in d.kinds and 0 in d.kinds for d in ds) >= 30
    assert all(d.chunk % 16 == 0 for d in ds) and any(d.chunk % 2048 for d in ds) and any(d.chunk < 256 for d in ds)
    assert set(fm_paths.INPUTS) | {"silent"} <= _seen(ds, "inputs")


def test_fused_family_coverage(draws):
    ds = draws["fused"]
    assert _seen(ds, "shape") == {"spec3", "spec1_boxcar", "spec1_p4"}
    assert all(d.kinds == [0] * len(d.kinds) and d.single_kind == 0 for d in ds)
    assert max(d.tags["D"] for d in ds if d.tags["shape"] == "spec3") > 200
    assert _seen([d for d in ds if d.tags["shape"] == "spec3"], "n_ch") >= {1, 8}


def test_no_draw_expects_a_refusal(draws):
    for fam, ds in draws.items():
        for d in ds:
            assert -1 not in d.kinds and d.single_kind != -1, (fam, d.seed)


def test_kernels_static_shared_memory():
    """The fit rules in fm_paths restate fm_plan_rows and fm_plan_segments, which subtract the kernels' static shared
    memory from what a CTA may have."""
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no ptxas log: librxb200 was not built in this tree")
    text = open(PTXAS_LOG).read()
    found = re.findall(r"Compiling entry function '(\w+)'.*?Used \d+ registers.*?(\d+) bytes smem", text, re.S)
    split = {int(s) for n, s in found if "fm_split_kernel" in n}
    fused = {int(s) for n, s in found if re.search(r"fm_fused_kernelILi\d+ELi[012]E", n)}
    assert split == {fm_paths.SPLIT_STATIC_SMEM}
    assert fused == {fm_paths.FUSED_STATIC_SMEM}


def test_port_matches_reference_golden(port):
    """The port against the reference's sha256 of the named edge cases (minted by golden/make_fm_paths_golden.py)."""
    gold = json.load(open(GOLDEN))
    cases = fm_paths.golden_cases()
    assert sorted(gold) == sorted(cases)
    for name, (p, chunk, x) in cases.items():
        assert gold[name]["params"] == {k: int(v) for k, v in vars(p).items()}, name
        got, lens, _ = port.fm_run(p, x, chunk, return_chunks=True)
        assert lens.tolist() == gold[name]["result_len"], name
        assert hashlib.sha256(got.tobytes()).hexdigest() == gold[name]["sha256"], name


def test_golden_covers_fallback_and_edges():
    cases = fm_paths.golden_cases()
    kinds = defaultdict(list)
    for name, (p, chunk, x) in cases.items():
        kinds[fm_paths.expected_kind(p, 1, x.size, chunk, {}, 0)].append(name)
    assert {0, 1, 3} <= set(kinds), kinds
    assert "cli_s1200k_F9_r48k_c450" in kinds[0] and "cli_s1200k_F9_c500" in kinds[0]
