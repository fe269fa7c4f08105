"""The rx_sdr down-converter model pinned: every named shape of tests/sdr_mix.py in all four recorded formats against
the hashes in tests/golden/sdr_mix_golden.json (tests/golden/make_sdr_mix_golden.py), and the rx_sdr shell's capture-mode
refusals, none of which opens the device or creates a file."""
import json
import os
import subprocess

import pytest

import sdr_mix as sm

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "sdr_mix_golden.json")))
SHELL = os.path.join(ROOT, "host", "rx_sdr_b200")


@pytest.mark.parametrize("name", list(sm.SHAPES))
def test_shape_hashes_every_format(name):
    g = GOLDEN[name]
    x = sm.case_capture(name)
    assert sm.digest(x) == g["input_sha256"]
    y, _ = sm.model(name, x)
    assert list(y.shape) == g["shape"]
    for fmt in sm.FORMATS:
        assert sm.digest(sm.convert(y, fmt)) == g[fmt], fmt


def test_golden_covers_every_shape():
    assert sorted(GOLDEN) == sorted(sm.SHAPES)


@pytest.mark.parametrize("args,env,needle", [
    (["-f", "100M", "-f", "101M", "-s", "250k", "-"], {}, "not to '-'"),
    (["-f", "100M", "-I", "CS8", "-F", "CS8", "out"], {}, "reads CS16"),
    (["-f", "100M", "-f", "100M", "out"], {}, "given twice"),
    (["-f", "100M", "-f", "101M", "-s", "250k", "out"], {"RXB200_CAPTURE_RATE": "2249999"}, "2250000"),
    (["-f", "100M", "-f", "101M", "-s", "250k", "out"], {"RXB200_CAPTURE_RATE": "2249999", "RXB200_CAPTURE_STAGES": "2"},
     "3000000"),
])
def test_shell_capture_refusals_create_no_file(tmp_path, args, env, needle):
    if not os.path.exists(SHELL):
        pytest.skip("host/rx_sdr_b200 not built")
    e = dict(os.environ)
    e.setdefault("RXB200_CAPTURE_RATE", "100000000")
    e.update({"RXB200_CAPTURE_RATE": env.get("RXB200_CAPTURE_RATE", "100000000")})
    if "RXB200_CAPTURE_STAGES" in env:
        e["RXB200_CAPTURE_STAGES"] = env["RXB200_CAPTURE_STAGES"]
    else:
        e.pop("RXB200_CAPTURE_STAGES", None)
    r = subprocess.run([SHELL, "-d", "driver=file,path=" + str(tmp_path / "none.cs16")] + args, cwd=tmp_path, env=e,
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and needle in r.stderr, r.stderr
    assert os.listdir(tmp_path) == []
