"""The rx_sdr drop-in shell (host/rx_sdr_b200) on the replay device.  Plain mode: byte for byte what the reference's own
rx_sdr (oracle/_ref/rx_sdr_ref) writes for every -I/-F pair it accepts, with -n, with the default and other -b, and with
read lengths that do not divide -b; without -n, the whole capture through rx_sdr's conversions.  Capture mode
(RXB200_CAPTURE_RATE): every channel's file of both kinds equals the numpy model, two sets of read lengths give the same
files, and -n N gives exactly N samples per file."""
import os
import subprocess

import numpy as np
import pytest

import fm_two_stage as fts
import sdr_inputs as SI
import sdr_mix as sm
from rx_tools_b200 import fm, power, sdr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SHELL = os.path.join(ROOT, "host", "rx_sdr_b200")
REF = os.path.join(ROOT, "oracle", "_ref", "rx_sdr_ref")
# every pair the reference accepts on the replay device, which streams CS16 and CS12 only
PAIRS = [("CS16", "CS16"), ("CS16", "CS8"), ("CS16", "CU8"), ("CS16", "CF32"), ("CS12", "CS16"), ("CS12", "CS12")]


def _run(exe, cap, args, tmp, env=None, reads=None):
    out = os.path.join(tmp, "out.bin")
    dev = f"driver=file,path={cap}" + (f",reads={reads}" if reads else "")
    e = dict(os.environ)
    e.pop("RXB200_CAPTURE_RATE", None)
    e.pop("RXB200_CAPTURE_STAGES", None)
    e.update(env or {})
    r = subprocess.run([exe, "-d", dev] + args + [out], capture_output=True, timeout=300, env=e)
    assert r.returncode == 0, r.stderr.decode()[-600:]
    return out


def _capture(tmp, fin):
    x = SI.cs12_capture() if fin == "CS12" else SI.cs16_capture()
    p = os.path.join(tmp, "cap.bin")
    np.ascontiguousarray(x).tofile(p)
    return x, p


@pytest.mark.parametrize("fin,fout", PAIRS)
@pytest.mark.parametrize("block,reads", [(16384, None), (16384, "5000:16384:777"), (1000, "999:3")])
def test_plain_mode_equals_reference(tmp_path, fin, fout, block, reads):
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/rx_sdr_ref not built")
    x, cap = _capture(str(tmp_path), fin)
    n = SI.N_ELEMS_12 if fin == "CS12" else SI.N_ELEMS
    args = ["-I", fin, "-F", fout, "-n", str(n), "-b", str(block)]
    want = open(_run(REF, cap, args, str(tmp_path), reads=reads), "rb").read()
    got = open(_run(SHELL, cap, args, str(tmp_path), reads=reads), "rb").read()
    assert got == want


@pytest.mark.parametrize("fout", ["CS16", "CS8", "CU8", "CF32"])
def test_plain_mode_whole_capture(tmp_path, fout):
    """Without -n the shell records until the replay ends: every sample through rx_sdr's conversion."""
    x, cap = _capture(str(tmp_path), "CS16")
    got = open(_run(SHELL, cap, ["-I", "CS16", "-F", fout, "-b", "16384"], str(tmp_path), reads="7000:11"), "rb").read()
    assert got == sm.convert(x, fout).tobytes()
    # -n N with N a whole number of reads: the count runs out exactly, and rx_sdr no longer limits the run
    got = open(_run(SHELL, cap, ["-F", fout, "-n", "14000", "-b", "7000"], str(tmp_path)), "rb").read()
    assert got == sm.convert(x, fout).tobytes()


TUNED = [100_000_000, 100_300_000, 100_950_000, 100_123_457]     # M = 5: M' = 8 for two stages


def _capture_case(two):
    x = np.random.default_rng(5).integers(-20000, 20001, size=2 * 200_003, dtype=np.int32).astype(np.int16)
    if two:
        plan, offs = fm.plan_capture_two_stage(TUNED, 250_000, 1 << 30)
        K, coarse, fine = fts.plan_stages(plan.coarse_decim * plan.fine_decim)
        return x, plan.capture_rate, sm.two_stage_model(x, plan.capture_rate, K, offs, coarse, fine)
    plan, offs = sdr.plan_sdr_capture(TUNED, 250_000, 1 << 30)
    dd = (plan.decim, power.ddc_lowpass(plan.decim, plan.n_taps, 15), 15)
    return x, plan.capture_rate, sm.single_model(x, plan.capture_rate, offs, dd)


@pytest.mark.parametrize("two", [False, True])
@pytest.mark.parametrize("fout", ["CS16", "CU8", "CF32"])
def test_capture_mode_files_equal_model(tmp_path, two, fout):
    x, R, want = _capture_case(two)
    cap = os.path.join(str(tmp_path), "cap.cs16")
    x.tofile(cap)
    env = {"RXB200_CAPTURE_RATE": str(R)}
    if two:
        env["RXB200_CAPTURE_STAGES"] = "2"
    args = sum((["-f", str(f)] for f in TUNED), []) + ["-s", "250k", "-F", fout]
    files = {}
    for reads in ("1000:7777", "40000:3:50001"):
        out = _run(SHELL, cap, args, str(tmp_path), env=env, reads=reads)
        files[reads] = [open(f"{out}.{f}", "rb").read() for f in TUNED]
    assert files["1000:7777"] == files["40000:3:50001"]
    for k in range(len(TUNED)):
        assert files["1000:7777"][k] == sm.convert(want[k], fout).tobytes(), k
    N = 3001
    out = _run(SHELL, cap, args + ["-n", str(N)], str(tmp_path), env=env, reads="4097")
    E = sdr.ELEM_BYTES[sdr.FORMATS[fout]]
    for k, f in enumerate(TUNED):
        b = open(f"{out}.{f}", "rb").read()
        assert len(b) == N * E and b == sm.convert(want[k], fout).tobytes()[:N * E]
