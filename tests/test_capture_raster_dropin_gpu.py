"""Both drop-in shells in capture mode with RXB200_CAPTURE_STAGES=raster on the replay device: the plan is
rxb200_fm_plan_capture_raster's and the handle a raster handle.  rx_sdr_b200: every channel's file in each -F format
equals the model under two sets of read lengths, -n N gives N samples per file, and the 100-station FM broadcast band
is recorded whole.  rx_fm_b200: every channel's file equals a raster FmMix handle fed the shell's blocks, under two sets
of read lengths.  In both shells the channel at the centre is byte for byte the default capture mode's file."""
import os
import subprocess

import numpy as np
import pytest

import fm_capture as fcp
import fm_raster as frs
import sdr_mix as sm
from rx_tools_b200 import fm, power, sdr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_SDR = os.path.join(ROOT, "host", "rx_sdr_b200")
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
READS = ("1000:7777", "40000:3:50001")


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(exe, argv, cap, out, env, reads):
    e = dict(os.environ)
    e.pop("RXB200_CAPTURE_STAGES", None)
    e.update(env)
    r = subprocess.run([exe, "-d", f"driver=file,path={cap},reads={reads}"] + argv + [str(out)], capture_output=True,
                       timeout=900, env=e)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r.stderr.decode()


# ---- rx_sdr_b200: four channels on a 200 kHz grid at -s 250k: fc = 100 MHz, M = 5, R = 1.25 Msps, K = 25
SDR_TUNED = [100_000_000, 100_200_000, 100_400_000, 99_600_000]


def _sdr_case():
    plan, bins = fm.plan_capture_raster(SDR_TUNED, 250_000, 1 << 30)
    x = np.random.default_rng(6).integers(-20000, 20001, size=2 * 150_007, dtype=np.int32).astype(np.int16)
    taps = power.ddc_lowpass(plan.decim, plan.n_taps, 15)
    want = frs.raster_model(x, plan.n_bins, bins, taps, plan.decim, plan.shift)[0]
    return plan, bins, x, want


@pytest.mark.parametrize("fout", ["CS16", "CS8", "CU8", "CF32"])
def test_rx_sdr_files_equal_model(tmp_path, fout):
    plan, bins, x, want = _sdr_case()
    assert (plan.centre_hz, plan.decim, plan.capture_rate, plan.n_bins) == (100_000_000, 5, 1_250_000, 25)
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    args = sum((["-f", str(f)] for f in SDR_TUNED), []) + ["-s", "250k", "-F", fout]
    env = {"RXB200_CAPTURE_RATE": str(plan.capture_rate), "RXB200_CAPTURE_STAGES": "raster"}
    files = {}
    for reads in READS:
        err = _run(RX_SDR, args, cap, tmp_path / "out", env, reads)
        assert (f"Capture mode: {plan.capture_rate} Hz centred at {plan.centre_hz} Hz as a raster: {plan.n_bins} bins, "
                f"decimation {plan.decim}, {plan.n_taps} taps, {len(SDR_TUNED)} channels") in err
        files[reads] = [open(f"{tmp_path / 'out'}.{f}", "rb").read() for f in SDR_TUNED]
    assert files[READS[0]] == files[READS[1]]
    for k in range(len(SDR_TUNED)):
        assert files[READS[0]][k] == sm.convert(want[k], fout).tobytes(), k
    # the channel at fc (bin 0) is the default capture mode's file
    env.pop("RXB200_CAPTURE_STAGES")
    _run(RX_SDR, args, cap, tmp_path / "dflt", env, READS[0])
    assert open(f"{tmp_path / 'dflt'}.{SDR_TUNED[0]}", "rb").read() == files[READS[0]][0]
    # -n N: N samples per file
    N = 3001
    env["RXB200_CAPTURE_STAGES"] = "raster"
    _run(RX_SDR, args + ["-n", str(N)], cap, tmp_path / "n", env, "4097")
    E = sdr.ELEM_BYTES[sdr.FORMATS[fout]]
    for k, f in enumerate(SDR_TUNED):
        b = open(f"{tmp_path / 'n'}.{f}", "rb").read()
        assert len(b) == N * E and b == sm.convert(want[k], fout).tobytes()[:N * E]


def test_rx_sdr_fm_broadcast_band(tmp_path):
    """One -f per station of the FM broadcast band at -s 250k: 100 files the model reproduces, K = 405, M = 81."""
    tuned = [88_100_000 + 200_000 * k for k in range(100)]
    plan, bins = fm.plan_capture_raster(tuned, 250_000, 25_000_000)
    x = np.random.default_rng(7).integers(-3000, 3001, size=2 * (81 * 400 + 55), dtype=np.int32).astype(np.int16)
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    args = sum((["-f", str(f)] for f in tuned), []) + ["-s", "250k", "-F", "CS16"]
    err = _run(RX_SDR, args, cap, tmp_path / "fm", {"RXB200_CAPTURE_RATE": "25000000", "RXB200_CAPTURE_STAGES": "raster"},
               "16384")
    assert "as a raster: 405 bins, decimation 81, 2593 taps, 100 channels" in err
    want = frs.raster_model(x, 405, bins, power.ddc_lowpass(81, 2593, 15), 81, 30)[0]
    for k, f in enumerate(tuned):
        assert open(f"{tmp_path / 'fm'}.{f}", "rb").read() == want[k].tobytes(), f


# ---- rx_fm_b200: three NBFM channels on a 25 kHz grid: c = 1.008 Msps, M = 2, R = 2.016 Msps, K = 2016
FM_F = ["162.4M", "162.425M", "162.45M"]


def _fm_expected(p, pl, bins, x):
    """A raster FmMix handle fed the shell's blocks: each channel's PCM, concatenated."""
    taps = power.ddc_lowpass(pl.decim, pl.n_taps, 15)
    h = fm.FmMix(p, ddc=(pl.decim, taps, pl.shift), raster=(pl.n_bins, bins))
    parts, at = [], 0
    for b in fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p)):
        parts.append(np.atleast_2d(h.process_read(x[2 * at:2 * (at + b)])))
        at += b
    h.close()
    return [np.concatenate([q[k] for q in parts]).tobytes() for k in range(len(bins))]


def test_rx_fm_files_equal_raster_handle(tmp_path):
    der = fm.derive_params(offset_tuning=1)
    freqs = fcp.freqs_of(FM_F)
    tuned = fcp.tuned_of(freqs, der)
    pl, bins = fm.plan_capture_raster(tuned, der.capture_rate, 10**10)
    assert (pl.decim, pl.capture_rate, pl.n_bins, pl.centre_hz) == (2, 2_016_000, 2016, tuned[1])
    dp, offs = fm.plan_capture(tuned, der.capture_rate, 10**10)
    x = fcp.capture(2 * 2 * fcp.CHUNK + 70001, pl.capture_rate, offs, 2300)
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    argv = [a for v in FM_F for a in ("-f", v)]
    env = {"RXB200_CAPTURE_RATE": "40000000", "RXB200_CAPTURE_STAGES": "raster"}
    want = _fm_expected(der.params, pl, bins, x)
    files = {}
    for reads in ("5000:12345:777", "131072"):
        err = _run(RX_FM, argv, cap, tmp_path / "out", env, reads)
        assert (f"Capture mode: {pl.capture_rate} Hz centred at {pl.centre_hz} Hz as a raster: {pl.n_bins} bins, "
                f"decimation {pl.decim}, {pl.n_taps} taps, 3 channels") in err
        files[reads] = [open(f"{tmp_path / 'out'}.{f}", "rb").read() for f in freqs]
        assert files[reads] == want and all(len(f) > 0 for f in want), reads
    # the channel at fc (bin 0) is the default capture mode's file
    env.pop("RXB200_CAPTURE_STAGES")
    _run(RX_FM, argv, cap, tmp_path / "dflt", env, "5000:12345:777")
    assert bins[1] == 0 and open(f"{tmp_path / 'dflt'}.{freqs[1]}", "rb").read() == want[1]
