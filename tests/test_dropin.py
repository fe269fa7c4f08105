"""Drop-in executables (host/rx_fm_b200, host/rx_power_b200): reference CLI in, reference byte format out,
SoapySDR stream surface served by the replay fake (`-d driver=file,path=...`).  Expected bytes come from the
port oracle driven chunk by chunk exactly as the shells read the stream."""
import os
import subprocess

import numpy as np
import pytest

import oracle
from rx_tools_b200 import fm, power, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
RX_POWER = os.path.join(ROOT, "host", "rx_power_b200")
CHUNK16 = 262144


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(cmd, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, capture_output=True, env=e, timeout=300)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


def _oracle_params(p):
    return oracle.FmParams(**p.reference_fields())


@pytest.mark.parametrize("args,kw", [
    (["-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k"], dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9)),
    (["-M", "wbfm"], dict(wbfm=1)),
    (["-M", "fm", "-s", "24k", "-A", "lut"], dict(rate_s=24000, custom_atan=2)),
    (["-M", "am", "-s", "12k", "-r", "6k"], dict(mode=fm.MODE_AM, rate_s=12000, rate_r=6000)),
    (["-M", "raw", "-s", "250k"], dict(mode=fm.MODE_RAW, rate_s=250000)),
    (["-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k", "-o", "2"],
     dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9, post_downsample=2)),
])
def test_rx_fm_output_bytes(tmp_path, port, args, kw):
    x = synth.cfg2_iq(4 * 131072, seed=31)
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    out = tmp_path / "out.raw"
    _run([RX_FM, "-f", "100M", "-d", f"driver=file,path={cap}"] + args + [str(out)])
    got = np.fromfile(out, dtype=np.int16)
    p = fm.derive_params(**kw).params
    want = port.fm_run(_oracle_params(p), x, CHUNK16)
    assert got.size == want.size
    assert np.array_equal(got, want)


def test_rx_fm_level_printing(tmp_path, port):
    # -L N: every N chunks print mean / max / max-of-max of the chunk rms and the squelch level (src/rtl_fm.c:792-806)
    loud = synth.cfg2_iq(3 * 131072, seed=34)
    quiet = synth.fm_iq(4 * 131072, fs=2.4e6, deviation_hz=75e3, tones=[(1000.0, 1.0)], amplitude=900.0, noise_lsb=2, seed=35)
    x = np.concatenate([loud, quiet])
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    out = tmp_path / "out.raw"
    r = _run([RX_FM, "-f", "100M", "-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k", "-L", "2",
              "-d", f"driver=file,path={cap}", str(out)])
    p = fm.derive_params(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9).params
    lv = port.fm_levels(_oracle_params(p), x, CHUNK16)
    want_lines, no, lsum, lmax, lmaxmax = [], 1, 0.0, 0, 0
    for sr in lv:
        no -= 1
        lsum += int(sr); lmax = max(lmax, int(sr)); lmaxmax = max(lmaxmax, int(sr))
        if no == 0:
            no = 2
            want_lines.append("%f, %d, %d, %d" % (lsum / 2, lmax, lmaxmax, 0))
            lmax, lsum = 0, 0.0
    got_lines = [ln for ln in r.stderr.decode().splitlines() if ln.count(",") == 3 and ln[0].isdigit()]
    assert len(want_lines) >= 3
    assert got_lines == want_lines
    # and the PCM is the same as without -L
    want = port.fm_run(_oracle_params(p), x, CHUNK16)
    assert np.array_equal(np.fromfile(out, dtype=np.int16), want)


def test_rx_fm_wav_header_and_squelch_zero(tmp_path, port):
    loud = synth.cfg2_iq(3 * 131072, seed=32)
    quiet = synth.fm_iq(5 * 131072, fs=2.4e6, deviation_hz=75e3, tones=[(1000.0, 1.0)], amplitude=40.0, noise_lsb=2, seed=33)
    x = np.concatenate([loud, quiet])
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    out = tmp_path / "out.wav"
    _run([RX_FM, "-f", "100M", "-M", "fm", "-s", "170k", "-A", "fast", "-r", "32k", "-l", "40", "-t", "1", "-E", "zero", "-E", "wav",
          "-d", f"driver=file,path={cap}", str(out)])
    raw = np.fromfile(out, dtype=np.uint8)
    hdr = raw[:44].tobytes()
    assert hdr[:4] == b"RIFF" and hdr[8:16] == b"WAVEfmt " and hdr[36:40] == b"data"
    assert int.from_bytes(hdr[24:28], "little") == 32000 and int.from_bytes(hdr[28:32], "little") == 64000
    got = raw[44:].view(np.int16)
    d = fm.derive_params(rate_s=170000, custom_atan=1, rate_r=32000, squelch_level=40)
    want, lens, hits = port.fm_run(_oracle_params(d.params), x, CHUNK16, return_chunks=True)
    # demod thread: squelch active (hits > conseq_squelch) with -E zero writes zeros (src/rtl_fm.c:928-941)
    pos = 0
    for n, h in zip(lens, hits):
        if h > 1:
            want[pos:pos + n] = 0
        pos += n
    assert np.any(hits > 1), "test signal never closed the squelch"
    assert np.array_equal(got, want)


def _power_capture(plan, hop_bufs, n_pass):
    """What the shell reads: per hop a flush read of 16384 elements after every retune, then buf_len elements whose
    first buf_len int16 are the hop buffer."""
    parts = []
    rng = np.random.default_rng(5)
    for p in range(n_pass):
        for h in range(plan.n_hops):
            retune = plan.n_hops > 1 or p == 0
            if retune:
                parts.append(rng.integers(-50, 50, size=2 * 16384, dtype=np.int32).astype(np.int16))
            parts.append(hop_bufs[p, h])
            parts.append(rng.integers(-50, 50, size=plan.buf_len, dtype=np.int32).astype(np.int16))
    return np.concatenate(parts)


@pytest.mark.parametrize("freq,crop,win", [("100M:101M:1k", "0%", "hamming"), ("24M:60M:1k", "28.5%", "blackman")])
def test_rx_power_csv(tmp_path, port, freq, crop, win):
    n_pass = 3
    plan = power.plan_range(freq, float(crop.strip("%")) / 100.0)
    hb = synth.power_hops(n_pass, plan.n_hops, plan.buf_len, seed=71)
    cap = tmp_path / "cap.cs16"
    _power_capture(plan, hb, n_pass).tofile(cap)
    out = tmp_path / "out.csv"
    _run([RX_POWER, "-f", freq, "-c", crop, "-w", win, "-i", "1h", "-d", f"driver=file,path={cap}", str(out)],
         env={"RXB200_MAX_SWEEPS": str(n_pass), "RXB200_FIXED_TIME": "2026-01-01, 00:00:00"})
    got = open(out).read()
    pp = oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len)
    avg, smp = port.power_scan(pp, power.window_table(win, 1 << plan.bin_e), hb, n_pass, plan.n_hops)
    want = power.csv_rows(plan, avg, smp, "2026-01-01, 00:00:00")
    assert got == want


def test_rx_power_csv_on_two_gpus(tmp_path, port):
    """RXB200_GPUS=2: hops sharded over two GPUs, one NCCL all-gather before the report; the CSV bytes are those of
    the single-GPU run (and of the oracle)."""
    from rx_tools_b200 import _lib
    if int(_lib.lib().rxb200_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    freq, crop, win, n_pass = "24M:60M:1k", "28.5%", "hamming", 2
    plan = power.plan_range(freq, 0.285)
    hb = synth.power_hops(n_pass, plan.n_hops, plan.buf_len, seed=72)
    cap = tmp_path / "cap.cs16"
    _power_capture(plan, hb, n_pass).tofile(cap)
    outs = []
    for g in ("1", "2"):
        out = tmp_path / f"out{g}.csv"
        _run([RX_POWER, "-f", freq, "-c", crop, "-w", win, "-i", "1h", "-d", f"driver=file,path={cap}", str(out)],
             env={"RXB200_MAX_SWEEPS": str(n_pass), "RXB200_FIXED_TIME": "2026-01-01, 00:00:00", "RXB200_GPUS": g})
        outs.append(open(out).read())
    pp = oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len)
    avg, smp = port.power_scan(pp, power.window_table(win, 1 << plan.bin_e), hb, n_pass, plan.n_hops)
    want = power.csv_rows(plan, avg, smp, "2026-01-01, 00:00:00")
    assert outs[0] == want
    assert outs[1] == want
