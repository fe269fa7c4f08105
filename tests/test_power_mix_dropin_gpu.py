"""The rx_power shell in capture mode (RXB200_CAPTURE_RATE): one tune, one flush read, then passes of M * buf_len int16
gathered from reads of whatever length the replay device returns (reads= caps that do not divide a pass).  The CSV bytes
must equal csv_rows of the port's result on the model's hop buffers; a rate cap below what the span needs exits 1
before anything is read."""
import os
import subprocess

import numpy as np
import pytest

import power_mix as pm
from rx_tools_b200 import power

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RX_POWER = os.path.join(ROOT, "host", "rx_power_b200")
TSTR = "2026-01-01, 00:00:00"
FLUSH = 16384                        # BUFFER_DUMP: complex elements of the flush read after the one tune


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(cmd, env):
    e = dict(os.environ)
    e.update(env)
    return subprocess.run(cmd, capture_output=True, env=e, timeout=300)


@pytest.mark.parametrize("name,crop,win,reads", [("fm_band", "0%", "hamming", (5000, 12345, 777)),
                                                  ("hf_crop285", "28.5%", "blackman", (40000, 3, 9999))])
def test_capture_mode_csv(tmp_path, port, name, crop, win, reads):
    c = pm.SHAPES[name]
    plan, _, R, offs, dd = pm.shape(name)
    window = power.window_table(win, 1 << plan.bin_e)
    n_pass = 3
    x = pm.capture(n_pass * dd[0] * plan.buf_len // 2, R, offs, 4242 + len(name))
    flush_n = min(FLUSH, reads[0])                 # the flush read is capped like every other read
    rng = np.random.default_rng(9)
    junk = rng.integers(-30000, 30000, size=2 * flush_n, dtype=np.int32).astype(np.int16)
    tail = rng.integers(-30000, 30000, size=2 * 1001, dtype=np.int32).astype(np.int16)   # a partial pass: discarded
    cap = tmp_path / "cap.cs16"
    np.concatenate([junk, x, tail]).tofile(cap)
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", c["freq"], "-c", crop, "-w", win, "-i", "1h",
              "-d", f"driver=file,path={cap},reads={':'.join(map(str, reads))}", str(out)],
             {"RXB200_CAPTURE_RATE": "40000000", "RXB200_MAX_SWEEPS": str(n_pass), "RXB200_FIXED_TIME": TSTR})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert f"Capture mode: {R} Hz centred at" in r.stderr.decode()
    hb = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    avg, smp = pm.port_result(port, plan, window, hb)
    assert open(out).read() == power.csv_rows(plan, avg, smp, TSTR)


def test_capture_mode_stream_running_dry_reports_whole_passes(tmp_path, port):
    """Without a sweep limit the shell reads until the stream runs dry, reports the whole passes and exits."""
    plan, _, R, offs, dd = pm.shape("peak_hold")
    c = pm.SHAPES["peak_hold"]
    window = power.window_table("rectangle", 1 << plan.bin_e)
    x = pm.capture(2 * dd[0] * plan.buf_len // 2, R, offs, 77)
    cap = tmp_path / "cap.cs16"
    np.concatenate([np.zeros(2 * 7000, np.int16), x, x[:2 * 5000]]).tofile(cap)      # the flush read takes 7000
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", c["freq"], "-c", "10%", "-P", "-i", "1h", "-d", f"driver=file,path={cap},reads=7000",
              str(out)], {"RXB200_CAPTURE_RATE": "20000000", "RXB200_FIXED_TIME": TSTR})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    hb = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    avg, smp = pm.port_result(port, plan, window, hb)
    assert open(out).read() == power.csv_rows(plan, avg, smp, TSTR)


def test_capture_rate_below_the_span_exits_before_reading(tmp_path):
    cap = tmp_path / "cap.cs16"
    np.zeros(1024, np.int16).tofile(cap)
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", "88M:108M:10k", "-d", f"driver=file,path={cap}", str(out)],
             {"RXB200_CAPTURE_RATE": "19999999"})
    assert r.returncode == 1
    assert "needs a capture rate of 20000000 Hz" in r.stderr.decode()
    assert not out.exists()
    r = _run([RX_POWER, "-f", "88M:108M:10k", "-d", f"driver=file,path={cap}", str(out)],
             {"RXB200_CAPTURE_RATE": "40000000", "RXB200_GPUS": "2"})
    assert r.returncode == 1 and not out.exists()
