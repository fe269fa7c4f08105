"""The drop-in shells with RXB200_DEVICE_FORMAT on replay files in the device's own CS8, CU8 or CS12 format, read in
ragged lengths.  Each shell's files (rx_power: its CSV under RXB200_FIXED_TIME) must equal byte for byte those of the
same shell without the variable on the file's CS16 widening (tests/device_format.py), in capture mode and rx_power's
tile mode, with and without RXB200_DEVICE_RATE on a device that runs only at that rate.  And plain rx_sdr records CS8
and CU8 as read, as the reference's rx_sdr does with the same bytes."""
import os
import subprocess

import pytest

import device_format as df

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOST = os.path.join(ROOT, "host")
READS = "5000:12345:777:3"
TSTR = "2026-01-01, 00:00:00"
NOAA_F = [f"{162_400 + 25 * k}k" for k in range(7)]
SDR4 = [100_000_000, 100_025_000, 100_500_000, 100_950_000]

CASES = {
    # name: (shell, argv without -d and the output, variables, device samples, device rate)
    "rx_fm": ("rx_fm_b200", ["-M", "fm", "-s", "24k"] + [a for v in NOAA_F for a in ("-f", v)],
              {"RXB200_CAPTURE_RATE": "100000000"}, 700_001, 2_500_000),
    "rx_fm_raster": ("rx_fm_b200", ["-M", "fm", "-s", "24k"] + [a for v in NOAA_F for a in ("-f", v)],
                     {"RXB200_CAPTURE_RATE": "100000000", "RXB200_CAPTURE_STAGES": "raster"}, 700_001, 2_500_000),
    "rx_sdr": ("rx_sdr_b200", sum((["-f", str(f)] for f in SDR4), []) + ["-s", "250k", "-F", "CS16"],
               {"RXB200_CAPTURE_RATE": "100000000"}, 300_007, 2_400_000),
    "rx_sdr_two_stage_cf32": ("rx_sdr_b200", sum((["-f", str(f)] for f in SDR4), []) + ["-s", "250k", "-F", "CF32"],
                              {"RXB200_CAPTURE_RATE": "100000000", "RXB200_CAPTURE_STAGES": "2"}, 300_007, 2_400_000),
    "rx_power": ("rx_power_b200", ["-f", "88M:108M:10k", "-i", "1h"],
                 {"RXB200_CAPTURE_RATE": "40000000", "RXB200_MAX_SWEEPS": "2", "RXB200_FIXED_TIME": TSTR},
                 500_000, 25_000_000),
    "rx_power_tiles": ("rx_power_b200", ["-f", "100M:110M:1M", "-w", "rectangle", "-i", "1h"],
                       {"RXB200_TILE_RATE": "10000000", "RXB200_MAX_SWEEPS": "2", "RXB200_FIXED_TIME": TSTR},
                       2_000_000, 3_200_000),
}


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", HOST, "-s"], check=True)


def _run(argv, env):
    e = {k: v for k, v in os.environ.items() if not k.startswith("RXB200_")}
    e.update(env)
    r = subprocess.run(argv, capture_output=True, timeout=900, env=e)
    assert r.returncode == 0, r.stderr.decode()[-3000:]
    return r.stderr.decode()


def _outputs(tmp_path, power, tag):
    if power:
        return [(tmp_path / tag).read_bytes()]
    return [p.read_bytes() for p in sorted(tmp_path.glob(f"{tag}.*"))]


@pytest.mark.parametrize("rate", [False, True], ids=["capture_rate", "device_rate"])
@pytest.mark.parametrize("fmt", list(df.FORMATS))
@pytest.mark.parametrize("name", sorted(CASES))
def test_shell_files_equal_the_widened_cs16_run(tmp_path, name, fmt, rate):
    exe, argv, env, n_dev, R_dev = CASES[name]
    narrow, cs16 = df.write_replay(str(tmp_path), fmt, df.narrow_stream(n_dev, fmt, 60 + len(name)))
    keys = f"reads={READS}" + (f",rate={R_dev}" if rate else "")
    if rate:
        env = dict(env, RXB200_DEVICE_RATE=str(R_dev))
    power = exe == "rx_power_b200"
    want_err = _run([os.path.join(HOST, exe), "-d", f"driver=file,path={cs16},{keys}"] + argv + [str(tmp_path / "want")],
                    env)
    want = _outputs(tmp_path, power, "want")
    assert want and all(len(w) > 0 for w in want)
    got_err = _run([os.path.join(HOST, exe), "-d", f"driver=file,path={narrow},{keys}"] + argv +
                   [str(tmp_path / "got")], dict(env, RXB200_DEVICE_FORMAT=fmt))
    assert _outputs(tmp_path, power, "got") == want, (name, fmt, rate)
    # the banners are the same
    assert got_err.replace(narrow, "").replace(str(tmp_path / "got"), "") == \
        want_err.replace(cs16, "").replace(str(tmp_path / "want"), "")


def _ref_written_as_read(oracle, b, fmt, n, workdir):
    """The reference rx_sdr's bytes for -I fmt -F fmt -n n over bytes b.  A reference linked against a replay device
    that predates its 8-bit streams cannot open b as fmt; its written-as-read path (src/rtl_sdr.c, input format equal
    to the output format: the read buffer goes to the file unchanged) is then run on the same bytes as n / 2 CS16
    elements, which is the same path over the same bytes."""
    try:
        return oracle.ref_rx_sdr(b, fmt, fmt, n, workdir=workdir)
    except RuntimeError as e:
        if "setupStream failed" not in str(e):
            raise
    assert n % 2 == 0 and b.size > 2 * n
    return oracle.ref_rx_sdr(b, "CS16", "CS16", n // 2, block=8192, workdir=workdir)


@pytest.mark.parametrize("fmt", ["CS8", "CU8"])
def test_plain_rx_sdr_written_as_read_equals_the_reference(tmp_path, fmt):
    """Plain rx_sdr -I fmt -F fmt on the replay device writes the bytes it reads, cut at -n: the file's first 2 n bytes,
    as the reference's rx_sdr writes them."""
    import oracle
    n = 70_000
    b = df.narrow_stream(n + 20_000, fmt, 70)
    cap = tmp_path / "cap.bin"
    b.tofile(cap)
    out = tmp_path / "out.bin"
    _run([os.path.join(HOST, "rx_sdr_b200"), "-d", f"driver=file,path={cap}", "-I", fmt, "-F", fmt, "-n", str(n),
          "-b", "16384", str(out)], {})
    assert out.read_bytes() == b[:2 * n].tobytes()
    if not os.path.exists(oracle.REF_SDR_BIN):
        pytest.skip("oracle/_ref/rx_sdr_ref not built")
    assert out.read_bytes() == _ref_written_as_read(oracle, b, fmt, n, str(tmp_path))
