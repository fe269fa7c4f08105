"""The drop-in shells with RXB200_DEVICE_RATE on captures synthesised at the device's rate R_dev and replayed by a device
that runs only at that rate (rate=R_dev) in reads of ragged lengths.

Bytes.  Each shell's files must equal what it writes, or the library handle it drives writes, on the same capture
resampled to the plan's rate R by the resampler (an rxb200_resample handle, whose bytes tests/test_resample_gpu.py pins
to the model in tests/resample.py):
  - rx_fm, whose plans on these channel sets do not change with the guard band: the shell without the variable on the
    resampled capture (the existing drop-in tests pin that run to the port), single stage, two stages and raster,
    with squelch and -E zero;
  - rx_sdr: the single-stage and raster handles at the _at plan, CS16 and CF32;
  - rx_power: capture mode's and tile mode's CSV against a power mixing handle at the _at plan fed the resampled
    passes, or each tile's resampled burst with its first E outputs dropped.
The read lengths never change the files.

Physics, the point of the feature: a tone at f_k + delta_k for each rx_sdr channel must come out at +delta_k, within
one FFT bin; the same replay without the variable (the shell asks for R, the device runs at R_dev) puts it
where the rate error moves it."""
import os
import subprocess

import numpy as np
import pytest

import device_rate as dr
import resample as rsm
import sdr_mix as sm
from rx_tools_b200 import fm, power, sdr
from rx_tools_b200 import resample as rs

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
RX_SDR = os.path.join(ROOT, "host", "rx_sdr_b200")
RX_POWER = os.path.join(ROOT, "host", "rx_power_b200")
READS = ("5000:12345:777", "40000:3:50001")
TSTR = "2026-01-01, 00:00:00"
FLUSH = 16384                        # rx_power's flush read after a retune (BUFFER_DUMP)
VARS = ("RXB200_CAPTURE_RATE", "RXB200_TILE_RATE", "RXB200_DEVICE_RATE", "RXB200_CAPTURE_STAGES", "RXB200_GPUS")


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(argv, env):
    e = {k: v for k, v in os.environ.items() if k not in VARS}
    e.update(env)
    r = subprocess.run(argv, capture_output=True, timeout=900, env=e)
    assert r.returncode == 0, r.stderr.decode()[-3000:]
    return r.stderr.decode()


def _noise(n_complex, seed, amp=12000):
    return np.random.default_rng(seed).integers(-amp, amp + 1, size=2 * n_complex, dtype=np.int32).astype(np.int16)


def _tones(n_complex, R_dev, freqs, seed, amp=3000.0, noise=200):
    """Complex tones at freqs (Hz, relative to the centre) at the device rate, with a little noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_complex, dtype=np.float64)
    z = sum(amp * np.exp(2j * np.pi * (f / R_dev * t + rng.uniform())) for f in freqs)
    x = np.empty(2 * n_complex, np.int64)
    x[0::2], x[1::2] = np.rint(z.real), np.rint(z.imag)
    x += rng.integers(-noise, noise + 1, size=x.size)
    return np.clip(x, -32768, 32767).astype(np.int16)


def _resampled(x, R_dev, R, span):
    r = rs.plan_resample(R_dev, R, span)
    assert r.up <= r.down and (r.up, r.down) != (1, 1)
    with rs.Resampler(r.up, r.down, rs.lowpass(r.up, r.down, r.taps_per_phase)) as h:
        return h.process(x), r


def _banner(r, R_dev, R):
    return f"Device rate: {R_dev} Hz, resampled by {r.up}/{r.down} with {r.taps_per_phase} taps per phase to {R} Hz"


# ---------------------------------------------------------------- rx_fm
NOAA_F = [f"{162_400 + 25 * k}k" for k in range(7)]
FM30_F = [f"{98_000 + 800 * k}k" for k in range(6)]       # wbfm 6 stations 800 kHz apart: two stages at M' = 8
FM_CASES = {
    "noaa_2.4M": (NOAA_F, ["-M", "fm", "-s", "24k"], 2_400_000, None),
    "noaa_2.5M_squelch": (NOAA_F, ["-M", "fm", "-s", "24k", "-l", "200", "-t", "0"], 2_500_000, None),
    "noaa_2.4M_zero": (NOAA_F, ["-M", "fm", "-s", "24k", "-l", "200", "-t", "0", "-E", "zero"], 2_400_000, None),
    "noaa_2.4M_raster": (NOAA_F, ["-M", "fm", "-s", "24k"], 2_400_000, "raster"),
    "fm30_two_stage": (FM30_F, ["-M", "wbfm"], 30_720_000, "2"),
}


@pytest.mark.parametrize("name", sorted(FM_CASES))
def test_rx_fm_files_equal_the_shell_on_the_resampled_capture(tmp_path, name):
    fvals, opts, R_dev, stages = FM_CASES[name]
    freqs = [int(float(v[:-1]) * 1000) for v in fvals]
    der = fm.derive_params(offset_tuning=1, wbfm=int("wbfm" in opts), rate_s=0 if "wbfm" in opts else 24000)
    tuned = [f + (16000 if "wbfm" in opts else 0) for f in freqs]
    planner = fm.plan_capture_two_stage if stages == "2" else fm.plan_capture_raster if stages else fm.plan_capture
    p_at, _ = planner(tuned, der.capture_rate, 10**10, device_rate=R_dev)
    p0, _ = planner(tuned, der.capture_rate, 10**10)
    assert p_at == p0                                      # the guard band fits these plans' slack
    R = p0.capture_rate
    dec = p0.coarse_decim * p0.fine_decim if stages == "2" else p0.decim
    span = 2 * max(abs(t - p0.centre_hz) for t in tuned) + der.capture_rate
    r = rs.plan_resample(R_dev, R, span)
    n_dev = rs.in_len(r.up, r.down, 0, 2 * dec * 131072 + 50_001)    # two blocks and a partial one
    if "-l" in opts:                                    # tones on every other channel: the rest squelch
        x = _tones(n_dev, R_dev, [t - p0.centre_hz + 500 for t in tuned][::2], 5, amp=6000.0, noise=20)
    else:
        x = _noise(n_dev, 7 + len(name))
    y, r = _resampled(x, R_dev, R, span)
    env = {"RXB200_CAPTURE_RATE": "100000000"}
    if stages:
        env["RXB200_CAPTURE_STAGES"] = stages
    argv = opts + [a for v in fvals for a in ("-f", v)]
    (tmp_path / "cap_r.cs16").write_bytes(y.tobytes())
    _run([RX_FM, "-d", f"driver=file,path={tmp_path / 'cap_r.cs16'},reads={READS[0]}"] + argv + [str(tmp_path / "want")],
         env)
    want = [(tmp_path / f"want.{f}").read_bytes() for f in freqs]
    assert sum(len(w) for w in want) > 0
    (tmp_path / "cap.cs16").write_bytes(x.tobytes())
    for reads in READS:
        err = _run([RX_FM, "-d", f"driver=file,path={tmp_path / 'cap.cs16'},reads={reads},rate={R_dev}"] + argv +
                   [str(tmp_path / "got")], dict(env, RXB200_DEVICE_RATE=str(R_dev)))
        assert _banner(r, R_dev, R) in err
        assert [(tmp_path / f"got.{f}").read_bytes() for f in freqs] == want, reads


# ---------------------------------------------------------------- rx_sdr
FM100 = dr.FM100


def _sdr_expected(x, R_dev, tuned, s, raster, fout):
    if raster:
        pl, bins = fm.plan_capture_raster(tuned, s, 10**10, device_rate=R_dev)
        taps = power.ddc_lowpass(pl.decim, pl.n_taps, 15)
        h = sdr.SdrMix(ddc=(pl.decim, taps, pl.shift), raster=(pl.n_bins, bins))
    else:
        pl, offs = sdr.plan_sdr_capture(tuned, s, 10**10, device_rate=R_dev)
        h = sdr.SdrMix(pl.capture_rate, offs, (pl.decim, power.ddc_lowpass(pl.decim, pl.n_taps, 15), 15))
    span = 2 * max(abs(t - pl.centre_hz) for t in tuned) + s
    y, r = _resampled(x, R_dev, pl.capture_rate, span)
    out = h.process(y)
    h.close()
    return pl, r, [sm.convert(out[k], fout).tobytes() for k in range(len(tuned))]


SDR_CASES = {
    "sdr4_2.4M": (dr.SDR4, 2_400_000, False, 300_007),
    "fm100_raster_30.72M": (FM100, 30_720_000, True, 700_001),
}


@pytest.mark.parametrize("name", sorted(SDR_CASES))
@pytest.mark.parametrize("fout", ["CS16", "CF32"])
def test_rx_sdr_files_equal_the_handle_on_the_resampled_capture(tmp_path, name, fout):
    tuned, R_dev, raster, n_dev = SDR_CASES[name]
    x = _noise(n_dev, 11)
    pl, r, want = _sdr_expected(x, R_dev, tuned, 250_000, raster, fout)
    assert all(len(w) > 0 for w in want)
    (tmp_path / "cap.cs16").write_bytes(x.tobytes())
    env = {"RXB200_CAPTURE_RATE": "100000000", "RXB200_DEVICE_RATE": str(R_dev)}
    if raster:
        env["RXB200_CAPTURE_STAGES"] = "raster"
    argv = sum((["-f", str(f)] for f in tuned), []) + ["-s", "250k", "-F", fout]
    for reads in READS:
        err = _run([RX_SDR, "-d", f"driver=file,path={tmp_path / 'cap.cs16'},reads={reads},rate={R_dev}"] + argv +
                   [str(tmp_path / "out")], env)
        assert _banner(r, R_dev, pl.capture_rate) in err
        got = [(tmp_path / f"out.{f}").read_bytes() for f in tuned]
        assert got == want, reads


def _spectra(path, rate, tuned):
    """Each channel file's Hann-windowed magnitude spectrum, its frequencies (Hz at rate) and bin width."""
    out = []
    for f in tuned:
        z = np.fromfile(f"{path}.{f}", np.int16).astype(np.float64).reshape(-1, 2)
        z = z[len(z) // 8:]                                # past the filters' start
        c = z[:, 0] + 1j * z[:, 1]
        out.append((np.abs(np.fft.fft(c * np.hanning(c.size))), np.fft.fftfreq(c.size, 1.0 / rate), rate / c.size))
    return out


def _level_at(spec, freq):
    """The spectrum's largest value within one bin of freq, over its largest value anywhere: about 1 for a tone there,
    below 0.03 (the Hann window's sidelobes) for none."""
    S, fr, bin_hz = spec
    return float(S[np.abs(fr - freq) <= bin_hz].max() / S.max())


@pytest.mark.parametrize("R_dev", [2_400_000, 1_280_000])
def test_rx_sdr_tones_come_out_where_they_are(tmp_path, R_dev):
    """Tones at f_k + delta_k: at +delta_k with the resampler.  Without RXB200_DEVICE_RATE the shell takes the device's
    samples as rate R samples, and tone k comes out at (o_k + delta_k) R / R_dev - o_k instead; on the 1.28 M device
    that error (up to 11 kHz) stays inside the channel, so the test can see it."""
    tuned, s = dr.SDR4, 250_000
    pl, offs = sdr.plan_sdr_capture(tuned, s, 10**10, device_rate=R_dev)
    delta = [3_000, -7_000, 11_000, -2_000]
    x = _tones(600_000, R_dev, [o + d for o, d in zip(offs, delta)], 21)
    (tmp_path / "cap.cs16").write_bytes(x.tobytes())
    argv = sum((["-f", str(f)] for f in tuned), []) + ["-s", "250k", "-F", "CS16"]
    dev = f"driver=file,path={tmp_path / 'cap.cs16'},reads=7777,rate={R_dev}"
    _run([RX_SDR, "-d", dev] + argv + [str(tmp_path / "rs")],
         {"RXB200_CAPTURE_RATE": "100000000", "RXB200_DEVICE_RATE": str(R_dev)})
    # neighbouring channels overlap (25 kHz apart), so a channel also holds its neighbour's tone at the same level
    for spec, d in zip(_spectra(tmp_path / "rs", s, tuned), delta):
        assert _level_at(spec, d) > 0.5, d
    if R_dev != 1_280_000:
        return
    p0, offs0 = sdr.plan_sdr_capture(tuned, s, 10**10)
    assert p0.capture_rate == pl.capture_rate == 1_250_000
    _run([RX_SDR, "-d", dev] + argv + [str(tmp_path / "raw")], {"RXB200_CAPTURE_RATE": "100000000"})
    R = p0.capture_rate
    moved = 0
    for spec, d, o in zip(_spectra(tmp_path / "raw", s, tuned), delta, offs0):
        want = (o + d) * R / R_dev - o
        assert _level_at(spec, want) > 0.5, (d, want)
        moved += abs(want - d) > 4 * spec[2] and _level_at(spec, d) < 0.03
    assert moved >= 3


# ---------------------------------------------------------------- rx_power
def _power_handle(plan, R, offs, T, M, win):
    return power.PowerMix(plan, R, offs, (M, power.ddc_lowpass(M, T, 15), 15), win)


@pytest.mark.parametrize("reads", [(5000, 12345, 777), (40000, 3, 9999)])
def test_rx_power_capture_mode_csv(tmp_path, reads):
    freq, R_dev, n_pass = "88M:108M:10k", 30_720_000, 3
    plan = power.plan_range(freq)
    win = power.window_table("hamming", 1 << plan.bin_e)
    cp, offs = power.plan_capture(plan, 40_000_000, device_rate=R_dev)
    assert (cp.decim, cp.capture_rate) == (9, 22_500_000)
    span = 2 * max(abs(o) for o in offs) + plan.rate
    r = rs.plan_resample(R_dev, cp.capture_rate, span)
    pass_c = cp.decim * plan.buf_len // 2
    n_dev = rs.in_len(r.up, r.down, 0, n_pass * pass_c)
    x = _noise(n_dev, 31, 4000)
    y, _ = _resampled(x, R_dev, cp.capture_rate, span)
    assert y.size == 2 * n_pass * pass_c
    b = _power_handle(plan, cp.capture_rate, offs, cp.n_taps, cp.decim, win)
    b.accumulate(y)
    want = power.csv_rows(plan, *b.read(), TSTR)
    b.close()
    flush = _noise(min(FLUSH, reads[0]), 32)
    cap = tmp_path / "cap.cs16"
    np.concatenate([flush, x, _noise(1001, 33)]).tofile(cap)
    out = tmp_path / "out.csv"
    err = _run([RX_POWER, "-f", freq, "-w", "hamming", "-i", "1h", "-d",
                f"driver=file,path={cap},reads={':'.join(map(str, reads))},rate={R_dev}", str(out)],
               {"RXB200_CAPTURE_RATE": "40000000", "RXB200_DEVICE_RATE": str(R_dev),
                "RXB200_MAX_SWEEPS": str(n_pass), "RXB200_FIXED_TIME": TSTR})
    assert f"Capture mode: {cp.capture_rate} Hz centred at {cp.centre_hz} Hz, decimation 9" in err
    assert _banner(r, R_dev, cp.capture_rate) in err
    assert out.read_text() == want


@pytest.mark.parametrize("freq,cap_rate,R_dev,reads", [("100M:110M:1M", 10_000_000, 3_200_000, (5000, 12345, 777)),
                                                       ("100M:103M:1k", 10_000_000, 3_200_000, (40000, 3, 9999))])
def test_rx_power_tile_mode_csv(tmp_path, freq, cap_rate, R_dev, reads):
    plan = power.plan_range(freq)
    win = power.window_table("rectangle", 1 << plan.bin_e)
    tl, tiles, offs = power.plan_tiles(plan, cap_rate, device_rate=R_dev)
    assert tl.n_tiles > 1
    b = _power_handle(plan, tl.capture_rate, offs, tl.n_taps, tl.decim, win)
    span = 2 * max(abs(o) for o in offs) + plan.rate
    r = rs.plan_resample(R_dev, tl.capture_rate, span)
    h = rs.lowpass(r.up, r.down, r.taps_per_phase)
    E = rsm.ceil_div((r.taps_per_phase - 1) * r.up, r.down)
    n_dev = rs.in_len(r.up, r.down, 0, E + b.burst_int16(1) // 2)
    k, parts, seed = 0, [], 40
    n_sweeps = 2
    for _ in range(n_sweeps):
        for (hb, he, _) in tiles:
            got = 0
            fl = min(FLUSH, reads[k % len(reads)])             # the flush read after each retune takes one capped read
            k += 1
            parts.append(_noise(fl, seed)); seed += 1
            while got < n_dev:
                got += min(n_dev - got, reads[k % len(reads)])
                k += 1
            x = _noise(n_dev, seed, 4000); seed += 1
            parts.append(x)
            with rs.Resampler(r.up, r.down, h) as rr:
                b.accumulate_burst(hb, he, rr.process(x)[2 * E:])
    want = power.csv_rows(plan, *b.read(), TSTR)
    b.close()
    cap = tmp_path / "cap.cs16"
    np.concatenate(parts).tofile(cap)
    out = tmp_path / "out.csv"
    err = _run([RX_POWER, "-f", freq, "-w", "rectangle", "-i", "1h", "-d",
                f"driver=file,path={cap},reads={':'.join(map(str, reads))},rate={R_dev}", str(out)],
               {"RXB200_TILE_RATE": str(cap_rate), "RXB200_DEVICE_RATE": str(R_dev),
                "RXB200_MAX_SWEEPS": str(n_sweeps), "RXB200_FIXED_TIME": TSTR})
    assert f"Tile mode: {tl.n_tiles} tiles of up to {tl.hops_per_tile} hops, {tl.capture_rate} Hz" in err
    assert _banner(r, R_dev, tl.capture_rate) in err
    assert out.read_text() == want


# ---------------------------------------------------------------- the device reports another rate
def _shell_run(argv, env):
    e = {k: v for k, v in os.environ.items() if k not in VARS}
    e.update(env)
    return subprocess.run(argv, capture_output=True, timeout=900, env=e)


REPLAN = {
    # shell: (argv without -d and the output, capture variables, device samples, rate the device runs at, rate asked)
    "rx_fm": (RX_FM, ["-M", "fm", "-s", "24k"] + [a for v in NOAA_F for a in ("-f", v)],
              {"RXB200_CAPTURE_RATE": "100000000"}, 700_001, 2_500_000, 2_400_000),
    "rx_sdr": (RX_SDR, sum((["-f", str(f)] for f in dr.SDR4), []) + ["-s", "250k", "-F", "CS16"],
               {"RXB200_CAPTURE_RATE": "100000000"}, 300_007, 2_400_000, 2_500_000),
    "rx_power": (RX_POWER, ["-f", "88M:108M:10k", "-i", "1h"],
                 {"RXB200_CAPTURE_RATE": "40000000", "RXB200_MAX_SWEEPS": "2", "RXB200_FIXED_TIME": TSTR},
                 500_000, 25_000_000, 30_720_000),
}


def _outputs(tmp_path, shell, tag):
    if shell == "rx_power":
        return [(tmp_path / tag).read_bytes()]
    return [p.read_bytes() for p in sorted(tmp_path.glob(f"{tag}.*"))]


@pytest.mark.parametrize("shell", sorted(REPLAN))
def test_a_device_at_another_rate_is_planned_from_the_rate_it_reports(tmp_path, shell):
    """A device that runs at X when asked for Y: the shell plans and resamples from X, so its files equal those of the
    run that asked for X in the first place."""
    exe, argv, env, n_dev, X, Y = REPLAN[shell]
    cap = tmp_path / "cap.cs16"
    _noise(n_dev, 51, 4000).tofile(cap)
    dev = ["-d", f"driver=file,path={cap},reads=5000:12345:777,rate={X}"]
    r = _shell_run([exe] + dev + argv + [str(tmp_path / "want")], dict(env, RXB200_DEVICE_RATE=str(X)))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert "planning again" not in r.stderr.decode()
    want = _outputs(tmp_path, shell, "want")
    assert want and all(len(w) > 0 for w in want)
    r = _shell_run([exe] + dev + argv + [str(tmp_path / "got")], dict(env, RXB200_DEVICE_RATE=str(Y)))
    err = r.stderr.decode()
    assert r.returncode == 0, err[-2000:]
    assert f"The device reports {X} Hz, not RXB200_DEVICE_RATE={Y} Hz: planning again." in err
    assert f"Device rate: {X} Hz, resampled by" in err
    assert _outputs(tmp_path, shell, "got") == want


@pytest.mark.parametrize("shell", ["rx_fm", "rx_power"])
def test_a_reported_rate_that_is_not_a_rate_ends_the_run(tmp_path, shell):
    """A driver that does not report its rate returns 0; here the replay device reports one above 2^31 - 1.  Either way
    the shell exits 1 instead of taking the samples as the plan's rate."""
    exe, argv, env, n_dev, X, Y = REPLAN[shell]
    cap = tmp_path / "cap.cs16"
    _noise(n_dev, 52).tofile(cap)
    r = _shell_run([exe, "-d", f"driver=file,path={cap},rate=3000000000"] + argv + [str(tmp_path / "out")],
                   dict(env, RXB200_DEVICE_RATE=str(Y)))
    err = r.stderr.decode()
    assert r.returncode == 1 and "reports a sample rate of 3000000000 Hz" in err, err[-2000:]
    assert not [p for p in tmp_path.glob("out*") if p.stat().st_size > 0]


# ---------------------------------------------------------------- physics in rx_fm and rx_power
def test_rx_fm_nbfm_carriers_demodulate_to_zero(tmp_path):
    """An unmodulated carrier exactly on each NOAA channel: with the resampler every channel's PCM has a mean near zero.
    Without RXB200_DEVICE_RATE on the same 2.048 M device (the shell asks for R = 2.016 M) channel k sits
    o_k (R / R_dev - 1) off, up to 1.2 kHz, and the discriminator turns that offset into a clearly non-zero mean whose
    sign follows o_k."""
    R_dev = 2_048_000
    der = fm.derive_params(offset_tuning=1, rate_s=24000)
    freqs = [int(float(v[:-1]) * 1000) for v in NOAA_F]
    p, offs = fm.plan_capture(freqs, der.capture_rate, 10**10, device_rate=R_dev)
    assert (p.decim, p.capture_rate) == (2, 2_016_000) and fm.plan_capture(freqs, der.capture_rate, 10**10)[0] == p
    cap = tmp_path / "cap.cs16"
    _tones(600_000, R_dev, offs, 61, amp=3000.0, noise=20).tofile(cap)
    argv = [RX_FM, "-d", f"driver=file,path={cap},reads=7777,rate={R_dev}", "-M", "fm", "-s", "24k"]
    argv += [a for v in NOAA_F for a in ("-f", v)]

    def means(tag, env):
        _run(argv + [str(tmp_path / tag)], dict(env, RXB200_CAPTURE_RATE="100000000"))
        out = []
        for f in freqs:
            pcm = np.fromfile(f"{tmp_path / tag}.{f}", np.int16).astype(np.float64)
            assert pcm.size > 4000
            out.append(float(pcm[pcm.size // 4:].mean()))
        return out

    for m in means("rs", {"RXB200_DEVICE_RATE": str(R_dev)}):
        assert abs(m) < 60, m
    raw = means("raw", {})
    for m, o in zip(raw, offs):
        if o == 0:
            assert abs(m) < 60, m
        else:
            assert abs(m) > 200, (m, o)
    assert len({np.sign(m) * np.sign(o) for m, o in zip(raw, offs) if o}) == 1


def test_rx_power_tone_lands_in_its_bin(tmp_path):
    """A tone at 101.2191 MHz in a 88-108 MHz sweep taken from a 30.72 M device: the loudest bin of the CSV is within a
    bin and a half of it.  The tone is weak (amplitude 100): rx_power's fixed-point FFT, made for 8-bit samples, wraps
    on strong ones, in the reference as here."""
    freq, R_dev = "88M:108M:10k", 30_720_000
    plan = power.plan_range(freq)
    cp, _ = power.plan_capture(plan, 40_000_000, device_rate=R_dev)
    f_tone = 101_219_100
    cap = tmp_path / "cap.cs16"
    _tones(700_000, R_dev, [f_tone - cp.centre_hz], 71, amp=100.0, noise=10).tofile(cap)
    out = tmp_path / "out.csv"
    _run([RX_POWER, "-f", freq, "-i", "1h", "-d", f"driver=file,path={cap},rate={R_dev}", str(out)],
         {"RXB200_CAPTURE_RATE": "40000000", "RXB200_DEVICE_RATE": str(R_dev), "RXB200_MAX_SWEEPS": "2",
          "RXB200_FIXED_TIME": TSTR})
    best, best_f, step = -1e9, None, None
    for line in out.read_text().splitlines():
        v = [s.strip() for s in line.split(",")]
        low, step = int(v[2]), float(v[4])
        db = np.array([float(s) for s in v[6:-1]])          # the last value repeats the last bin
        j = int(np.argmax(db))
        if db[j] > best:
            best, best_f = db[j], low + j * step
    assert abs(best_f - f_tone) <= 1.5 * step, (best_f, f_tone, step)
