"""The rx_fm shell in capture mode with RXB200_CAPTURE_STAGES=2 on the replay device: the plan is
rxb200_fm_plan_capture_two_stage's and the handle a two-stage mixing handle.  Every channel's file must equal the port
run on that channel's decimated stream (the two-stage model) one block at a time, with the squelch rule and -E zero
applied per block, and read lengths do not change the files."""
import os
import subprocess

import pytest

import fm_capture as fcp
import fm_two_stage as fts
from rx_tools_b200 import fm, power

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")

# name -> (-f values, other arguments, derive_params keywords, (capture samples, per-channel stop sample or None))
SHAPES = {
    # three NBFM channels 2 MHz apart: c = 1.008 Msps, M = 5 -> M' = 8, K = 4; the last block is partial
    "nbfm_3ch": (["162M", "164M", "166M"], [], {}, (2 * 8 * fcp.CHUNK + 70001, None)),
    # squelch: channels that fall quiet at different blocks, -t 0
    "squelch_3ch": (["100M:104M:2M"], ["-l", "60", "-t", "0"], dict(squelch_level=60),
                    (3 * 8 * fcp.CHUNK + 5000, [int(1.3 * 8 * fcp.CHUNK), int(2.6 * 8 * fcp.CHUNK), None])),
    # fm2b's command line (P = 3): 2.4 Msps chain, M = 5 -> M' = 8 at 19.2 Msps
    "fm2b_f9": (["96M", "100M", "104M"], ["-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k"],
                dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9), (8 * fcp.CHUNK + 999, None)),
}


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _case(name, seed=0):
    fvals, args, kw, (n, stops) = SHAPES[name]
    der = fm.derive_params(offset_tuning=1, **kw)
    freqs = fcp.freqs_of(fvals)
    tuned = fcp.tuned_of(freqs, der, wbfm=bool(kw.get("wbfm")))
    pl, offs = fm.plan_capture_two_stage(tuned, der.capture_rate, 10**10)
    x = fcp.capture(n, pl.capture_rate, offs, 2100 + seed + len(name), stops,
                    deviation=75000.0 if kw.get("wbfm") else 2500.0)
    argv = [a for v in fvals for a in ("-f", v)] + args
    return argv, der.params, freqs, pl, offs, x


def _stages(pl):
    return ((pl.coarse_decim, power.ddc_lowpass(pl.coarse_decim, pl.coarse_taps, 15), pl.coarse_shift),
            (pl.fine_decim, power.ddc_lowpass(pl.fine_decim, pl.fine_taps, 15), pl.fine_shift))


def _run(tmp_path, argv, x, reads, tag="out"):
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    out = tmp_path / tag
    r = subprocess.run([RX_FM] + argv + ["-d", f"driver=file,path={cap},reads={reads}", str(out)], capture_output=True,
                       timeout=600, env=dict(os.environ, RXB200_CAPTURE_RATE="40000000", RXB200_CAPTURE_STAGES="2"))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return out, r.stderr.decode()


@pytest.mark.parametrize("name,zero", [("nbfm_3ch", False), ("squelch_3ch", False), ("squelch_3ch", True),
                                       ("fm2b_f9", False)])
def test_shape_files_equal_the_port(tmp_path, port, name, zero):
    argv, p, freqs, pl, offs, x = _case(name)
    argv = argv + (["-E", "zero"] if zero else [])
    out, err = _run(tmp_path, argv, x, "5000:12345:777")
    M = pl.coarse_decim * pl.fine_decim
    assert (f"Capture mode: {pl.capture_rate} Hz centred at {pl.centre_hz} Hz in two stages: {pl.n_bins} bins, "
            f"coarse decimation {pl.coarse_decim} with {pl.coarse_taps} taps, fine decimation 4 with 129 taps, "
            f"{len(freqs)} channels") in err
    lens = fcp.chain_reads(fcp.blocks(x.size // 2, M, fcp.min_chunk(p)), M)
    coarse, fine = _stages(pl)
    decs = fts.two_stage_model(x, pl.capture_rate, pl.n_bins, offs, coarse, fine)
    conseq = int(argv[argv.index("-t") + 1]) if "-t" in argv else 10
    n_quiet = 0
    for k, f in enumerate(freqs):
        pcm, rl, hits = fcp.port_channel(port, p, decs[k], lens)
        want = fcp.squelched(pcm, rl, hits, conseq, p.squelch_level, zero).tobytes()
        got = open(f"{out}.{f}", "rb").read()
        assert got == want and (len(got) > 0 or p.squelch_level), (name, k)
        n_quiet += int(p.squelch_level and (hits > 0).any())
    if p.squelch_level:
        assert n_quiet == 2


def test_read_lengths_do_not_change_the_files(tmp_path):
    argv, p, freqs, pl, offs, x = _case("squelch_3ch", seed=3)
    a, _ = _run(tmp_path, argv, x, "5000:12345:777", tag="a")
    b, _ = _run(tmp_path, argv, x, "131072", tag="b")
    fa = [open(f"{a}.{f}", "rb").read() for f in freqs]
    fb = [open(f"{b}.{f}", "rb").read() for f in freqs]
    assert fa == fb and all(len(f) > 0 for f in fa)
