"""The rx_fm shell's capture mode on the CPU: the planner (rxb200_fm_plan_capture) against the rule restated in Python
over seeded -f sets, its refusals, the block rule, the port against the unmodified reference on every channel of every
named command line, the golden hashes tests/golden/fm_capture_golden.json records, and the shell's refusals, which
exit 1 before the device is opened and create no file."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_capture as fcp
from rx_tools_b200 import _lib, fm

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "fm_capture_golden.json")
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")


def _draws():
    """About 200 seeded command lines: (-f values, derive keywords, -E edge)."""
    rng = np.random.default_rng(2026)
    kinds = [({}, False), (dict(mode=fm.MODE_AM), False), (dict(wbfm=1), False), ({}, True), (dict(wbfm=1), True),
             (dict(rate_s=170000, use_F=1, comp_fir_size=9), False)]
    out = []
    for i in range(200):
        kw, edge = kinds[i % len(kinds)]
        r = i % 5
        base = int(rng.integers(24_000_000, 1_700_000_000))
        if r == 0:                                         # an NBFM raster
            step = int(rng.choice([6250, 12500, 25000]))
            vals = [str(base + step * int(k)) for k in sorted(rng.choice(40, size=int(rng.integers(2, 8)), replace=False))]
        elif r == 1:                                       # arbitrary Hz
            vals = [str(base + int(v)) for v in rng.choice(3_000_000, size=int(rng.integers(2, 6)), replace=False)]
        elif r == 2:                                       # a:b:step range
            step = int(rng.choice([25000, 100000, 1_100_000]))
            vals = [f"{base}:{base + step * int(rng.integers(1, 20))}:{step}"]
        elif r == 3:                                       # one channel
            vals = [str(base)]
        else:                                              # scaled values
            vals = [f"{base / 1e6:.4f}M", f"{(base + 250_000) / 1e6:.4f}M", f"{(base - 37_500) / 1e3:.1f}k"]
        out.append((vals, kw, edge))
    return out


def test_planner_equals_the_rule():
    n_plans = n_caps = 0
    for vals, kw, edge in _draws():
        der = fm.derive_params(offset_tuning=1, **kw)
        freqs = fcp.freqs_of(vals)
        if len(set(freqs)) < len(freqs):
            continue
        t = fcp.tuned_of(freqs, der, wbfm=bool(kw.get("wbfm")), edge=edge)
        want = fcp.plan_rule(t, der.capture_rate, 10**12)
        if isinstance(want, str):
            with pytest.raises(_lib.Rxb200Error) as e:
                fm.plan_capture(t, der.capture_rate, 10**12)
            assert e.value.code == (_lib.EINVAL if want == "rate" else _lib.EUNSUPPORTED), (vals, kw)
            continue
        fc, M, R, T, offs = want
        pl, got = fm.plan_capture(t, der.capture_rate, 10**12)
        assert (pl.centre_hz, pl.decim, pl.capture_rate, pl.n_taps, got) == (fc, M, R, T, offs), (vals, kw, edge)
        n_plans += 1
        # the cap at R takes the plan, at R - 1 refuses it with the rate in the message
        assert fm.plan_capture(t, der.capture_rate, R)[0] == pl
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.plan_capture(t, der.capture_rate, R - 1)
        assert e.value.code == _lib.EINVAL and f"need a capture rate of {R} Hz" in str(e.value)
        n_caps += 1
    assert n_plans >= 150 and n_caps == n_plans


def test_named_plans():
    der = fm.derive_params(offset_tuning=1)
    assert der.capture_rate == 1_008_000
    pl, offs = fm.plan_capture([162_400_000 + 25_000 * k for k in range(7)], der.capture_rate, 40_000_000)
    assert (pl.centre_hz, pl.decim, pl.capture_rate, pl.n_taps) == (162_475_000, 2, 2_016_000, 65)
    assert offs == [-75_000 + 25_000 * k for k in range(7)]
    p, freqs, pl, offs, taps = fcp.plan_of(*fcp.WBFM19[:3])
    assert len(freqs) == 19 and freqs[-1] == 107_900_000
    assert (pl.decim, pl.capture_rate, pl.n_taps) == (21, 21_420_000, 673) and taps.sum() == 1 << 15
    pl, offs = fm.plan_capture([433_920_000], der.capture_rate, 40_000_000)     # one channel: at fc, M = 1
    assert (pl.centre_hz, pl.decim, pl.capture_rate, pl.n_taps, offs) == (433_920_000, 1, 1_008_000, 33, [0])


def test_planner_refusals():
    c = 1_008_000
    for t, cap in (([], 10**9), ([100_000_000], 0), ([-5], 10**9), ([1 << 61], 10**9), ([0, 2**31], 10**12)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.plan_capture(t, c, cap)
        assert e.value.code == _lib.EINVAL, t
    assert fm.plan_capture([100_000_000, 100_000_000 + 127 * c], c, 10**10)[0].decim == 255   # M = 255 fits
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture([100_000_000, 100_000_000 + 128 * c], c, 10**10)                    # M = 257
    assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:                 # offsets of 1 Hz: period R > 2^20
        fm.plan_capture([100_000_000, 100_000_001], c, 10**9)
    assert e.value.code == _lib.EUNSUPPORTED and "2^20" in str(e.value)
    assert fcp.plan_rule([100_000_000, 100_000_001], c, 10**9) == "period"
    L = _lib.lib()
    assert L.rxb200_fm_plan_capture(None, 1, c, 10**9, None, None) == _lib.EINVAL
    assert fm.plan_capture([5, 5], c, 10**9)[1] == [0, 0]       # equal frequencies: g = 0, fc = tmin
    with pytest.raises(_lib.Rxb200Error):
        fm.plan_capture([5], 0, 10**9)


def test_block_rule():
    M, B = 3, 3 * fcp.CHUNK
    assert fcp.blocks(2 * B, M, 2) == [B, B]
    assert fcp.blocks(2 * B + 2, M, 2) == [B, B]               # decimates to 0 samples
    assert fcp.blocks(2 * B + 3, M, 2) == [B, B, 3]
    assert fcp.blocks(B + 47, M, 32) == [B]                    # 15 samples: 30 int16 < 32, dropped
    assert fcp.blocks(B + 48, M, 32) == [B, 48]                # 16 samples: handed on
    assert fcp.chain_reads([B, B, 48], M) == [2 * fcp.CHUNK, 2 * fcp.CHUNK, 32]
    p = fac.P(mode=0, downsample=8, downsample_passes=3)
    assert fcp.min_chunk(p) == 16
    assert fcp.min_chunk(fac.with_(fac.FM24K_LUT, squelch_level=5)) == 84 and fcp.min_chunk(fac.FM24K_LUT) == 2


def test_shapes_cover_the_named_cases():
    for name in fcp.SHAPES:
        argv, p, freqs, pl, offs, taps, x = fcp.case(name)
        blk = fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p))
        assert len(blk) >= 2 and blk[-1] < pl.decim * fcp.CHUNK, name        # whole blocks and a partial one
    _, p, _, pl, _, _, x = fcp.case("fm2b_f9")
    assert p.downsample_passes == 3 and fcp.min_chunk(p) == 16
    gold = json.load(open(GOLDEN))["squelch_3ch"]
    first = [next((i for i, h in enumerate(c["hits"]) if h > 0), None) for c in gold["channels"]]
    assert first[0] is not None and first[1] is not None and first[0] < first[1] and first[2] is None


def _channels(name, seed=0):
    argv, p, freqs, pl, offs, taps, x = fcp.case(name, seed)
    lens = fcp.chain_reads(fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p)), pl.decim)
    return p, [d[:sum(lens)] for d in fcp.decimated(x, pl, offs, taps)], lens


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(fcp.SHAPES))
def test_channels_port_equals_reference(name, port, ref_fm):
    p, decs, lens = _channels(name, seed=1)
    op = fcp.oracle_params(p)
    for c, y in enumerate(decs):
        a = fac.port_run_seq(port, op, y, lens, return_chunks=True)
        b = fac.ref_run_seq(ref_fm, op, y, lens, return_chunks=True)
        assert a[0].tobytes() == b[0].tobytes(), (name, c)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (name, c)


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fcp.SHAPES)
    for name in fcp.SHAPES:
        argv, p, freqs, pl, offs, taps, x = fcp.case(name)
        g = gold[name]
        assert g["argv"] == argv and g["params"] == {k: int(v) for k, v in vars(fcp.oracle_params(p)).items()}, name
        assert (g["centre_hz"], g["decim"], g["capture_rate"], g["n_taps"], g["offsets"]) == \
            (pl.centre_hz, pl.decim, pl.capture_rate, pl.n_taps, offs), name
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        blk = fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p))
        assert g["blocks"] == blk, name
        lens = fcp.chain_reads(blk, pl.decim)
        for c, dec in enumerate(fcp.decimated(x, pl, offs, taps)):
            gc = g["channels"][c]
            assert gc["freq"] == freqs[c]
            assert hashlib.sha256(dec[:sum(lens)].tobytes()).hexdigest() == gc["dec_sha256"], (name, c)
            pcm, rl, hits = fcp.port_channel(port, p, dec, lens)
            assert rl.tolist() == gc["result_len"] and hits.tolist() == gc["hits"], (name, c)
            assert hashlib.sha256(pcm.tobytes()).hexdigest() == gc["sha256"], (name, c)


@pytest.fixture(scope="module")
def shell():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)
    return RX_FM


NOAA3 = ["-f", "162.4M", "-f", "162.425M", "-f", "162.45M"]


@pytest.mark.parametrize("args,filename,env_rate,needle", [
    (NOAA3, "-", "40000000", "'-' as the filename"),
    (NOAA3 + ["-L", "4"], "out", "40000000", "does not take -L"),
    (NOAA3 + ["-o", "2"], "out", "40000000", "does not take -o"),
    (NOAA3 + ["-f", "162.425M"], "out", "40000000", "162425000 Hz is given twice"),
    (["-f", "162.4M:162.45M:25k"] + NOAA3[:2], "out", "40000000", "162400000 Hz is given twice"),
    (NOAA3, "out", "2015999", "need a capture rate of 2016000 Hz"),
    (["-f", "162.4M", "-f", "162.400001M"], "out", "40000000", "2^20"),
])
def test_shell_refusals_exit_before_the_device(tmp_path, shell, args, filename, env_rate, needle):
    cap = tmp_path / "cap.cs16"
    np.zeros(4096, np.int16).tofile(cap)
    argv = [shell] + args + ["-d", f"driver=file,path={cap}"]
    env = dict(os.environ, RXB200_CAPTURE_RATE=env_rate)
    r = subprocess.run(argv + ([filename] if filename != "-" else []), capture_output=True, env=env, timeout=120,
                       cwd=tmp_path)
    err = r.stderr.decode()
    assert r.returncode == 1, err
    assert needle in err, err
    assert "Using device" not in err                          # the device was never opened
    assert sorted(os.listdir(tmp_path)) == ["cap.cs16"]       # and no file was created


def test_shell_without_capture_mode_still_asks_for_a_squelch_level(tmp_path, shell):
    env = {k: v for k, v in os.environ.items() if k != "RXB200_CAPTURE_RATE"}
    r = subprocess.run([shell, "-f", "162.4M", "-f", "162.425M", "out"], capture_output=True, env=env, timeout=120,
                       cwd=tmp_path)
    assert r.returncode == 1 and "Please specify a squelch level" in r.stderr.decode()
    assert os.listdir(tmp_path) == []
