"""rx_power's planners at a device rate and the shells' RXB200_DEVICE_RATE refusals, without a GPU.

rxb200_power_plan_capture against the rule rx_power_b200 used to compute inline, rxb200_power_plan_capture_at and
rxb200_power_plan_tiles_at against their restatements (tests/power_device_rate.py) over seeded plans, refusals included;
for every accepted plan the resampler fits each tile and no tile runs above the device rate, and a burst's device count
(rxb200_resample_in_len) emits exactly the outputs it is asked for.  The shells refuse a bad RXB200_DEVICE_RATE before
they open the device."""
import os
import random
import subprocess

import pytest

import power_device_rate as pdr
import resample as rsm
from rx_tools_b200 import _lib, power
from rx_tools_b200 import resample as rs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "host")
DEVICE_RATES = (1_000_000, 2_048_000, 2_400_000, 2_500_000, 3_200_000, 10_000_000, 20_000_000, 30_720_000,
                61_440_000, 122_880_000)


def _plans(n, seed):
    """n seeded rx_power plans, spans from one hop to thousands, crops and -F included."""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        lo = rng.randrange(24_000_000, 1_700_000_000, 1000)
        width = rng.choice((200_000, 900_000, 2_000_000, 5_000_000, 20_000_000, 80_000_000, 400_000_000))
        width = rng.randrange(width // 2, width + 1, 1000)
        step = rng.choice(("1k", "5k", "10k", "50k", "1M", "2.4M"))
        crop = rng.choice((0.0, 0.1, 0.285, 0.5))
        boxcar, fir = rng.choice(((1, 0), (0, 9)))
        try:
            out.append(power.plan_range(f"{lo}:{lo + width}:{step}", crop, boxcar, fir, 0))
        except _lib.Rxb200Error:
            continue
    return out


def _capture(plan, cap, R_dev=None):
    try:
        p, offs = power.plan_capture(plan, cap, device_rate=R_dev)
    except _lib.Rxb200Error as e:
        return e.code
    return p, offs


def test_plan_capture_is_the_old_inline_rule():
    rng = random.Random(11)
    n_refused = 0
    for plan in _plans(320, 1):
        cap = rng.choice((plan.rate, 2_500_000, 20_000_000, 40_000_000, 200_000_000, 1 << 40))
        want, got = pdr.inline_rule(plan, cap), _capture(plan, cap)
        if want == "rate":
            n_refused += 1
            assert got == _lib.EINVAL
            assert "needs a capture rate of" in _lib.lib().rxb200_last_error().decode()
            continue
        fc, offs, M, R, T = want
        p, o = got
        assert (p.centre_hz, p.decim, p.capture_rate, p.n_taps, o) == (fc, M, R, T, offs)
    assert 20 < n_refused < 300


def test_plan_capture_at_matches_restatement():
    rng = random.Random(12)
    seen = {}
    for plan in _plans(320, 2):
        R_dev = rng.choice(DEVICE_RATES + (0, -5, 1 << 31))
        cap = rng.choice((20_000_000, 200_000_000, 1 << 40))
        want, got = pdr.capture_at_rule(plan, cap, R_dev), _capture(plan, cap, R_dev)
        code = {"device_rate": _lib.EINVAL, "rate": _lib.EINVAL, "device": _lib.EUNSUPPORTED}
        seen[want if isinstance(want, str) else "ok"] = 1
        if isinstance(want, str):
            assert got == code[want], (want, got)
            if want == "device":
                msg = _lib.lib().rxb200_last_error().decode()
                assert str(R_dev) in msg and "device rate" in msg
            continue
        fc, offs, M, R, T, span = want
        p, o = got
        assert (p.centre_hz, p.decim, p.capture_rate, p.n_taps, o) == (fc, M, R, T, offs)
        assert R <= R_dev
        L, N, _, _ = rsm.plan_rule(R_dev, R, span)          # the span leaves the guard band (J L may still be refused)
        assert L <= N
    assert set(seen) == {"ok", "device_rate", "rate", "device"}


def test_plan_capture_at_refusal_order():
    plan = power.plan_range("88M:108M:10k")                 # 8 hops at 2.5 M: M = 8 today, 9 with a 625 k guard
    assert _capture(plan, 1 << 40, 0) == _lib.EINVAL           # the device rate first, whatever else is wrong
    assert _capture(plan, 1, 0) == _lib.EINVAL
    assert _capture(plan, 1, 20_000_000) == _lib.EINVAL        # the cap before R > R_dev
    assert _capture(plan, 1 << 40, 20_000_000) == _lib.EUNSUPPORTED
    p, _ = _capture(plan, 1 << 40, 30_720_000)
    assert (p.decim, p.capture_rate) == (9, 22_500_000)
    p0, _ = _capture(plan, 1 << 40)
    assert (p0.decim, p0.capture_rate) == (8, 20_000_000)


def _tiles(plan, cap, R_dev):
    try:
        return power.plan_tiles(plan, cap, device_rate=R_dev)
    except _lib.Rxb200Error as e:
        return e.code


def test_plan_tiles_at_matches_restatement_and_fits_the_device():
    rng = random.Random(13)
    n_ok = n_multi = 0
    for plan in _plans(320, 3):
        R_dev = rng.choice(DEVICE_RATES + (0,))
        cap = rng.choice((plan.rate, 5_000_000, 20_000_000, 40_000_000, 1 << 40))
        want, got = pdr.tiles_at_rule(plan, cap, R_dev), _tiles(plan, cap, R_dev)
        if isinstance(want, str):
            assert got == _lib.EINVAL, (want, got)
            continue
        n_tiles, h, M, R, T, offs, tiles = want
        tl, tt, o = got
        assert (tl.n_tiles, tl.hops_per_tile, tl.decim, tl.capture_rate, tl.n_taps) == (n_tiles, h, M, R, T)
        assert o == offs and [t[:3] for t in tiles] == tt
        assert R <= R_dev and R <= cap
        for (_, _, _, span) in tiles:
            L, N, _, _ = rsm.plan_rule(R_dev, R, span)             # the guard band fits every tile
            assert L <= N
        n_ok += 1
        n_multi += n_tiles > 1
    assert n_ok > 100 and n_multi > 20


def test_plan_tiles_without_device_rate_unchanged():
    """_tiles_at's rule at G = 0 is rxb200_power_plan_tiles; the entry without a device rate keeps its plans."""
    for plan in _plans(60, 4):
        for cap in (5_000_000, 40_000_000):
            tl, tiles, offs = power.plan_tiles(plan, cap)
            a = power.plan_tiles(plan, cap, device_rate=None)
            assert (tl, tiles, offs) == a


def test_plan_tiles_at_one_hop_too_wide():
    plan = power.plan_range("100M:110M:1M")                     # hops at 1 M
    assert _tiles(plan, 1 << 40, 1_000_000) == _lib.EINVAL       # one hop needs 1 M + 31 250 Hz
    tl, _, _ = _tiles(plan, 1 << 40, 2_048_000)
    assert tl.decim == 2 and tl.capture_rate == 2_000_000 and tl.hops_per_tile == 1


def test_burst_in_len_is_exact():
    """A burst of P passes at a device rate: E = ceil((J - 1) L / N) outputs whose window reaches before the burst, then
    G + P M buf_len / 2.  With L <= N, rxb200_resample_in_len's count emits exactly that many."""
    rng = random.Random(14)
    n = 0
    for plan in _plans(200, 5):
        R_dev = rng.choice(DEVICE_RATES)
        got = _tiles(plan, 1 << 40, R_dev)
        if isinstance(got, int):
            continue
        tl, tiles, _ = got
        T, Mt = tl.n_taps, tl.decim
        lead = Mt * rsm.ceil_div(T - 1, Mt)
        b, e, _ = tiles[0]
        c = (e - b - 1) * plan.freq_step // 2
        span = 2 * max(c, (e - b - 1) * plan.freq_step - c) + plan.rate
        L, N, J, _ = rsm.plan_rule(R_dev, tl.capture_rate, span)
        E = rsm.ceil_div((J - 1) * L, N)
        for P in (1, 3):
            want = E + lead + P * Mt * plan.buf_len // 2
            cin = rs.in_len(L, N, 0, want)
            assert rsm.out_count(0, cin, L, N) == want
            assert rsm.out_count(0, cin - 1, L, N) == want - 1
        n += 1
    assert n > 50


@pytest.fixture(scope="module")
def shells():
    subprocess.run(["make", "-C", HOST, "-s"], check=True)


def _shell(tmp_path, exe, args, env):
    e = dict(os.environ)
    for k in ("RXB200_CAPTURE_RATE", "RXB200_TILE_RATE", "RXB200_DEVICE_RATE", "RXB200_CAPTURE_STAGES"):
        e.pop(k, None)
    e.update(env)
    missing = tmp_path / "no_such_capture.cs16"        # opening the device fails: a refusal must come first
    return subprocess.run([os.path.join(HOST, exe)] + args[:-1] + ["-d", f"driver=file,path={missing}", args[-1]],
                          capture_output=True, env=e, timeout=60)


SHELL_CASES = {
    "rx_fm": ("rx_fm_b200", ["-M", "fm", "-s", "24k", "-l", "50", "-f", "162.4M", "-f", "162.55M"]),
    "rx_sdr": ("rx_sdr_b200", ["-s", "250k", "-F", "CS16", "-f", "100M", "-f", "100.95M"]),
    "rx_power": ("rx_power_b200", ["-f", "88M:108M:10k", "-1"]),
}


@pytest.mark.parametrize("shell", sorted(SHELL_CASES))
def test_shell_refusals_before_the_device(tmp_path, shells, shell):
    exe, args = SHELL_CASES[shell]
    out = tmp_path / "out"
    # without a capture (or tile) variable
    r = _shell(tmp_path, exe, args + [str(out)], {"RXB200_DEVICE_RATE": "2400000"})
    assert r.returncode == 1 and "RXB200_DEVICE_RATE" in r.stderr.decode(), r.stderr.decode()
    assert "Failed to open" not in r.stderr.decode() and not list(tmp_path.glob("out*"))
    # a device rate that is not a rate
    r = _shell(tmp_path, exe, args + [str(out)], {"RXB200_CAPTURE_RATE": "100000000", "RXB200_DEVICE_RATE": "fast"})
    assert r.returncode == 1 and "RXB200_DEVICE_RATE" in r.stderr.decode()
    assert "Failed to open" not in r.stderr.decode() and not list(tmp_path.glob("out*"))
    # the plan needs more than the device rate: R > R_dev, or no room for the guard band
    slow = {"rx_fm": "100000", "rx_sdr": "1000000", "rx_power": "20000000"}[shell]
    r = _shell(tmp_path, exe, args + [str(out)], {"RXB200_CAPTURE_RATE": "100000000", "RXB200_DEVICE_RATE": slow})
    err = r.stderr.decode()
    assert r.returncode == 1 and f"device rate of {slow} Hz" in err, err
    assert "Failed to open" not in err and not list(tmp_path.glob("out*"))


def test_rx_power_tile_mode_refusals_before_the_device(tmp_path, shells):
    exe, args = SHELL_CASES["rx_power"]
    out = tmp_path / "out"
    r = _shell(tmp_path, exe, args + [str(out)], {"RXB200_TILE_RATE": "10000000", "RXB200_DEVICE_RATE": "1000000"})
    err = r.stderr.decode()
    assert r.returncode == 1 and "Tile mode" in err and "Failed to open" not in err and not out.exists()
    r = _shell(tmp_path, exe, args + [str(out)], {"RXB200_TILE_RATE": "10000000", "RXB200_DEVICE_RATE": "0"})
    assert r.returncode == 1 and "RXB200_DEVICE_RATE" in r.stderr.decode() and not out.exists()


def test_rx_power_capture_refusal_wording_unchanged(tmp_path, shells):
    """Without RXB200_DEVICE_RATE the capture mode's refusal reads as it did before the planner moved into the
    library."""
    out = tmp_path / "out"
    r = _shell(tmp_path, "rx_power_b200", ["-f", "88M:108M:10k", str(out)], {"RXB200_CAPTURE_RATE": "19999999"})
    assert r.returncode == 1 and not out.exists()
    assert r.stderr.decode().endswith(
        "Capture mode: the span needs a capture rate of 20000000 Hz, above RXB200_CAPTURE_RATE=19999999.\n")


def _replay(tmp_path, exe, args, env, keywords):
    cap = tmp_path / "cap.cs16"
    cap.write_bytes(bytes(4096))
    e = {k: v for k, v in os.environ.items() if not k.startswith("RXB200_")}
    e.update(env)
    return subprocess.run([os.path.join(HOST, exe), "-d", f"driver=file,path={cap},{keywords}"] + args,
                          capture_output=True, env=e, timeout=60)


@pytest.mark.parametrize("bad", ["abc", "0", "-5", "2.4Mx", ""])
def test_replay_device_refuses_a_bad_rate(tmp_path, shells, bad):
    """rate= must be a positive number of Hz: a typo must not turn the device into one that honours any rate."""
    r = _replay(tmp_path, "rx_sdr_b200", ["-F", "CS16", str(tmp_path / "out")], {}, f"rate={bad}")
    assert r.returncode == 1 and "Failed to open sdr device" in r.stderr.decode()
    assert not (tmp_path / "out").exists()


def test_rx_sdr_refuses_a_reported_rate_that_is_not_a_rate(tmp_path, shells):
    """A device that reports no usable rate (a driver without getSampleRate reports 0; here one above 2^31 - 1) ends the
    run before any sample is taken, instead of falling back to treating its samples as the plan's rate."""
    args = ["-s", "250k", "-F", "CS16", "-f", "100M", "-f", "100.95M", str(tmp_path / "out")]
    r = _replay(tmp_path, "rx_sdr_b200", args, {"RXB200_CAPTURE_RATE": "100000000", "RXB200_DEVICE_RATE": "2400000"},
                "rate=3000000000")
    err = r.stderr.decode()
    assert r.returncode == 1 and "reports a sample rate of 3000000000 Hz" in err, err
    assert not list(tmp_path.glob("out*"))
