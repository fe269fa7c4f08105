"""The mixer and the DDC at the lengths and channel counts of real captures, where their launch rules leave the corner
every short call lands in (tests/mix_scale.py restates the rules; each case asserts the regime it claims):

  a. rxb200_mix_device at two or more grid-stride trips, on all four fm_mix_kernel instantiations (VEC x SMEM);
  b. rxb200_ddc_device with U set by the staging room ("span"), T < M, T = M and T > M, 1 to 32 lanes per output, both
     accumulators; and once with U set by the share of the outputs ("n_out");
  c. rxb200_ddc_device with U set by the reach of the table offsets ("reach"): M = 4096 on a 1 GiB capture, L = 2^20;
  d. plain mixing handles with 257 and 600 channels (2 and 3 grid rows), with every grid row's tables in shared memory
     and with tables far beyond it, over ragged reads and one call long enough for two trips at that grid;
  e. decimating handles at the tool's operating point (19.2 Msps, M = 64, T = 257) with 8 and 257 channels, with 4096-
     and 8192-tap filters over reads shorter than the filter, and with T < M over reads at every phase of M.

The kernels alone (a-c) are compared bit for bit with the numpy mixer and the sparse DDC model; the handles (d, e) with
the port on the models' streams.  Every output buffer has a guard past its end that must stay untouched."""
import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_handles as fh
import fm_mix as fmx
import mix_scale as ms
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

GUARD = 64              # int16 past the last output that must stay zero


def _capture(n_complex, seed):
    """A random full-range capture of n_complex samples, generated on the device."""
    torch = fh.torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-32768, 32768, (2 * n_complex,), dtype=torch.int16, device="cuda", generator=g)


# ---- a. the mixer alone at two or more trips ----------------------------------------------------------------------
@pytest.mark.parametrize("rate,f", [(2_400_000, 37500), (1_000_000, 33001), (1 << 20, 1)])
@pytest.mark.parametrize("vec", [True, False])
def test_mix_device_two_trips(rate, f, vec):
    torch = fh.torch()
    sms = ms.device_sms()
    n = 2 * sms * 8 * 2048 + 5
    assert ms.mix_trips_at_least(n, 1, sms) >= 2
    t = fm.mix_table(rate, f)
    L = t.shape[0]
    assert ms.mix_uses_smem([L]) == (L == 64)                       # SMEM at L = 64; L > 12 288 reads through L1
    x = np.random.default_rng(L + vec).integers(-32768, 32768, size=2 * n).astype(np.int16)
    pad = 8 if vec else 2                                            # 16 bytes: vectors; 4 bytes: word accesses
    src = torch.from_numpy(np.concatenate([np.zeros(pad, np.int16), x])).cuda()
    dst = torch.zeros(pad + 2 * n + GUARD, dtype=torch.int16, device="cuda")
    assert ((src.data_ptr() + 2 * pad) % 16 == 0) == vec and ((dst.data_ptr() + 2 * pad) % 16 == 0) == vec
    for phase in (0, L - 1, (1 << 40) + 3):
        dst.fill_(0)
        fm.mix_device(rate, f, phase, src.data_ptr() + 2 * pad, n, dst.data_ptr() + 2 * pad)
        torch.cuda.synchronize()
        got = dst[pad:pad + 2 * n].cpu().numpy()
        want = fmx.mix_model(x, t, phase % L)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (rate, f, vec, phase, bad[:4])
        assert not dst[:pad].any().item() and not dst[pad + 2 * n:].any().item(), (rate, f, vec, phase)


# ---- b, c. the DDC alone ------------------------------------------------------------------------------------------
def _taps(kind, M, T, seed):
    """(taps, shift): a Q15 low-pass (the int accumulator) or random taps of 2^19 to 2^20 either sign at S = 3 (the
    long long one, with outputs that saturate)."""
    if kind == "lowpass":
        return fdd.lowpass(T, 0.45 / M), 15
    rng = np.random.default_rng(seed)
    mag = rng.integers(1 << 19, 1 << 20, size=T)
    return (mag * rng.choice([-1, 1], size=T)).astype(np.int32), 3


def _ddc_device_check(rate, f, ddc, x, n, phases, regime, what):
    """rxb200_ddc_device on the first n samples of the device capture x at each phase, against the sparse model; the
    call's launch must be in `regime`."""
    torch = fh.torch()
    M, taps, S = ddc
    t = fm.mix_table(rate, f)
    L = t.shape[0]
    n_out = n // M
    U, which = ms.ddc_regime(n_out, M, taps.size, 1, ms.device_sms())
    assert which == regime, (what, U, which)
    dst = torch.zeros(2 * n_out + GUARD, dtype=torch.int16, device="cuda")
    for phase in phases:
        dst.fill_(0)
        fm.ddc_device(rate, f, phase, ddc, x.data_ptr(), n, dst.data_ptr())
        torch.cuda.synchronize()
        want, _ = ms.ddc_sparse(x[:2 * n], t, taps, M, S, table_phase=phase % L)
        assert want.size == 2 * n_out
        got = dst[:2 * n_out].cpu().numpy()
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (what, U, phase, bad[:4])
        assert not dst[2 * n_out:].any().item(), (what, phase)


# (M, T, lanes per output, regime): T > M, T = M and T < M; the last two share the outputs out instead
DDC_DEVICE_CASES = [(64, 257, 32, "span"), (1, 1, 1, "span"), (2, 2, 2, "span"), (100, 31, 32, "span"),
                    (16, 7, 8, "span"), (7, 29, 32, "span"), (7, 29, 32, "n_out"), (64, 257, 32, "n_out")]


@pytest.mark.parametrize("taps_kind", ["lowpass", "random"])
@pytest.mark.parametrize("M,T,lpo,regime", DDC_DEVICE_CASES)
def test_ddc_device_regimes(M, T, lpo, regime, taps_kind):
    assert ms.ddc_lanes(T) == lpo
    taps, S = _taps(taps_kind, M, T, M * 1000 + T)
    assert fdd.wide(taps, S) == (taps_kind == "random")
    span, ctas = ms.ddc_span(M, T), ms.ddc_ctas(1, ms.device_sms())
    # span: every CTA but the last stages (span - 1) * ws + T samples, the last 3 outputs; n_out: half the room
    n_out = ctas * span + 3 if regime == "span" else ctas * max(1, span // 2) + 1
    n = n_out * M + M - 1
    x = _capture(n, M * 7 + T)
    _ddc_device_check(2_400_000, 37500, (M, taps, S), x, n, (0, (1 << 40) + 3), regime, (M, T, taps_kind))


def test_ddc_device_reach():
    """M = 4096, T <= 16: U = 256 outputs per CTA cover 2^20 capture samples, the most the table offsets may span; with
    L = 2^20, one phase puts every CTA's first staged sample at table entry L - 1, so base + ddc_off runs up to
    2^21 - 4096 + T - 1."""
    torch = fh.torch()
    sms = ms.device_sms()
    M = 4096
    n = (2 * sms * 256 + 64) * M                                  # 1.03 GiB on 132 SMs
    x = _capture(n, 4096)
    rate, f = 1 << 20, 1
    L = fm.mix_table(rate, f).shape[0]
    assert L == 1 << 20
    for T, kind in ((1, "lowpass"), (5, "random"), (16, "random"), (16, "lowpass")):
        taps, S = _taps(kind, M, T, T)
        U, _ = ms.ddc_regime(n // M, M, T, 1, sms)
        assert U * M == 1 << 20
        # CTA b's first staged sample is b * 2^20 + M - T: at phase L - 1 - (M - T) it takes entry L - 1
        _ddc_device_check(rate, f, (M, taps, S), x, n, (L - 1, L - 1 - (M - T)), "reach", (T, kind))
    del x
    torch.cuda.empty_cache()


# ---- d. plain mixing handles with more than one grid row ----------------------------------------------------------
# name -> (capture rate, the distinct offsets, channels).  Channel k takes distinct offset (19 k) mod 47: neighbours
# differ, and 47 is prime to 256, so a channel read from another grid row's slot differs too.
PLAIN_LAYOUTS = {
    # a 400 kHz raster at 19.2 Msps: periods 48 / gcd(48, j) <= 48, so 256 channels' tables fit 96 KiB
    "smem_k600": (19_200_000, [400_000 * j for j in range(-23, 24)], 600),
    # a 25 kHz raster of odd multiples: periods of 768 or 256 entries, about 1.5 MB per grid row
    "l1_k257": (19_200_000, [25_000 * (-367 + 16 * i) for i in range(47)], 257),
}


def _cycle(distinct, k):
    return [distinct[(19 * c) % len(distinct)] for c in range(k)]


def _two_trip_call(n_groups, chunk_complex):
    """The shortest call of whole chunks whose every grid row makes two trips."""
    sms = ms.device_sms()
    k = 1
    while ms.mix_trips_at_least(k * chunk_complex, n_groups, sms) < 2:
        k += 1
    return k * chunk_complex


@pytest.mark.parametrize("name", sorted(PLAIN_LAYOUTS))
def test_plain_handle_many_channels(name, port):
    torch = fh.torch()
    rate, distinct, K = PLAIN_LAYOUTS[name]
    p = fmx.SHAPES["fm5a_lut_d100"][0]                            # D = 100 lut: small PCM
    offs = _cycle(distinct, K)
    periods = [fm.mix_table(rate, f).shape[0] for f in offs]
    n_groups = ms.groups(K)
    assert n_groups == (3 if K > 512 else 2)
    smem = name.startswith("smem")
    assert ms.mix_uses_smem(periods) == smem
    assert all(sum(periods[:g * 256]) > 0 for g in range(1, n_groups))   # rows >= 1 stage from lo != 0
    chunk = 2 * 25000
    n_call = _two_trip_call(n_groups, chunk // 2)
    reads = fmx.READS
    n_reads = sum(reads) // 2
    x = fmx.capture(n_reads + n_call, rate, distinct[::8], 960 + K)
    cap = torch.from_numpy(x).cuda()
    mx = fm.FmMix(p, rate, offs)
    stride = max(mx.max_output(2 * n_call, chunk), max(mx.max_output(n, n) for n in reads)) + 64
    out = torch.zeros((K, stride), dtype=torch.int16, device="cuda")
    parts, pos = [], 0
    for n16 in reads:
        k = mx.process_read_device(cap.data_ptr() + 2 * pos, n16, out.data_ptr(), stride, sync=True)
        parts.append(out[:, :k].cpu().numpy())
        pos += n16
    out.zero_()
    k = mx.process_device(cap.data_ptr() + 2 * pos, 2 * n_call, chunk, out.data_ptr(), stride, sync=True)
    parts.append(out[:, :k].cpu().numpy())
    assert not out[:, k:].any().item()
    got = np.concatenate(parts, axis=1)
    mx.close()
    del cap, out
    lens = list(reads) + [chunk] * (2 * n_call // chunk)
    for f in distinct:
        want = fac.port_run_seq(port, p, fmx.mix_model(x, fm.mix_table(rate, f)), lens)
        for c in [c for c in range(K) if offs[c] == f]:
            fh.compare(p, got[c], want, (name, c, f))


# ---- e. decimating handles at scale -------------------------------------------------------------------------------
def _ddc_handle_check(port, p, rate, offs, ddc, x, ops, what, reset_again=False):
    """Runs ops -- ("call", n16, chunk16) through process_device, ("read", n16) through process_read_device -- over the
    device capture x on a decimating handle, and compares every channel with the port on the sparse model's decimated
    stream.  Returns the launch regimes of the calls.  reset_again: reset and run the same ops again, byte for byte."""
    torch = fh.torch()
    M, taps, S = ddc
    K = len(offs)
    sms = ms.device_sms()
    total = sum(op[1] for op in ops)
    mx = fm.FmMix(p, rate, offs, ddc=ddc)
    bound = max(mx.max_output(op[1], op[2] if op[0] == "call" else max(op[1], 2)) for op in ops)
    stride = bound + 64

    def run():
        out = torch.zeros((K, stride), dtype=torch.int16, device="cuda")
        parts, lens, regimes, pos = [], [], [], 0
        for op in ops:
            n16 = op[1]
            n_dec = mx.decimated_len(n16)
            if n_dec:
                regimes.append(ms.ddc_regime(n_dec // 2, M, taps.size, K, sms))
            out.zero_()
            if op[0] == "call":
                k = mx.process_device(x.data_ptr() + 2 * pos, n16, op[2], out.data_ptr(), stride, sync=True)
                lens += [fdd.decimated_len(pos // 2 + a // 2, min(op[2], n16 - a), M) for a in range(0, n16, op[2])]
            else:
                k = mx.process_read_device(x.data_ptr() + 2 * pos, n16, out.data_ptr(), stride, sync=True)
                lens.append(n_dec)
            parts.append(out[:, :k].cpu().numpy())
            assert not out[:, k:].any().item(), (what, op)
            pos += n16
        return np.concatenate(parts, axis=1), [v for v in lens if v], regimes

    got, lens, regimes = run()
    if reset_again:
        mx.reset()
        again, _, _ = run()
        assert again.tobytes() == got.tobytes(), what
    mx.close()
    for j, f in enumerate(offs):
        y, _ = ms.ddc_sparse(x[:total], fm.mix_table(rate, f), taps, M, S)
        assert y.size == sum(lens), (what, j)
        want = fac.port_run_seq(port, p, y, lens)
        fh.compare(p, got[j], want, (what, j, f))
    return regimes


def _op_point_offsets(K):
    if K == 8:
        return [-9_000_000, -2_400_000, -25_000, 0, 25_000, 1_200_000, 4_800_000, 9_000_000]
    return [25_000 * (j - K // 2) for j in range(K)]


@pytest.mark.parametrize("K", [8, 257])
def test_ddc_handle_operating_point(K, port):
    """19.2 Msps, M = 64, T = 257 into a D = 12 lut chain: one span-bound call of 2.36 M samples, then ragged reads."""
    p, rate, _, ddc, _, _ = fdd.SHAPES["nbfm_m64_t257"]
    M = ddc[0]
    chunk = 2 * M * 4096
    ops = [("call", 9 * chunk, chunk)] + [("read", n) for n in fdd.READS]
    offs = _op_point_offsets(K)
    x = _capture(sum(op[1] for op in ops) // 2, 1900 + K)
    regimes = _ddc_handle_check(port, p, rate, offs, ddc, x, ops, ("op_point", K))
    assert regimes[0] == (124, "span"), regimes


LONG_READS = [2 * 3001, 2 * 1777, 2 * 4093, 2 * 37, 2 * 2503]      # each shorter than T - 1 below


@pytest.mark.parametrize("M", [8, 64])
@pytest.mark.parametrize("T", [4096, 8192])
def test_ddc_handle_long_filter(M, T, port):
    """Reads shorter than the filter, several in a row: the history spans several calls, and every CTA of a call (not
    only the first) reads some of it.  Then a reset and the same reads again."""
    p = fdd.SHAPES["raw_m100"][0]                                   # raw, chain D = 1
    rate, offs = 2_400_000, [0, 24000, -48000]
    ddc = (M, fdd.lowpass(T, 0.45 / M), 15)
    ops = [("read", n) for n in LONG_READS * 3]
    x = _capture(sum(op[1] for op in ops) // 2, T + M)
    regimes = _ddc_handle_check(port, p, rate, offs, ddc, x, ops, ("long", M, T), reset_again=True)
    assert regimes and all(T - 1 > U * M for U, _ in regimes), regimes      # CTA 1 on starts inside the history
    if T == 8192:
        assert all(r == (1, "span") for r in regimes), regimes         # room for one window per CTA


def test_ddc_handle_taps_fewer_than_decim(port):
    """M = 100, T = 31: windows do not overlap, and the reads move the phase within M through many values."""
    p = fdd.SHAPES["raw_m100"][0]
    rate, offs = 2_400_000, [0, 24000, -48000]
    M = 100
    ddc = (M, fdd.lowpass(31, 6000 / 2.4e6), 15)
    lens = [2 * 1013, 2 * 37, 2 * 2999, 2 * 461, 2 * 7, 2 * 5003, 2 * 251]
    ops = [("read", n) for n in lens * 6]
    phases = np.cumsum([0] + [op[1] // 2 for op in ops])[:-1] % M
    assert len(set(phases.tolist())) >= 30
    x = _capture(sum(op[1] for op in ops) // 2, 3100)
    regimes = _ddc_handle_check(port, p, rate, offs, ddc, x, ops, ("t_lt_m",))
    assert {w for _, w in regimes} == {"n_out"}, regimes
