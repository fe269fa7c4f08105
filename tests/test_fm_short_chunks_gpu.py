"""rx_fm on chunks shorter than the boxcar, against the port, on every route that runs without fifth_order passes.

A chunk that completes no boxcar leaves fm_demod's carried sample at (0, 0) (src/rtl_fm.c:612-613, as the pinned
reference reads it), so the next emitting chunk's first output is exactly 0 in every atan mode.  Each route -- the fused
kernel's SPEC 0, 1 and 3, the stream path, SPEC 2 with -o 2, the any-length kernel -- runs one long call (also with
segments of 64 samples, so that empty chunks fall inside halos and at item starts), 1 and 3 channels, call sequences cut
where a chunk emitted nothing and where both sides emit, the four entry points, and reset.  am/usb/lsb/raw, which never
read the carried sample, are the controls.  Then the mixing handle, the plain group and the decimating mixing group."""
import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_disc as fd
import fm_mix as fmx
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

D10 = fac.SHORT_STD
WB10 = fac.P(mode=fac.M_FM, downsample=10, custom_atan=1, deemph=1, deemph_a=7, rate_out=100000, rate_out2=32000)
NEVER = str(1 << 40)        # RXB200_FM_STREAM_MIN above any call: the fused SPEC 1 kernel

# name -> (parameters, chunk in complex samples, RXB200_FM_STREAM_MIN or None, kernel_kind of a whole call); every chunk
# is shorter than the boxcar, so that some complete none
ROUTES = {
    "spec0_std_d10": (D10, 8, None, 0),
    "spec0_ale_d10": (fac.with_(D10, custom_atan=3), 8, None, 0),
    "spec0_lut_d10_offset": (fac.with_(D10, custom_atan=2, offset_tuning=1), 8, None, 0),
    "spec1_fast_d10_deemph": (WB10, 8, NEVER, 0),
    "stream_fast_d10_deemph": (WB10, 8, "0", 3),
    "spec3_lut_d100_c96": (fac.FM5A, 96, None, 0),
    "spec3_lut_d100_c8": (fac.FM5A, 8, None, 0),
    "spec3_lut_d12_c8": (fac.NBFM12, 8, None, 0),
    # the any-length kernel: chunks that are not a multiple of 8 complex samples
    "any_std_d10": (D10, 7, None, 0),
    "any_ale_d10": (fac.with_(D10, custom_atan=3), 9, None, 0),
    "any_fast_d10_deemph": (WB10, 9, None, 0),
    "any_lut_d100": (fac.FM5A, 57, None, 0),
    "any_lut_d12": (fac.NBFM12, 5, None, 0),
    # controls
    "am_d42": (fac.AM, 16, None, 0),
    "usb_d42": (fac.USB, 8, None, 0),
    "lsb_d42": (fac.LSB, 16, None, 0),
    "raw_d42": (fac.RAW, 8, None, 0),
}


def _handle(monkeypatch, name, n_ch=1):
    p, _, env, _ = ROUTES[name]
    if env is None:
        monkeypatch.delenv("RXB200_FM_STREAM_MIN", raising=False)
    else:
        monkeypatch.setenv("RXB200_FM_STREAM_MIN", env)
    return fm.FmDemod(p, n_channels=n_ch)


def _zero_after_empty(p):
    """The discriminator's output reaches the PCM unchanged: no de-emphasis, resampler or -o after it."""
    return p.mode == fac.M_FM and not (p.deemph or p.rate_out2 > 0 or p.post_downsample > 1)


def _check(p, got, want, rl, what):
    """got against the port's want; rl the port's result_len per chunk.  The first output after a chunk with none is
    exactly 0 in every atan mode; the fp64 atan2 allowance of -A std applies to the other samples only."""
    assert got.size == want.size, (what, got.size, want.size)
    if _zero_after_empty(p):
        z = fac.after_empty(rl)
        assert z.size > 0 and np.all(want[z] == 0), what
        assert np.all(got[z] == 0), (what, z[got[z] != 0][:5], got[z][got[z] != 0][:5])
        keep = np.ones(got.size, bool)
        keep[z] = False
        got, want = got[keep], want[keep]
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    near = fd.port_met_near_integer()
    if fac.INTEGER(p) or not near:
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    else:       # the port met an atan2 value within 2^-30 of an integer: CUDA's libm may truncate it the other way
        assert np.count_nonzero(diff) <= max(2, int(1e-4 * diff.size)), (what, np.flatnonzero(diff)[:5])
        if _zero_after_empty(p):
            assert diff.max(initial=0) <= 1, what


def _dec(p, c, n):
    """Decimated samples of each chunk of c complex samples over a stream of n (the boxcar's count from a fresh start)."""
    ends = np.minimum(np.arange(1, -(-n // c) + 1) * c, n)
    return np.diff(np.concatenate([[0], ends // p.downsample]))


def _len(name, n_chunks):
    """A stream of n_chunks chunks with a shorter last one; a whole number of 8-sample blocks on the fused routes."""
    c = ROUTES[name][1]
    return n_chunks * c - (8 if c % 8 == 0 else 3)


@pytest.mark.parametrize("n_ch", [1, 3])
@pytest.mark.parametrize("seg", [0, 64])
@pytest.mark.parametrize("name", sorted(ROUTES))
def test_one_long_call(name, seg, n_ch, port, monkeypatch):
    p, c, _, kind = ROUTES[name]
    n = _len(name, (60_000 if p.downsample >= 42 else 20_000) // c)
    x = np.stack([fac.signal(n, 30 + 7 * k + seg) for k in range(n_ch)])
    d = _handle(monkeypatch, name, n_ch)
    if seg:
        d.tune(segment_len=seg)
    got = d.full_demod(x, 2 * c)
    assert d.stats()["kernel_kind"] == kind, d.stats()
    for k in range(n_ch):
        want, rl, _ = port.fm_run(p, x[k], 2 * c, return_chunks=True)
        assert np.any(_dec(p, c, n) == 0), name
        _check(p, got[k], want, rl, (name, seg, k))
    d.close()


def _device(x16, align4):
    """x16 on the device at a 4-byte (align4) or 256-byte aligned address."""
    import torch
    off = 2 if align4 else 0
    buf = torch.zeros(x16.size + off, dtype=torch.int16, device="cuda")
    buf[off:] = torch.from_numpy(np.ascontiguousarray(x16).reshape(-1)).cuda()
    t = buf[off:]
    assert (t.data_ptr() % 16 == 4) == align4
    return buf, t


def _call(d, kind, part, c):
    """One call of entry point `kind` on `part` (one channel); reads take one chunk each."""
    import torch
    if kind == "host":
        return d.full_demod(part, 2 * c)
    if kind == "read":
        return np.concatenate([d.process_read(part[j:j + 2 * c]) for j in range(0, part.size, 2 * c)])
    out = []
    for j in range(0, part.size, part.size if kind == "device" else 2 * c):
        piece = part[j:j + (part.size if kind == "device" else 2 * c)]
        # whole-block chunk calls keep the 32-byte alignment rule; the any-length kernel reads at 4 bytes
        _keep, t = _device(piece, kind == "read_device" or c % 8 != 0)
        cap = d.max_output(piece.size, 2 * c) + 8
        o = torch.zeros(cap, dtype=torch.int16, device="cuda")
        if kind == "device":
            n_pcm = d.process_device(t.data_ptr(), piece.size, 2 * c, o.data_ptr(), cap, sync=True)
        else:
            n_pcm = d.process_read_device(t.data_ptr(), piece.size, o.data_ptr(), cap, sync=True)
        out.append(o[:n_pcm].cpu().numpy())
    return np.concatenate(out)


@pytest.mark.parametrize("name", sorted(ROUTES))
def test_call_sequences(name, port, monkeypatch):
    """Calls cut after chunks that emitted nothing and between two emitting chunks (a call whose last chunk emits, then
    one whose first chunk emits), through host, device, process_read and process_read_device in turn."""
    p, c, _, kind = ROUTES[name]
    n_chunks = 240 if p.downsample < 42 else 600
    x = fac.signal(n_chunks * c, 11)
    want, rl, _ = port.fm_run(p, x, 2 * c, return_chunks=True)
    dec = _dec(p, c, n_chunks * c)
    empty_end = [i for i in range(1, n_chunks) if dec[i - 1] == 0]
    emit_emit = [i for i in range(1, n_chunks) if dec[i - 1] > 0 and dec[i] > 0]
    # chunks shorter than half the boxcar never emit twice in a row
    assert empty_end and (emit_emit or 2 * c < p.downsample), name
    rng = np.random.default_rng(len(name))
    cuts = sorted(set(rng.choice(empty_end, min(10, len(empty_end)), replace=False).tolist()) |
                  set(rng.choice(emit_emit, min(10, len(emit_emit)), replace=False).tolist()))
    d = _handle(monkeypatch, name)
    parts, lo = [], 0
    for j, hi in enumerate(cuts + [n_chunks]):
        ep = ("host", "device", "read", "read_device")[j % 4]
        parts.append(_call(d, ep, x[2 * c * lo:2 * c * hi], c))
        if ep == "host":
            assert d.stats()["kernel_kind"] == kind, name
        lo = hi
    _check(p, np.concatenate(parts), want, rl, name)
    d.close()


@pytest.mark.parametrize("name", sorted(ROUTES))
def test_reset_after_an_empty_chunk(name, port, monkeypatch):
    p, c, _, _ = ROUTES[name]
    n = _len(name, 300)
    x = fac.signal(n, 12)
    want, rl, _ = port.fm_run(p, x, 2 * c, return_chunks=True)
    dec = _dec(p, c, n)
    end = [i for i in range(1, n // c) if dec[i - 1] == 0][-1]       # the prefix ends with a chunk that emitted nothing
    y = x[::-1].copy()
    d = _handle(monkeypatch, name)
    d.full_demod(x[:2 * c * end], 2 * c)
    d.reset()
    _check(p, d.full_demod(x, 2 * c), want, rl, name)
    d.reset()
    wy, rly, _ = port.fm_run(p, y, 2 * c, return_chunks=True)
    _check(p, d.full_demod(y, 2 * c), wy, rly, (name, "reversed"))
    d.close()


@pytest.mark.parametrize("n_ch", [1, 3])
@pytest.mark.parametrize("name", ["any_std_d10", "any_ale_d10", "any_fast_d10_deemph", "any_lut_d100", "any_lut_d12",
                                  "am_d42", "raw_d42"])
def test_reads_of_one_to_two_boxcars(name, n_ch, port):
    """process_read over reads of 1 to 2D complex samples, odd lengths among them."""
    p = ROUTES[name][0]
    rng = np.random.default_rng(n_ch * 100 + p.downsample)
    lens = fac.ragged_lens(rng, 150, 1, 2 * p.downsample)
    n = fac.seq_len(lens)
    x = np.stack([fac.signal(n, 40 + k) for k in range(n_ch)])
    d = fm.FmDemod(p, n_channels=n_ch)
    got = np.concatenate([d.process_read(x[:, pos:pos + m]) for pos, m in fac.seq_bounds(x.shape[1], lens)], axis=1)
    for k in range(n_ch):
        want, rl, _ = fac.port_run_seq(port, p, x[k], lens, return_chunks=True)
        _check(p, got[k], want, rl, (name, k))
    d.close()


@pytest.mark.parametrize("n_ch", [1, 3])
@pytest.mark.parametrize("cycle", ["whole_blocks", "any"])
@pytest.mark.parametrize("atan", [0, 2])
def test_post_downsample_2_with_empty_chunks(atan, cycle, n_ch, port):
    """-o 2 (the SPEC 2 kernel) at D = 12, one call per chunk, each decimating to 0 or 2 samples: whole 8-sample blocks
    (the fused kernel) or any lengths (mostly the any-length kernel), through the chunk and the read entry point."""
    p = fac.with_(fac.NBFM12, custom_atan=atan, post_downsample=2)
    lens = [2 * v for v in ([24, 8, 16] if cycle == "whole_blocks" else fac.O2_CYCLE)]
    n = 30 * sum(lens) // 2
    x = np.stack([fac.signal(n, 50 + k) for k in range(n_ch)])
    d = fm.FmDemod(p, n_channels=n_ch)
    parts = []
    for j, (pos, m) in enumerate(fac.seq_bounds(n * 2, lens)):
        part = x[:, pos:pos + m]
        parts.append(d.full_demod(part, m) if j % 2 else d.process_read(part))
        if cycle == "whole_blocks":
            assert d.stats()["kernel_kind"] == 0
    got = np.concatenate(parts, axis=1)
    for k in range(n_ch):
        want, rl, _ = fac.port_run_seq(port, p, x[k], lens, return_chunks=True)
        assert np.any(rl == 0) and set(rl.tolist()) <= {0, 1}       # -o 2 makes one output of two samples
        _check(p, got[k], want, rl, (atan, cycle, k))
    d.close()


# ---- the handles that produce short chain reads themselves
MIX_READS = [2 * 37, 2 * 8, 2 * 150, 2 * 3, 2 * 1021, 2 * 99]


def test_mixing_handle_reads_shorter_than_the_boxcar(port):
    p, rate, offs, _ = fmx.SHAPES["fm5a_lut_d100"]
    x = fmx.capture(6 * sum(MIX_READS) // 2, rate, offs, 21)
    mx = fm.FmMix(p, rate, offs)
    got = np.concatenate([mx.process_read(x[pos:pos + m]) for pos, m in fac.seq_bounds(x.size, MIX_READS)], axis=1)
    for k, f in enumerate(offs):
        y = fmx.mix_model(x, fm.mix_table(rate, f))
        want, rl, _ = fac.port_run_seq(port, p, y, MIX_READS, return_chunks=True)
        _check(p, got[k], want, rl, f)
    mx.close()


def test_group_chunks_shorter_than_the_boxcar(port):
    p, n_ch, c = fac.FM5A, 5, 8
    n = 40_000 - 8
    x = np.stack([fac.signal(n, 60 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices=[0, 0, 0])
    got = g.full_demod(x, 2 * c)
    for k in range(n_ch):
        want, rl, _ = port.fm_run(p, x[k], 2 * c, return_chunks=True)
        _check(p, got[k], want, rl, k)
    g.close()


def test_decimating_mixing_group_reads_that_decimate_to_a_few_samples(port):
    p, rate, offs, ddc, x, reads = fdd.case_input("nbfm_m64_t257_short", seed=2)
    grp = fm.FmMixGroup(p, rate, offs, devices=[0, 0], ddc=ddc)
    got = np.concatenate([grp.process_read(x[pos:pos + m]) for pos, m in fac.seq_bounds(x.size, reads)], axis=1)
    for k, f in enumerate(offs):
        y, lens = fdd.nonempty(fdd.decimated_reads(x, fm.mix_table(rate, f), ddc, reads))
        assert min(lens) < 2 * p.downsample
        want, rl, _ = fac.port_run_seq(port, p, y, lens, return_chunks=True)
        _check(p, got[k], want, rl, f)
    grp.close()
