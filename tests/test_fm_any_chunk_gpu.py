"""rx_fm on chunks of any whole number of complex samples (shapes without fifth_order passes) against the port: uniform
chunks that are not multiples of 8 complex with a short last chunk over every mode and optional stage, several channels
of odd length, ragged sequences of calls with the squelch hits and -L levels after each, the device entry point from a
4-byte (not 16-byte) aligned input that ends where its allocation ends, the golden hashes of the reference, a seeded
sweep, the kernels that calls of whole 8-sample blocks keep, the refusals that stay, and rx_fm_b200 reading a device
that returns packets of odd lengths."""
import hashlib
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

import fm_any_chunk as fac
import oracle
from rx_tools_b200 import _lib, fm, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
GOLDEN = os.path.join(HERE, "golden", "fm_any_chunk_golden.json")
SHAPES = fac.shapes()


def _input(p, n_complex, seed):
    return fac.loud_quiet(n_complex, seed) if p.squelch_level else fac.signal(n_complex, seed)


def _compare(p, got, want, what):
    assert got.size == want.size, (what, got.size, want.size)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    if fac.INTEGER(p):
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    else:
        # every sample through fp64 atan2 (CUDA libm vs glibc): a last-ulp difference may move an isolated sample by
        # 1 LSB, and the serial stages after it may smear such a flip over a few outputs
        assert np.count_nonzero(diff) <= max(2, int(1e-4 * diff.size)), (what, np.flatnonzero(diff)[:5])
        if not p.deemph and p.rate_out2 <= 0 and not p.dc_block_audio:
            assert diff.max(initial=0) <= 1, what


def _levels_handle(p):
    q = fm.FmParams.from_any(p)
    q.report_levels = 1
    return fm.FmDemod(q)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_uniform_odd_chunks(name, port):
    p = SHAPES[name]
    d = fm.FmDemod(p)
    for i, c in enumerate((1001, 4093, 131071)):
        n = (3 if c > 5000 else 9) * c + 2 * p.downsample + 5 * i + 1         # a short last chunk
        x = _input(p, n, 20 + i)
        want, wl, wh = port.fm_run(p, x, 2 * c, return_chunks=True)
        d.reset()
        got, gl = d.full_demod(x, 2 * c, return_chunks=True)
        assert d.stats()["kernel_kind"] == 0
        assert np.array_equal(gl, wl), (name, c)
        _compare(p, got, want, (name, c))
        if p.squelch_level:
            assert d.squelch_hits()[0] == wh[-1]
    d.close()


@pytest.mark.parametrize("name", ["fm_lut_d100", "fm_fast_d1_deemph181", "fm_lut_d42_squelch", "am_d42_rdc_adc", "raw",
                                  "fm_ale_d8_adc"])
def test_channels_of_odd_length(name, port):
    p = SHAPES[name]
    n_ch, n, c = 3, 3 * 2003 + 457, 2003
    x = np.stack([_input(p, n, 60 + k) for k in range(n_ch)])
    d = fm.FmDemod(p, n_channels=n_ch)
    got = d.full_demod(x, 2 * c)
    for k in range(n_ch):
        _compare(p, got[k], port.fm_run(p, x[k], 2 * c), (name, k))
    d.close()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_ragged_call_sequences(name, port):
    """One call per chunk, each of its own length, the handle carrying the state: the PCM, the squelch hits after every
    call, and -L's level of every call."""
    p = SHAPES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    lens = fac.ragged_lens(rng, 12, 2 * p.downsample, 5000)
    lens[3] = 2 * 8 * (p.downsample + 1)                      # one whole number of 8-sample blocks among them
    x = _input(p, fac.seq_len(lens), 70)
    want, wl, wh = fac.port_run_seq(port, p, x, lens, return_chunks=True)
    want_lv = fac.port_levels_seq(port, p, x, lens)
    d, dl = fm.FmDemod(p), _levels_handle(p)        # report_levels selects the reduction-stage kernel: a second handle
    parts, parts_l = [], []
    for c, (pos, n) in enumerate(fac.seq_bounds(x.size, lens)):
        parts.append(d.full_demod(x[pos:pos + n], n))
        parts_l.append(dl.full_demod(x[pos:pos + n], n))
        assert parts[-1].size == wl[c] and parts_l[-1].size == wl[c], (name, c)
        assert dl.levels()[0].tolist() == [want_lv[c]], (name, c)
        if p.squelch_level:
            assert d.squelch_hits()[0] == wh[c] and dl.squelch_hits()[0] == wh[c], (name, c)
    _compare(p, np.concatenate(parts), want, name)
    _compare(p, np.concatenate(parts_l), want, (name, "levels"))
    d.close()
    dl.close()


def test_device_entry_at_4_byte_alignment(port):
    """Odd n, two channels, the input 4 bytes into its allocation and ending where the allocation ends: the partial
    last block of the last channel is read up to the last sample and no further."""
    import torch
    p = SHAPES["fm_fast_d1_deemph181"]
    n_ch, n, c = 2, 5 * 10007 + 3, 10007
    x = np.stack([_input(p, n, 90 + k) for k in range(n_ch)])
    buf = torch.zeros(x.size + 2, dtype=torch.int16, device="cuda")
    buf[2:] = torch.from_numpy(x.reshape(-1)).cuda()
    dx = buf[2:]
    assert dx.data_ptr() % 16 == 4
    d = fm.FmDemod(p, n_channels=n_ch)
    cap = d.max_output(2 * n, 2 * c) + 8
    out = torch.zeros(n_ch * cap, dtype=torch.int16, device="cuda")
    n_pcm = d.process_device(dx.data_ptr(), 2 * n, 2 * c, out.data_ptr(), cap, sync=True)
    got = out.view(n_ch, cap)[:, :n_pcm].cpu().numpy()
    for k in range(n_ch):
        _compare(p, got[k], port.fm_run(p, x[k], 2 * c), k)
    # calls of whole blocks keep the 32-byte alignment rule
    with pytest.raises(_lib.Rxb200Error) as e:
        d.process_device(buf[8:8 + 2 * n_ch * 8000].data_ptr(), 2 * 8000, 2 * 8000, out.data_ptr(), cap)
    assert e.value.code == _lib.EINVAL
    d.close()


def test_golden_hashes(port):
    gold = json.load(open(GOLDEN))
    for name, (p, x, lens) in sorted(fac.golden_cases().items()):
        g = gold[name]
        d = fm.FmDemod(p)
        if len(lens) == 1:
            got, rl = d.full_demod(x, lens[0], return_chunks=True)
            assert d.stats()["kernel_kind"] == 0, name
        else:
            parts, rl = [], []
            for pos, n in fac.seq_bounds(x.size, lens):
                parts.append(d.full_demod(x[pos:pos + n], n))
                rl.append(parts[-1].size)
            got = np.concatenate(parts)
        d.close()
        assert list(rl) == g["result_len"], name
        if fac.INTEGER(p):
            assert hashlib.sha256(got.tobytes()).hexdigest() == g["sha256"], name
        else:
            _compare(p, got, fac.port_run_seq(port, p, x, lens), name)


def _random_case(rng):
    mode = int(rng.choice([0, 0, 0, 1, 2, 3, 4]))
    D = int(rng.choice([1, 2, 3, 6, 7, 10, 42, 100, 257]))
    p = dict(mode=mode, downsample=D, custom_atan=int(rng.integers(0, 4)), output_scale=int(rng.choice([1, 4, 64])),
             offset_tuning=int(rng.random() < 0.3))
    rate_out = int(rng.choice([24000, 48000, 170000, 300000, 1000000]))
    p["rate_out"] = rate_out
    if rng.random() < 0.6 and mode != 4:
        p["rate_out2"] = int(rate_out // rng.choice([1, 2, 3, 5, 6]) - rng.integers(0, 50))
    if rng.random() < 0.6:
        p["deemph"] = 1
        p["deemph_a"] = int(rng.choice([1, 2, 7, 13, 16, 23, 64, 77, 181, 300]))
    opt = rng.random()
    if opt < 0.15:
        p["squelch_level"] = int(rng.choice([5, 40, 200]))
    elif opt < 0.3:
        p["dc_block_raw"] = 1
        p["rdc_block_const"] = int(rng.choice([1, 9, 30]))
    elif opt < 0.45:
        p["dc_block_audio"] = 1
    # any chunk length, down to one sample when no per-chunk stage is on (such a stage refuses a chunk that decimates
    # to nothing); a stream with a shorter last chunk
    lo = D if "squelch_level" in p or "dc_block_raw" in p or "dc_block_audio" in p else 1
    chunk_c = int(rng.integers(lo, min(131072, D * int(rng.integers(2, 400))) + 1))
    n_chunks = int(rng.integers(2, 9))
    tail = int(rng.integers(lo, chunk_c + 1))
    return oracle.FmParams(**p), chunk_c, (n_chunks - 1) * chunk_c + tail


@pytest.mark.parametrize("seed", range(40))
def test_random_configuration_any_chunk(seed, port):
    rng = np.random.default_rng(5000 + seed)
    p, chunk_c, n_c = _random_case(rng)
    x = synth.uniform_iq(n_c, -3000, 3000, seed) if rng.random() < 0.3 else _input(p, n_c, seed)
    want, wl, wh = port.fm_run(p, x, 2 * chunk_c, return_chunks=True)
    d = fm.FmDemod(p)
    if rng.random() < 0.5:
        d.tune(segment_len=int(rng.choice([0, 64, 256, 1024])))
    try:
        if rng.random() < 0.5:
            got, gl = d.full_demod(x, 2 * chunk_c, return_chunks=True)
            assert np.array_equal(gl, wl)
        else:       # split into calls on chunk boundaries: carry across calls
            cuts = sorted(set(int(c) * 2 * chunk_c for c in rng.integers(1, max(2, x.size // (2 * chunk_c) + 1), size=2)))
            parts, pos = [], 0
            for c in cuts + [x.size]:
                if c > pos:
                    parts.append(d.full_demod(x[pos:c], 2 * chunk_c))
                    pos = c
            got = np.concatenate(parts)
    except _lib.Rxb200Error as e:
        if e.code == _lib.EUNSUPPORTED:         # a de-emphasis warm-up longer than a CTA's PCM buffer holds
            pytest.skip(f"shape not supported: {e}")
        raise
    _compare(p, got, want, (vars(p), chunk_c, n_c))
    if p.squelch_level:
        assert d.squelch_hits()[0] == wh[-1]
    d.close()


def test_whole_block_calls_keep_their_kernels():
    """Calls of whole 8-sample blocks keep the stream path, the row kernel and the specialised fused kernels; the same
    shapes one sample off take the any-length kernel (kernel_kind 0)."""
    fm2a = fm.FmParams.from_any(fac.FM2A)
    x = synth.cfg2_iq(1 << 20)
    d = fm.FmDemod(fm2a)
    d.full_demod(x, 262144)
    assert d.stats()["kernel_kind"] == 3
    d.reset()
    d.full_demod(x, 262142)
    assert d.stats()["kernel_kind"] == 0
    d.close()
    fm2b = fm.derive_params(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9).params
    d = fm.FmDemod(fm2b)
    d.full_demod(x, 262144)
    assert d.stats()["kernel_kind"] == 1
    d.close()


@pytest.mark.parametrize("P", [1, 3, 6])
def test_passes_keep_their_granule(P):
    """With fifth_order passes a chunk stays a multiple of max(16, 2 * 2^P) int16, the last one included."""
    p = fm.FmParams(downsample=1 << P, downsample_passes=P, custom_atan=fm.ATAN_FAST, rate_out=300000)
    d = fm.FmDemod(p)
    x = fac.signal(4 * 1024, 3)
    g = max(16, 2 << P)
    for n16, chunk in ((x.size, 2002), (x.size - 2, 2048), (x.size, g + 2)):
        with pytest.raises(_lib.Rxb200Error) as e:
            d.full_demod(x[:n16], chunk)
        assert e.value.code == _lib.EUNSUPPORTED, (n16, chunk)
    assert d.full_demod(x, 2048).size > 0
    d.close()


def test_refusals_that_stay(port):
    p = fm.FmParams.from_any(SHAPES["fm_lut_d42_squelch"])
    d = fm.FmDemod(p)
    x = fac.signal(4000, 1)
    for n16, chunk in ((x.size - 1, 2000), (x.size, 2001), (x.size, 262146)):       # half a complex sample; too long
        with pytest.raises(_lib.Rxb200Error) as e:
            d.full_demod(x[:n16], chunk)
        assert e.value.code == _lib.EUNSUPPORTED, (n16, chunk)
    with pytest.raises(_lib.Rxb200Error) as e:        # a chunk with no decimated sample: 1000 = 23 x 42 + 34, then 4
        d.full_demod(x[:2 * 1000 + 2 * 4], 2 * 1000)
    assert e.value.code == _lib.EUNSUPPORTED
    d.close()
    q = fm.FmParams(downsample=4, custom_atan=fm.ATAN_FAST, rate_out=100000, post_downsample=2)
    d = fm.FmDemod(q)
    with pytest.raises(_lib.Rxb200Error) as e:                                      # -o 2, a chunk of 5 boxcars
        d.full_demod(x[:2 * 200], 2 * 20)
    assert e.value.code == _lib.EUNSUPPORTED
    assert d.full_demod(x[:2 * 200], 2 * 24).size > 0                               # 3 complex blocks, 6 boxcars
    d.close()


# ---- rx_fm_b200 over a device that reads in packets of odd lengths
READS = [1021, 333, 4093]


@pytest.fixture(scope="module")
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, timeout=300)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r


SHORT_READS = [1021, 5, 333, 17, 41, 4093]      # reads of 5, 17 and 41 samples complete no boxcar at D = 42


def _capture(tmp_path, x, reads=READS):
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    return f"driver=file,path={cap},reads={':'.join(map(str, reads))}"


def _stream(n_complex, seed, reads=READS):
    # whole cycles of reads plus a last read that still holds two boxcars
    n = (n_complex // sum(reads)) * sum(reads) + 611
    return fac.signal(n, seed)


def _dropin_equals_port(tmp_path, port, args, p, reads):
    x = _stream(120_000, 5, reads)
    out = tmp_path / "out.raw"
    _run([RX_FM, "-f", "100M", "-d", _capture(tmp_path, x, reads)] + args + [str(out)])
    want = fac.port_run_seq(port, p, x, [2 * r for r in reads])
    got = np.fromfile(out, dtype=np.int16)
    assert got.size == want.size
    assert np.array_equal(got, want)


@pytest.mark.parametrize("args,p", [
    (["-M", "fm", "-s", "24k", "-A", "lut"], fac.FM24K_LUT),
    (["-M", "wbfm"], fac.WBFM),
    (["-M", "am"], fac.AM),
    (["-M", "raw"], fac.RAW),
])
def test_dropin_reads_of_odd_lengths(tmp_path, port, built, args, p):
    _dropin_equals_port(tmp_path, port, args, p, READS)


@pytest.mark.parametrize("args,p", [
    (["-M", "fm", "-s", "24k", "-A", "lut"], fac.FM24K_LUT),
    (["-M", "wbfm"], fac.WBFM),
])
def test_dropin_reads_shorter_than_the_boxcar(tmp_path, port, built, args, p):
    """Without -o, passes or a per-chunk stage every read is handed on as it came, reads too short to complete a
    boxcar included."""
    _dropin_equals_port(tmp_path, port, args, p, SHORT_READS)


def test_dropin_level_printing_per_read(tmp_path, port, built):
    x = np.concatenate([_stream(60_000, 6), fac.signal(20_000, 7, quiet=True)])
    x = x[:2 * ((x.size // 2 - 611) // sum(READS) * sum(READS) + 611)]
    out = tmp_path / "out.raw"
    r = _run([RX_FM, "-f", "100M", "-M", "am", "-L", "3", "-d", _capture(tmp_path, x), str(out)])
    lens = [2 * v for v in READS]
    lv = fac.port_levels_seq(port, fac.AM, x, lens)
    want_lines, no, lsum, lmax, lmaxmax = [], 1, 0.0, 0, 0
    for sr in lv:
        no -= 1
        lsum += int(sr); lmax = max(lmax, int(sr)); lmaxmax = max(lmaxmax, int(sr))
        if no == 0:
            no = 3
            want_lines.append("%f, %d, %d, %d" % (lsum / 3, lmax, lmaxmax, 0))
            lmax, lsum = 0, 0.0
    got_lines = [ln for ln in r.stderr.decode().splitlines() if ln.count(",") == 3 and ln[0].isdigit()]
    assert len(want_lines) >= 10
    assert got_lines == want_lines
    assert np.array_equal(np.fromfile(out, dtype=np.int16), fac.port_run_seq(port, fac.AM, x, lens))


def test_dropin_squelch_zero_per_read(tmp_path, port, built):
    loud = fac.signal(30 * sum(READS), 8)
    quiet = fac.signal(30 * sum(READS) + 611, 9, quiet=True)
    x = np.concatenate([loud, quiet])
    out = tmp_path / "out.raw"
    _run([RX_FM, "-f", "100M", "-M", "fm", "-s", "24k", "-A", "lut", "-l", "60", "-t", "1", "-E", "zero",
          "-d", _capture(tmp_path, x), str(out)])
    p = fac.with_(fac.FM24K_LUT, squelch_level=60)
    want, lens, hits = fac.port_run_seq(port, p, x, [2 * r for r in READS], return_chunks=True)
    pos = 0
    for n, h in zip(lens, hits):            # squelch active (hits > conseq_squelch) with -E zero writes zeros
        if h > 1:
            want[pos:pos + n] = 0
        pos += n
    assert np.any(hits > 1) and np.any(hits == 0), "the squelch never closed or never opened"
    assert np.array_equal(np.fromfile(out, dtype=np.int16), want)
