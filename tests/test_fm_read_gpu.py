"""rxb200_fm_process_read with fifth_order passes against the port: read sequences that meet every residue of the read
length with the squelch hits and -L level after each read, a seeded sweep, several channels, the device entry point at
4-byte alignment ending where its allocation ends, reads on the read kernel followed on one handle by calls of the row
and fused kernels and the reverse, the golden hashes of the reference, refusals that leave the state alone, and
rx_fm_b200 -M wbfm -s 300k -F 9 -r 48k over a device that returns reads of other lengths than the passes' granule."""
import hashlib
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_disc as fd
import fm_read as frd
import oracle
from rx_tools_b200 import _lib, fm, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
GOLDEN = os.path.join(HERE, "golden", "fm_read_golden.json")
SHAPES = frd.shapes()


def _compare(p, got, want, what):
    assert got.size == want.size, (what, got.size, want.size)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    near = fd.port_met_near_integer()
    if fac.INTEGER(p) or not near:
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    else:       # the port met an atan2 value within 2^-30 of an integer: CUDA's libm may truncate it the other way
        assert np.count_nonzero(diff) <= max(2, int(1e-4 * diff.size)), (what, np.flatnonzero(diff)[:5])


def _off_granule(n16, p_):
    return n16 % max(16, 2 << p_) != 0


def _run_reads(d, x, lens, check=None):
    parts = []
    for c, (pos, n) in enumerate(fac.seq_bounds(x.size, lens)):
        parts.append(d.process_read(x[pos:pos + n]))
        if _off_granule(n, d.params.downsample_passes):
            assert d.stats()["kernel_kind"] == 0
        if check:
            check(c, parts[-1])
    return np.concatenate(parts)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_read_sequences(name, port):
    """One read per call, each of its own length: the PCM, and after every read its length, the squelch hits and the
    -L level (a second handle with report_levels)."""
    p = SHAPES[name]
    lens = frd.read_lens(p.downsample_passes, zlib.crc32(name.encode()), even_dec=p.post_downsample > 1)
    x = frd.stream_for(lens, 30, quiet_half=bool(p.squelch_level))
    want, wl, wh = fac.port_run_seq(port, p, x, lens, return_chunks=True)
    want_lv = fac.port_levels_seq(port, p, x, lens)
    q = fm.FmParams.from_any(p)
    q.report_levels = 1
    d, dl = fm.FmDemod(p), fm.FmDemod(q)

    def check(c, part):
        assert part.size == wl[c], (name, c)
        if p.squelch_level:
            assert d.squelch_hits()[0] == wh[c], (name, c)

    got = _run_reads(d, x, lens, check)
    got_l = []
    for c, (pos, n) in enumerate(fac.seq_bounds(x.size, lens)):
        got_l.append(dl.process_read(x[pos:pos + n]))
        assert dl.levels()[0].tolist() == [want_lv[c]], (name, c)
        if p.squelch_level:
            assert dl.squelch_hits()[0] == wh[c], (name, c)
    _compare(p, got, want, name)
    _compare(p, np.concatenate(got_l), want, (name, "levels"))
    d.close()
    dl.close()


def _random_case(rng):
    p_ = int(rng.integers(1, 11))
    mode = int(rng.choice([0, 0, 0, 1, 2, 3, 4]))
    kw = dict(mode=mode, custom_atan=int(rng.integers(0, 4)), output_scale=int(rng.choice([1, 4])),
              offset_tuning=int(rng.random() < 0.3))
    if rng.random() < 0.5 and mode != 4:
        kw["rate_out2"] = int(kw.get("rate_out", max(24000, 2400000 >> p_)) // rng.choice([1, 2, 3, 5]))
    if rng.random() < 0.4:
        kw["deemph"], kw["deemph_a"] = 1, int(rng.choice([1, 2, 7, 13, 16, 23, 64]))
    opt = rng.random()
    if opt < 0.15:
        kw["squelch_level"] = int(rng.choice([5, 40, 200]))
    elif opt < 0.3:
        kw["dc_block_raw"], kw["rdc_block_const"] = 1, int(rng.choice([1, 9, 30]))
    elif opt < 0.45:
        kw["dc_block_audio"] = 1
    return frd.passes(p_, fir=bool(rng.random() < 0.7), **kw)


@pytest.mark.parametrize("seed", range(24))
def test_random_read_sequences(seed, port):
    rng = np.random.default_rng(7000 + seed)
    p = _random_case(rng)
    lens = frd.read_lens(p.downsample_passes, seed, n_extra=int(rng.integers(2, 12)))
    x = frd.stream_for(lens, seed) if rng.random() < 0.7 else synth.uniform_iq(sum(lens) // 2, -3000, 3000, seed)
    want = fac.port_run_seq(port, p, x, lens)
    d = fm.FmDemod(p)
    if rng.random() < 0.5:
        d.tune(segment_len=int(rng.choice([0, 1024, 4096])))
    try:
        got = _run_reads(d, x, lens)
    except _lib.Rxb200Error as e:
        if e.code == _lib.EUNSUPPORTED:         # a de-emphasis warm-up longer than a CTA's PCM buffer holds
            pytest.skip(f"shape not supported: {e}")
        raise
    _compare(p, got, want, (vars(p), lens))
    d.close()


@pytest.mark.parametrize("n_ch", [1, 2, 3, 4])
def test_channels(n_ch, port):
    p = SHAPES["fm_lut_p4_fir"] if n_ch % 2 else frd.FM2B
    lens = [2 * 1021, 2 * 333, 2 * 4093, 2 << p.downsample_passes, 2 * 2044]
    xs = [frd.stream_for(lens, 40 + k) for k in range(n_ch)]
    d = fm.FmDemod(p, n_channels=n_ch)
    parts = []
    for pos, n in fac.seq_bounds(xs[0].size, lens):
        parts.append(d.process_read(np.stack([x[pos:pos + n] for x in xs])))
    got = np.concatenate(parts, axis=1)
    for k in range(n_ch):
        _compare(p, got[k], fac.port_run_seq(port, p, xs[k], lens), (n_ch, k))
    d.close()


def test_device_entry_at_4_byte_alignment(port):
    """Two channels of an off-granule read, 4 bytes into the allocation and ending where it ends; then a read of whole
    rows at that alignment (the any-length kernel, not the row kernel), and the same read 32-byte aligned."""
    import torch
    p = frd.FM2B
    n_ch = 2
    for n in (4093, 8192):
        x = np.stack([frd.stream_for([2 * n], 90 + k) for k in range(n_ch)])
        buf = torch.zeros(x.size + 2, dtype=torch.int16, device="cuda")
        buf[2:] = torch.from_numpy(x.reshape(-1)).cuda()
        dx = buf[2:]
        assert dx.data_ptr() % 16 == 4
        d = fm.FmDemod(p, n_channels=n_ch)
        cap = d.max_output(2 * n, 2 * n) + 8
        out = torch.zeros(n_ch * cap, dtype=torch.int16, device="cuda")
        n_pcm = d.process_read_device(dx.data_ptr(), 2 * n, out.data_ptr(), cap, sync=True)
        assert d.stats()["kernel_kind"] == 0
        got = out.view(n_ch, cap)[:, :n_pcm].cpu().numpy()
        for k in range(n_ch):
            _compare(p, got[k], port.fm_run(p, x[k], 2 * n), (n, k))
        d.close()
    with pytest.raises(_lib.Rxb200Error) as e:
        d = fm.FmDemod(p)
        d.process_read_device(buf.data_ptr() + 2, 2 * 4093, out.data_ptr(), cap)
    assert e.value.code == _lib.EINVAL


def test_read_kernel_then_row_and_fused_kernels(port):
    """A desynchronised I/Q window, a swapped fm_demod carry and an unequal droop history go from the read kernel into
    the row kernel (kernel_kind 1) and the fused kernel on one handle, and back."""
    p = frd.FM2B
    x = synth.cfg2_iq(1 << 20)
    for lens in ([2 * 4093, 2 * 131072, 2 * 333, 2 * 4096, 2 * 1021],          # read, rows, read, fused, read
                 [2 * 131072, 2 * 4096, 2 * 2045, 2 * 131072, 2 * 4096]):      # rows, fused, read, rows, fused
        n = sum(lens)
        want = fac.port_run_seq(port, p, x[:n], lens)
        d = fm.FmDemod(p)
        parts, kinds = [], []
        for pos, m in fac.seq_bounds(n, lens):
            parts.append(d.process_read(x[pos:pos + m]))
            kinds.append(d.stats()["kernel_kind"])
        assert kinds == [1 if m == 2 * 131072 else 0 for m in lens], kinds
        _compare(p, np.concatenate(parts), want, lens)
        d.close()
    # the generic passes: the packed SPEC 0 kernel after the read kernel, P = 5 (three packed levels, two scalar)
    q = SHAPES["fm_fast_p5_fir"]
    lens = [2 * 1001, 2 * 4096, 2 * 999, 2 * 2048]
    want = fac.port_run_seq(port, q, x[:sum(lens)], lens)
    d = fm.FmDemod(q)
    got = np.concatenate([d.process_read(x[pos:pos + m]) for pos, m in fac.seq_bounds(sum(lens), lens)])
    _compare(q, got, want, "p5")
    d.close()


def test_golden_hashes(port):
    gold = json.load(open(GOLDEN))
    for name, (p, x, lens) in sorted(frd.golden_cases().items()):
        g = gold[name]
        d = fm.FmDemod(p)
        parts = [d.process_read(x[pos:pos + n]) for pos, n in fac.seq_bounds(x.size, lens)]
        d.close()
        assert [v.size for v in parts] == g["result_len"] or p.mode == fac.M_RAW, name
        got = np.concatenate(parts)
        if fac.INTEGER(p):
            assert hashlib.sha256(got.tobytes()).hexdigest() == g["sha256"], name
        else:
            _compare(p, got, fac.port_run_seq(port, p, x, lens), name)


def test_refusals_leave_the_state_alone(port):
    p = SHAPES["fm_lut_p4_squelch"]
    lens = [2 * 1001, 2 * 777]
    x = frd.stream_for(lens, 3)
    want, _, wh = fac.port_run_seq(port, p, x, lens, return_chunks=True)
    d = fm.FmDemod(p)
    a = d.process_read(x[:lens[0]])
    for bad in (x[lens[0]:lens[0] + 31], x[lens[0]:lens[0] + 30], np.zeros(262146, dtype=np.int16)):
        with pytest.raises(_lib.Rxb200Error) as e:        # half a complex sample; under 2^P complex; too long
            d.process_read(bad)
        assert e.value.code == _lib.EUNSUPPORTED
    h = fm.FmDemod(fm.FmParams.from_any(frd.passes(2, post_downsample=2)))
    with pytest.raises(_lib.Rxb200Error) as e:            # -o 2 and a read of 5 decimated samples
        h.process_read(x[:2 * 21])
    assert e.value.code == _lib.EUNSUPPORTED
    h.close()
    b = d.process_read(x[lens[0]:])
    assert d.squelch_hits()[0] == wh[-1]
    _compare(p, np.concatenate([a, b]), want, "after refusals")
    d.close()
    # rxb200_fm_process keeps its granule with passes
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmDemod(frd.FM2B).full_demod(x[:2 * 1001], 2 * 1001)
    assert e.value.code == _lib.EUNSUPPORTED


# ---- rx_fm_b200 -M wbfm -s 300k -F 9 -r 48k over a device that reads in packets
@pytest.fixture(scope="module")
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


@pytest.mark.parametrize("reads", [[1021, 333, 4093], [2044]])
@pytest.mark.parametrize("levels", [False, True])
def test_dropin_fm2b_reads(tmp_path, port, built, reads, levels):
    x = synth.cfg2_iq(200_000 // sum(reads) * sum(reads) + 611)
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    out = tmp_path / "out.raw"
    dev = f"driver=file,path={cap},reads={':'.join(map(str, reads))}"
    cmd = [RX_FM, "-f", "100M", "-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k"] + (["-L", "3"] if levels else [])
    r = subprocess.run(cmd + ["-d", dev, str(out)], capture_output=True, timeout=300)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    lens = [2 * v for v in reads]
    want = fac.port_run_seq(port, frd.FM2B, x, lens)
    got = np.fromfile(out, dtype=np.int16)
    assert got.size == want.size
    assert np.count_nonzero(got != want) == 0
    if levels:
        lv = fac.port_levels_seq(port, frd.FM2B, x, lens)
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
