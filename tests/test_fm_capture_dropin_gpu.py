"""The rx_fm shell in capture mode (RXB200_CAPTURE_RATE) on the replay device: every channel's file must equal the port
run on that channel's decimated stream one block at a time, with the squelch rule and -E zero applied per block, and
match the golden hashes where the shape has them.  The 19-channel FM-band plan builds its decimated streams with
rxb200_ddc_device over the whole capture.  Read lengths do not change the files, and a last partial block is handed on
or dropped by the block rule."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import fm_capture as fcp

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
GOLDEN = os.path.join(HERE, "golden", "fm_capture_golden.json")


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(tmp_path, argv, x, reads=None, rate="40000000", tag="out"):
    cap = tmp_path / "cap.cs16"
    x.tofile(cap)
    dev = f"driver=file,path={cap}" + (f",reads={reads}" if reads else "")
    out = tmp_path / tag
    r = subprocess.run([RX_FM] + argv + ["-d", dev, str(out)], capture_output=True, timeout=600,
                       env=dict(os.environ, RXB200_CAPTURE_RATE=rate))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return out, r.stderr.decode()


def _files(out, freqs):
    return [open(f"{out}.{f}", "rb").read() for f in freqs]


def _expected(port, p, decs, lens, argv):
    """Per channel: the bytes the shell writes, the port's PCM before the squelch, and its squelch hits per read."""
    conseq = int(argv[argv.index("-t") + 1]) if "-t" in argv else 10
    zero = "zero" in argv
    out = []
    for d in decs:
        pcm, rl, hits = fcp.port_channel(port, p, d, lens)
        out.append((fcp.squelched(pcm, rl, hits, conseq, p.squelch_level, zero).tobytes(), pcm, hits))
    return out


@pytest.mark.parametrize("name,zero", [("nbfm_3ch", False), ("am_wav", False), ("squelch_3ch", False),
                                       ("squelch_3ch", True), ("fm2b_f9", False)])
def test_shape_files_equal_the_port(tmp_path, port, name, zero):
    argv, p, freqs, pl, offs, taps, x = fcp.case(name)
    argv = argv + (["-E", "zero"] if zero else [])
    out, err = _run(tmp_path, argv, x, reads="5000:12345:777")
    assert (f"Capture mode: {pl.capture_rate} Hz centred at {pl.centre_hz} Hz, decimation {pl.decim}, "
            f"{pl.n_taps} taps, {len(freqs)} channels") in err
    lens = fcp.chain_reads(fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p)), pl.decim)
    want = _expected(port, p, fcp.decimated(x, pl, offs, taps), lens, argv)
    gold = json.load(open(GOLDEN))[name]
    head = fcp.wav_header(int(fcp.fm.derive_params(offset_tuning=1, **fcp.SHAPES[name][2]).output_rate),
                          p.mode == fcp.fm.MODE_RAW) if "wav" in argv else b""
    n_quiet = 0
    for k, got in enumerate(_files(out, freqs)):
        body, pcm, hits = want[k]
        assert got[:len(head)] == head, (name, k)
        assert got[len(head):] == body, (name, k)
        assert hashlib.sha256(pcm.tobytes()).hexdigest() == gold["channels"][k]["sha256"], (name, k)
        n_quiet += int(p.squelch_level and (hits > 0).any())
    if p.squelch_level:
        assert n_quiet == 2                                   # two of the three channels fall quiet, at different blocks


def test_read_lengths_do_not_change_the_files(tmp_path):
    argv, p, freqs, pl, offs, taps, x = fcp.case("squelch_3ch", seed=3)
    a, _ = _run(tmp_path, argv, x, reads="5000:12345:777", tag="a")
    b, _ = _run(tmp_path, argv, x, reads="131072", tag="b")
    fa, fb = _files(a, freqs), _files(b, freqs)
    assert fa == fb and all(len(f) > 0 for f in fa)


@pytest.mark.parametrize("tail,handed_on", [(16, True), (15, False)])
def test_last_partial_block(tmp_path, port, tail, handed_on):
    """fm2b's -F 9 (P = 3, M = 2): a tail of 16 capture samples decimates to 2^P samples and is handed on; 15 are
    dropped."""
    argv, p, freqs, pl, offs, taps, x = fcp.case("fm2b_f9")
    x = x[:2 * (pl.decim * fcp.CHUNK + tail)]
    blk = fcp.blocks(x.size // 2, pl.decim, fcp.min_chunk(p))
    assert len(blk) == (2 if handed_on else 1)
    out, _ = _run(tmp_path, argv, x, reads="7777")
    lens = fcp.chain_reads(blk, pl.decim)
    for k, got in enumerate(_files(out, freqs)):
        assert got == _expected(port, p, fcp.decimated(x, pl, offs, taps), lens, argv)[k][0], k


def test_fm_band_plan_of_19_wbfm_channels(tmp_path, port):
    import torch
    from rx_tools_b200 import fm
    argv, p, freqs, pl, offs, taps, x = fcp.case("wbfm19")
    assert (len(freqs), pl.decim, pl.capture_rate, pl.n_taps) == (19, 21, 21_420_000, 673)
    out, err = _run(tmp_path, argv, x, reads="100000:33333")
    n = x.size // 2
    lens = fcp.chain_reads(fcp.blocks(n, pl.decim, fcp.min_chunk(p)), pl.decim)
    assert len(lens) == 2
    d_x = torch.from_numpy(x).cuda()
    decs = []
    for o in offs:
        d_y = torch.empty(2 * (n // pl.decim), dtype=torch.int16, device="cuda")
        fm.ddc_device(pl.capture_rate, o, 0, (pl.decim, taps, 15), d_x.data_ptr(), n, d_y.data_ptr())
        torch.cuda.synchronize()
        decs.append(d_y.cpu().numpy())
    want = _expected(port, p, decs, lens, argv)
    for k, got in enumerate(_files(out, freqs)):
        assert got == want[k][0] and len(got) > 0, k
