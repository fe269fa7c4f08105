"""rx_fm parity: the CUDA path (through the C-ABI, host buffers) against the port oracle and the
committed golden vectors.  Integer discriminators must be bit-exact; the atan2 path is compared
byte for byte too, unless the port met a value within 2^-30 of an integer (fm_disc.port_met_near_integer): only then
may CUDA's atan2 truncate differently from glibc's, and the tolerance north_star states applies (1e-5 relative -> at
most 1 LSB on isolated samples)."""
import json
import os

import numpy as np
import pytest

import fm_disc as fd
import oracle
from cases import fm_cases, fm_optional_cases
from rx_tools_b200 import _lib, fm
from rx_tools_b200.synth import digest

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FM_GOLD = json.load(open(os.path.join(G, "fm_golden.json")))


def _compare(case, got, want):
    assert got.size == want.size
    near = fd.port_met_near_integer()
    if case.exact or not near:
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"{bad.size} mismatches, first at {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"
    else:
        # the port met an fp64 atan2 value within 2^-30 of an integer: CUDA's libm and glibc's may truncate it
        # differently, so an isolated sample may be 1 LSB off (north_star tolerance 1e-5 relative on the float path)
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        assert d.max() <= 1, d.max()
        assert np.count_nonzero(d) <= max(1, int(1e-5 * d.size)), np.count_nonzero(d)


@pytest.mark.parametrize("case", fm_cases(), ids=lambda c: c.name)
def test_fm_matches_oracle_and_golden(case, port):
    x = case.make_input()
    want, lens_w, _ = port.fm_run(case.params, x, case.chunk_int16, return_chunks=True)
    d = fm.FmDemod(case.params)
    got, lens = d.full_demod(x, case.chunk_int16, return_chunks=True)
    assert np.array_equal(lens, lens_w)
    _compare(case, got, want)
    if case.exact:
        assert digest(got) == FM_GOLD[case.name]["output_sha256"]
    d.close()


@pytest.mark.parametrize("seg", [64, 256, 4096])
@pytest.mark.parametrize("name", ["cfg2B", "cfg2A", "nbfm_D42_lut", "wbfm_default", "F9_P5_lut", "raw_D4", "zeros_deemph",
                                  "burst_then_silence", "fullscale_noise_P3", "murmur_deemph"])
def test_fm_small_segments(name, seg, port):
    """Tiny segments: every thread boundary falls inside chunks, replay regions overlap chunk starts, and the
    de-emphasis bracket rarely closes -> exercises the serial fix-up."""
    case = next(c for c in fm_cases() if c.name == name)
    x = case.make_input()[: 2 * 98304]
    chunk = 2 * 32768
    want = port.fm_run(case.params, x, chunk)
    d = fm.FmDemod(case.params)
    d.tune(segment_len=seg)
    got = d.full_demod(x, chunk)
    _compare(case, got, want)
    st = d.stats()
    assert st["segment_len"] % 8 == 0 and st["segments"] >= 1
    d.close()


@pytest.mark.parametrize("width", [128, 256])
@pytest.mark.parametrize("name", ["cfg2A", "cfg1_lut", "wbfm_default", "nbfm_D42_lut", "raw_D4"])
def test_fm_boxcar_both_cta_widths(name, width, port, monkeypatch):
    """The boxcar (P = 0) kernels are built for 128- and 256-thread CTAs and the library picks one
    (fm_cta_threads in csrc/fm_kernels.cu); RXB200_FM_THREADS forces one: both must give the reference's bytes."""
    monkeypatch.setenv("RXB200_FM_THREADS", str(width))
    case = next(c for c in fm_cases() if c.name == name)
    x = case.make_input()[: 2 * 262144]
    want = port.fm_run(case.params, x, case.chunk_int16)
    d = fm.FmDemod(case.params)
    got = d.full_demod(x, case.chunk_int16)
    _compare(case, got, want)
    assert d.stats()["segments"] % width == 0
    d.close()


def test_fixup_is_exercised(port):
    case = next(c for c in fm_cases() if c.name == "zeros_deemph")
    x = case.make_input()[: 2 * 262144]
    d = fm.FmDemod(case.params)
    d.tune(segment_len=8192)
    got = d.full_demod(x, 262144)
    assert np.array_equal(got, port.fm_run(case.params, x, 262144))
    assert d.stats()["fixup_segments"] > 0
    d.close()


@pytest.mark.parametrize("name", ["cfg2B", "cfg2A", "nbfm_D42_lut", "cfg5B"])
def test_fm_streaming_calls_carry_state(name, port):
    """Chunk-at-a-time calls (what the drop-in demod thread does) == one call over the whole stream."""
    case = next(c for c in fm_cases() if c.name == name)
    x = case.make_input()[: 2 * 262144]
    chunk = 2 * 32768
    want = port.fm_run(case.params, x, chunk)
    d = fm.FmDemod(case.params)
    parts = [d.full_demod(x[i:i + chunk], chunk) for i in range(0, x.size, chunk)]
    got = np.concatenate(parts)
    _compare(case, got, want)
    d.reset()
    again = d.full_demod(x, chunk)
    _compare(case, again, want)
    d.close()


def test_fm_multichannel(port):
    case = next(c for c in fm_cases() if c.name == "cfg5A")
    from rx_tools_b200 import synth
    n = 1 << 17
    xs = np.stack([synth.cfg5_iq(n, ch) for ch in range(5)])
    d = fm.FmDemod(case.params, n_channels=5)
    got = d.full_demod(xs, 262144)
    for ch in range(5):
        assert np.array_equal(got[ch], port.fm_run(case.params, xs[ch], 262144)), ch
    d.close()


@pytest.mark.parametrize("name,stream", [("cfg2A", True), ("cfg2B", False)])
def test_wbfm_multichannel(name, stream, port, monkeypatch):
    """Several channels through the wbfm kernels: the stream path (front kernel + fm_back_kernel: per-channel PCM scratch,
    items and look-back chains that must not cross a channel) and the split kernel with the row front end."""
    case = next(c for c in fm_cases() if c.name == name)
    if stream:
        monkeypatch.setenv("RXB200_FM_STREAM_MIN", "0")
        monkeypatch.setenv("RXB200_FM_STREAM_PIECE", "700")        # several items per channel
    x = case.make_input()
    n = (x.size // 3 // case.chunk_int16) * case.chunk_int16 or case.chunk_int16
    xs = np.stack([x[:n], x[x.size - n:], np.zeros(n, dtype=np.int16)])           # two different signals and silence
    d = fm.FmDemod(case.params, n_channels=3)
    got = d.full_demod(xs, case.chunk_int16)
    assert d.stats()["kernel_kind"] == (3 if stream else 1)
    for ch in range(3):
        _compare(case, got[ch], port.fm_run(case.params, xs[ch], case.chunk_int16))
    d.close()


def test_scale_identity_on_gpu(port):
    """All 65536 CS16 values through the scale stage (raw mode, D=1, offset tuning = no rotation)."""
    p = oracle.FmParams(mode=oracle.MODE_RAW, downsample=1, offset_tuning=1, rate_out=1000000)
    v = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    x = np.stack([v, v[::-1]], axis=1).reshape(-1)
    d = fm.FmDemod(p)
    got = d.full_demod(x, 2 * 65536)
    assert np.array_equal(got, port.fm_run(p, x, 2 * 65536))
    tab = port.scale_table()
    assert np.array_equal(got[0::2], tab)
    d.close()


def test_ragged_and_bad_shapes_fail_loudly():
    d = fm.FmDemod(fm.FmParams(downsample=8, downsample_passes=3, comp_fir_size=9, custom_atan=1, rate_out=300000))
    x = np.zeros(2 * 1001, dtype=np.int16)          # not a multiple of 16 int16
    with pytest.raises(_lib.Rxb200Error) as e:
        d.full_demod(x, 262144)
    assert e.value.code == _lib.EUNSUPPORTED
    assert d.full_demod(np.zeros(0, dtype=np.int16), 262144).size == 0   # empty input
    d.close()


@pytest.mark.parametrize("case", fm_optional_cases(), ids=lambda c: c.name)
def test_optional_stages(case, port):
    x = case.make_input()
    want = port.fm_run(case.params, x, case.chunk_int16)
    try:
        d = fm.FmDemod(case.params)
    except _lib.Rxb200Error as e:
        assert e.code == _lib.EUNSUPPORTED
        pytest.xfail("per-chunk reduction stages not implemented yet (SURVEY §8f row 2)")
    got = d.full_demod(x, case.chunk_int16)
    _compare(case, got, want)
    d.close()


@pytest.mark.parametrize("case", (fm_cases() + fm_optional_cases())[::2], ids=lambda c: c.name)
def test_levels(case, port):
    """-L statistics input: the rms() of every chunk (src/rtl_fm.c:792-806), and the PCM is unchanged."""
    import dataclasses
    x = case.make_input()
    want_pcm = port.fm_run(case.params, x, case.chunk_int16)
    want_lv = port.fm_levels(case.params, x, case.chunk_int16)
    p = fm.FmParams.from_any(case.params)
    p = dataclasses.replace(p, report_levels=1)
    d = fm.FmDemod(p)
    got = d.full_demod(x, case.chunk_int16)
    lv = d.levels()
    _compare(case, got, want_pcm)
    assert lv.shape == (1, want_lv.size)
    assert np.array_equal(lv[0], want_lv)
    # streaming: two calls, levels are those of the last call only
    d.reset()
    n_chunks = want_lv.size
    if n_chunks >= 2:
        cut = (n_chunks // 2) * case.chunk_int16
        d.full_demod(x[:cut], case.chunk_int16)
        assert np.array_equal(d.levels()[0], want_lv[:n_chunks // 2])
        d.full_demod(x[cut:], case.chunk_int16)
        assert np.array_equal(d.levels()[0], want_lv[n_chunks // 2:])
    d.close()
    # a handle without the switch refuses
    d2 = fm.FmDemod(case.params)
    with pytest.raises(_lib.Rxb200Error):
        d2.levels()
    d2.close()


@pytest.mark.parametrize("seg", [0, 32, 64])
@pytest.mark.parametrize("name", ["cfg2A", "zeros_deemph"])
def test_fused_kernel_on_undecimated_wbfm(name, seg, port, monkeypatch):
    """The undecimated wbfm shape on short-to-medium calls (streaming chunks) runs the fused kernel: per-thread segments,
    then the CTA's first warps run the serial stages.  RXB200_FM_STREAM_MIN above the call length keeps a test-sized call
    off the stream path."""
    case = next(c for c in fm_cases() if c.name == name)
    x = case.make_input()
    monkeypatch.setenv("RXB200_FM_STREAM_MIN", str(x.size // 2 + 1))
    want = port.fm_run(case.params, x, case.chunk_int16)
    d = fm.FmDemod(case.params)
    if seg:
        d.tune(segment_len=seg)
    got = d.full_demod(x, case.chunk_int16)
    _compare(case, got, want)
    assert d.stats()["kernel_kind"] == 0
    # streaming: the carry written by the fused kernel feeds the next call
    d.reset()
    cut = (x.size // 3 // case.chunk_int16) * case.chunk_int16 or case.chunk_int16
    got2 = np.concatenate([d.full_demod(x[:cut], case.chunk_int16), d.full_demod(x[cut:], case.chunk_int16)])
    _compare(case, got2, want)
    d.close()


@pytest.mark.parametrize("shape", [(128, 32), (128, 128), (256, 32), (256, 64)])
@pytest.mark.parametrize("piece", [0, 64, 300])
@pytest.mark.parametrize("name", ["cfg2A", "zeros_deemph", "wbfm_deemph_quiet"])
def test_stream_path_front_kernel_then_back_kernel(name, piece, shape, port, monkeypatch):
    """The undecimated wbfm shape on long calls runs two kernels: the front end of the whole call (PCM to global memory),
    then fm_back_kernel with pieces as long as the call allows.  RXB200_FM_STREAM_MIN=0 selects the path for a test-sized
    call; RXB200_FM_STREAM_PIECE sets the piece length (several items per channel, look-back between them);
    RXB200_FM_STREAM_WIN / _T pick the back kernel's window size and lanes per item."""
    names = [c.name for c in fm_cases()]
    if name not in names:
        pytest.skip("no such case")
    monkeypatch.setenv("RXB200_FM_STREAM_MIN", "0")
    monkeypatch.setenv("RXB200_FM_STREAM_WIN", str(shape[0]))
    monkeypatch.setenv("RXB200_FM_STREAM_T", str(shape[1]))
    if piece:
        monkeypatch.setenv("RXB200_FM_STREAM_PIECE", str(piece))
    case = next(c for c in fm_cases() if c.name == name)
    x = case.make_input()
    want = port.fm_run(case.params, x, case.chunk_int16)
    d = fm.FmDemod(case.params)
    got = d.full_demod(x, case.chunk_int16)
    _compare(case, got, want)
    assert d.stats()["kernel_kind"] == 3
    # streaming: the carry written by the two kernels feeds the next call
    d.reset()
    cut = (x.size // 3 // case.chunk_int16) * case.chunk_int16 or case.chunk_int16
    got2 = np.concatenate([d.full_demod(x[:cut], case.chunk_int16), d.full_demod(x[cut:], case.chunk_int16)])
    _compare(case, got2, want)
    d.close()


def test_row_kernel_is_the_one_that_runs(port):
    case = next(c for c in fm_cases() if c.name == "cfg2B")
    d = fm.FmDemod(case.params)
    d.full_demod(case.make_input(), case.chunk_int16)
    assert d.stats()["kernel_kind"] == 1 and d.stats()["kernel"] == "fm_split_kernel"
    d.close()
