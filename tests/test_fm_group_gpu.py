"""rx_fm on several GPUs through one group handle (rxb200_fm_group_*): the group's PCM, chunk result lengths, squelch hits
and -L levels equal those of ONE handle with every channel, after every call of a sequence that mixes process,
process_read and reset; the port checks a subset of the channels.  The shapes reach every kernel the single handle
runs.  Members repeat ordinal 0, so one H100 runs the whole group; the same cases run on distinct ordinals where the box
has that many GPUs.  Refused calls leave every member's carry where it was, and the caller's current device stays."""
import ctypes as C

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_read as frd
from rx_tools_b200 import _lib, fm, sharding

pytestmark = pytest.mark.gpu


def _n_gpus():
    return int(_lib.lib().rxb200_device_count())


LAYOUTS = [("same", [0, 0]), ("same", [0, 0, 0]), ("same", [0, 0, 0, 0]),
           ("distinct", [0, 1]), ("distinct", [0, 1, 2]), ("distinct", [0, 1, 2, 3])]
LAYOUT_IDS = [f"{k}-{len(d)}" for k, d in LAYOUTS]


def _devices(layout):
    kind, devs = layout
    if _n_gpus() < max(devs) + 1:
        pytest.skip(f"needs {max(devs) + 1} GPUs")
    return devs


def _with_levels(p):
    q = fm.FmParams.from_any(p)
    q.report_levels = 1
    return q


SQUELCH = fac.with_(fac.FM24K_LUT, squelch_level=60)

# name -> (parameters, "process" or "read", chunk int16, the calls' lengths in int16, kernel_kind every handle reports,
# input of one channel)
CASES = {
    # the split kernel with the row front end (fm2b shape): whole rows, 32 rows per call
    "rows": (frd.FM2B, "process", 8 * 2048, [2 * 32768, 2 * 32768], 1, fac.signal),
    # the stream path (fm2a shape): a call long enough for a member with a single channel
    "stream": (fac.FM2A, "process", 32768, [2 * 98304, 2 * 98304], 3, fac.signal),
    # the SPEC 3 fused kernel (fm5a shape): whole 8-sample blocks
    "spec3": (fac.FM5A, "process", 2 * 25000, [2 * 50000, 2 * 25000], 0, fac.signal),
    # the any-length kernel without passes: odd chunks, a short last chunk
    "any": (fac.FM5A, "process", 2 * 2003, [2 * 3 * 2003, 2 * (2 * 2003 + 457)], 0, fac.signal),
    # reads off the passes' granule (fm2b shape through process_read)
    "read_passes": (frd.FM2B, "read", 0, [2 * 1021, 2 * 333, 2 * 4093], 0, fac.signal),
    # per-chunk reduction stages: squelch and -L levels
    "squelch_levels": (_with_levels(SQUELCH), "process", 2 * 2003, [2 * 4 * 2003, 2 * (2003 + 457)], 0, fac.loud_quiet),
}


def _hits(d):
    h = np.zeros(d.n_channels, dtype=np.int32)
    _lib.check(_lib.lib().rxb200_fm_squelch_hits(d._h, h.ctypes.data_as(C.POINTER(C.c_int))))
    return h


def _member_kinds(g):
    kinds = []
    for i in range(g.n_dev):
        h = g.member(i)
        if h:
            s = _lib.FmStatsC()
            _lib.check(_lib.lib().rxb200_fm_last_stats(C.c_void_p(h), C.byref(s)))
            kinds.append(s.kernel_kind)
    return kinds


def _call(obj, mode, x, chunk):
    """One call on a FmDemod or a FmGroup: (pcm, chunk result lengths or None)."""
    if mode == "read":
        return obj.process_read(x), None
    return obj.full_demod(x, chunk, return_chunks=True)


def _same_as_single(g, d, mode, x, chunk, what):
    """One call on both; everything the group reports equals the single handle's."""
    got, gl = _call(g, mode, x, chunk)
    want, wl = _call(d, mode, x, chunk)
    assert got.shape == want.shape and got.tobytes() == want.tobytes(), what
    if wl is not None:
        assert gl.tolist() == wl.tolist(), what
    assert g.squelch_hits().tolist() == _hits(d).tolist(), what
    if g.params.report_levels:
        assert g.levels().tolist() == d.levels().tolist(), what
    return got


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_paths_match_one_handle_and_port(name, layout, port):
    devices = _devices(layout)
    p, mode, chunk, lens, kind, make = CASES[name]
    n_ch = 5
    x = np.stack([make(sum(lens) // 2, 100 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    parts, pos = [], 0
    for c, n in enumerate(lens):
        parts.append(_same_as_single(g, d, mode, x[:, pos:pos + n], chunk, (name, c)))
        assert _member_kinds(g) == [kind] * len(_member_kinds(g)), (name, c, _member_kinds(g))
        assert d.stats()["kernel_kind"] == kind, (name, c)
        pos += n
    got = np.concatenate(parts, axis=1)
    q = fm.FmParams.from_any(p)
    op = fac.P(**q.reference_fields())
    for k in (0, n_ch - 1):
        if mode == "read":
            want, _, wh = fac.port_run_seq(port, op, x[k], lens, return_chunks=True)
        else:
            want, _, wh = port.fm_run(op, x[k], chunk, return_chunks=True)
        assert got[k].tobytes() == want.tobytes(), (name, k)
        assert g.squelch_hits()[k] == wh[-1], (name, k)
    g.close()
    d.close()


@pytest.mark.parametrize("kind", ["same", "distinct"])
@pytest.mark.parametrize("n_dev", [2, 3, 4])
@pytest.mark.parametrize("n_ch", [1, 3, 5, 7])
def test_channel_counts_and_empty_members(n_ch, n_dev, kind):
    devices = _devices((kind, [0] * n_dev if kind == "same" else list(range(n_dev))))
    p, _, chunk, lens, _, make = CASES["any"]
    x = np.stack([make(sum(lens) // 2, 200 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    assert _lib.lib().rxb200_fm_group_size(g._g) == n_dev
    for i in range(n_dev):
        b, e = sharding.unit_range(i, n_dev, n_ch)
        assert (g.member(i) == 0) == (e == b), (n_ch, n_dev, i)
    assert g.member(n_dev) == 0 and g.member(-1) == 0
    d = fm.FmDemod(p, n_channels=n_ch)
    pos = 0
    for c, n in enumerate(lens):
        _same_as_single(g, d, "process", x[:, pos:pos + n], chunk, (n_ch, n_dev, c))
        pos += n
    g.close()
    d.close()


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
def test_mixed_call_sequence_then_reset(layout):
    """process and process_read calls of several lengths on one group, reset, and the sequence again: chunk result
    lengths, squelch hits and levels after every call."""
    devices = _devices(layout)
    p = CASES["squelch_levels"][0]
    n_ch = 7
    calls = [("process", 2 * 2003, 2 * 3 * 2003), ("read", 0, 2 * 1777), ("process", 2 * 4096, 2 * 8 * 4096),
             ("read", 0, 2 * 5003), ("process", 2 * 999, 2 * (5 * 999 + 431)), ("read", 0, 2 * 257)]
    x = np.stack([fac.loud_quiet(sum(n for _, _, n in calls) // 2, 300 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    for rnd in range(2):
        pos = 0
        for c, (mode, chunk, n) in enumerate(calls):
            _same_as_single(g, d, mode, x[:, pos:pos + n], chunk, (rnd, c, mode))
            pos += n
        g.reset()
        d.reset()
        assert g.squelch_hits().tolist() == [11] * n_ch
    g.close()
    d.close()


def _raw_process(g, x, chunk, stride, pcm=True):
    out = np.zeros((g.n_channels, max(stride, 1)), dtype=np.int16)
    n_pcm = C.c_size_t(0)
    return _lib.lib().rxb200_fm_group_process(g._g, x.ctypes.data, x.shape[1], chunk, out.ctypes.data if pcm else None,
                                              stride, C.byref(n_pcm), None)


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
def test_refusals_leave_every_member_alone(layout, port):
    devices = _devices(layout)
    # fifth_order passes (fm2b shape): chunk 8 rows
    p, chunk, n_ch = frd.FM2B, 8 * 2048, 5
    x = np.stack([fac.signal(3 * 8192, 400 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    a = _same_as_single(g, d, "process", x[:, :chunk], chunk, "first")
    rest = np.ascontiguousarray(x[:, chunk:])
    for obj in (g, d):
        with pytest.raises(_lib.Rxb200Error) as e:                 # a chunk off the passes' granule
            obj.full_demod(rest[:, :2 * 1001], 2 * 1001)
        assert e.value.code == _lib.EUNSUPPORTED
        with pytest.raises(_lib.Rxb200Error) as e:                 # half a complex sample in a read
            obj.process_read(rest[:, :31])
        assert e.value.code == _lib.EUNSUPPORTED
    assert _raw_process(g, rest, chunk, 1) == _lib.ECAPACITY      # pcm_stride below the call's output
    assert _raw_process(g, rest, chunk, 1 << 16, pcm=False) == _lib.EINVAL
    assert _lib.lib().rxb200_fm_group_process(g._g, None, rest.shape[1], chunk, rest.ctypes.data, 1 << 16, None,
                                              None) == _lib.EINVAL
    b = _same_as_single(g, d, "process", rest, chunk, "after the refusals")
    for k in (0, n_ch - 1):
        assert np.concatenate([a[k], b[k]]).tobytes() == port.fm_run(p, x[k], chunk).tobytes(), k
    g.close()
    d.close()
    # per-chunk reduction stages: a last chunk of 4 complex samples makes no decimated sample (the boxcar carries 10 of
    # its 42 there), so the call is refused before any member starts, and the squelch carry and levels stay
    q = CASES["squelch_levels"][0]
    x = np.stack([fac.loud_quiet(6000, 500 + k) for k in range(n_ch)])
    g = fm.FmGroup(q, n_ch, devices)
    d = fm.FmDemod(q, n_channels=n_ch)
    _same_as_single(g, d, "process", x[:, :2 * 3000], 2 * 1000, "first")
    lv = g.levels()
    for obj in (g, d):
        with pytest.raises(_lib.Rxb200Error) as e:
            obj.full_demod(x[:, 2 * 3000:2 * 3000 + 2 * 1004], 2 * 1000)
        assert e.value.code == _lib.EUNSUPPORTED
    assert g.levels().tolist() == lv.tolist()
    _same_as_single(g, d, "process", x[:, 2 * 3000:], 2 * 1000, "after the refusal")
    g.close()
    d.close()


def test_caller_device_is_kept():
    """A group whose members sit on another GPU leaves the caller's current device as it was, after every entry
    point."""
    if _n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    import torch
    p = CASES["squelch_levels"][0]
    x = np.stack([fac.loud_quiet(4000, 600 + k) for k in range(3)])
    for caller, members in ((0, [1, 1]), (1, [0, 0, 0])):
        torch.cuda.set_device(caller)
        g = fm.FmGroup(p, 3, members)
        assert torch.cuda.current_device() == caller
        g.full_demod(x, 2 * 1000)
        assert torch.cuda.current_device() == caller
        g.process_read(x[:, :2 * 999])
        assert torch.cuda.current_device() == caller
        g.squelch_hits()
        g.levels()
        g.reset()
        assert torch.cuda.current_device() == caller
        with pytest.raises(_lib.Rxb200Error):
            g.full_demod(x[:, :2 * 1004], 2 * 1000)
        assert torch.cuda.current_device() == caller
        g.close()
        assert torch.cuda.current_device() == caller
