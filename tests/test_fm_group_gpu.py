"""rx_fm on several GPUs through one group handle (rxb200_fm_group_*): the group's PCM, chunk result lengths, squelch hits
and -L levels equal those of ONE handle with every channel, after every call of a sequence that mixes process,
process_read and reset; the port checks a subset of the channels.  The shapes reach every kernel the single handle
runs.  Members repeat ordinal 0, so one H100 runs the whole group; the same cases run on distinct ordinals where the box
has that many GPUs.  Refused calls leave every member's carry where it was, and the caller's current device stays."""
import numpy as np
import pytest

import fm_any_chunk as fac
import fm_handles as fh
import fm_read as frd
from rx_tools_b200 import _lib, fm, sharding

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
@pytest.mark.parametrize("name", sorted(fh.ROUTES))
def test_paths_match_one_handle_and_port(name, layout, port):
    devices = fh.devices(layout)
    p, mode, chunk, lens, kind, make = fh.ROUTES[name]
    n_ch = 5
    x = np.stack([make(sum(lens) // 2, 100 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    parts, pos = [], 0
    for c, n in enumerate(lens):
        parts.append(fh.same_as_single(g, d, mode, x[:, pos:pos + n], chunk, (name, c)))
        kinds = fh.kernel_kinds(map(g.member, range(g.n_dev)))
        assert kinds == [kind] * len(kinds), (name, c, kinds)
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
    devices = fh.devices((kind, [0] * n_dev if kind == "same" else list(range(n_dev))))
    p, _, chunk, lens, _, make = fh.ROUTES["any"]
    x = np.stack([make(sum(lens) // 2, 200 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    assert _lib.lib().rxb200_fm_group_size(g._h) == n_dev
    for i in range(n_dev):
        b, e = sharding.unit_range(i, n_dev, n_ch)
        assert (g.member(i) == 0) == (e == b), (n_ch, n_dev, i)
    assert g.member(n_dev) == 0 and g.member(-1) == 0
    d = fm.FmDemod(p, n_channels=n_ch)
    pos = 0
    for c, n in enumerate(lens):
        fh.same_as_single(g, d, "process", x[:, pos:pos + n], chunk, (n_ch, n_dev, c))
        pos += n
    g.close()
    d.close()


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
def test_mixed_call_sequence_then_reset(layout):
    """process and process_read calls of several lengths on one group, reset, and the sequence again: chunk result
    lengths, squelch hits and levels after every call."""
    devices = fh.devices(layout)
    p = fh.ROUTES["squelch_levels"][0]
    n_ch = 7
    calls = [("process", 2 * 2003, 2 * 3 * 2003), ("read", 0, 2 * 1777), ("process", 2 * 4096, 2 * 8 * 4096),
             ("read", 0, 2 * 5003), ("process", 2 * 999, 2 * (5 * 999 + 431)), ("read", 0, 2 * 257)]
    x = np.stack([fac.loud_quiet(sum(n for _, _, n in calls) // 2, 300 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    for rnd in range(2):
        pos = 0
        for c, (mode, chunk, n) in enumerate(calls):
            fh.same_as_single(g, d, mode, x[:, pos:pos + n], chunk, (rnd, c, mode))
            pos += n
        g.reset()
        d.reset()
        assert g.squelch_hits().tolist() == [11] * n_ch
    g.close()
    d.close()


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
def test_refusals_leave_every_member_alone(layout, port):
    devices = fh.devices(layout)
    # fifth_order passes (fm2b shape): chunk 8 rows
    p, chunk, n_ch = frd.FM2B, 8 * 2048, 5
    x = np.stack([fac.signal(3 * 8192, 400 + k) for k in range(n_ch)])
    g = fm.FmGroup(p, n_ch, devices)
    d = fm.FmDemod(p, n_channels=n_ch)
    a = fh.same_as_single(g, d, "process", x[:, :chunk], chunk, "first")
    rest = np.ascontiguousarray(x[:, chunk:])
    for obj in (g, d):
        with pytest.raises(_lib.Rxb200Error) as e:                 # a chunk off the passes' granule
            obj.full_demod(rest[:, :2 * 1001], 2 * 1001)
        assert e.value.code == _lib.EUNSUPPORTED
        with pytest.raises(_lib.Rxb200Error) as e:                 # half a complex sample in a read
            obj.process_read(rest[:, :31])
        assert e.value.code == _lib.EUNSUPPORTED
    assert fh.raw_process(g, rest, chunk, 1) == _lib.ECAPACITY      # pcm_stride below the call's output
    assert fh.raw_process(g, rest, chunk, 1 << 16, pcm=False) == _lib.EINVAL
    assert _lib.lib().rxb200_fm_group_process(g._h, None, rest.shape[1], chunk, rest.ctypes.data, 1 << 16, None,
                                              None) == _lib.EINVAL
    b = fh.same_as_single(g, d, "process", rest, chunk, "after the refusals")
    for k in (0, n_ch - 1):
        assert np.concatenate([a[k], b[k]]).tobytes() == port.fm_run(p, x[k], chunk).tobytes(), k
    g.close()
    d.close()
    # per-chunk reduction stages: a last chunk of 4 complex samples makes no decimated sample (the boxcar carries 10 of
    # its 42 there), so the call is refused before any member starts, and the squelch carry and levels stay
    q = fh.ROUTES["squelch_levels"][0]
    x = np.stack([fac.loud_quiet(6000, 500 + k) for k in range(n_ch)])
    g = fm.FmGroup(q, n_ch, devices)
    d = fm.FmDemod(q, n_channels=n_ch)
    fh.same_as_single(g, d, "process", x[:, :2 * 3000], 2 * 1000, "first")
    lv = g.levels()
    for obj in (g, d):
        with pytest.raises(_lib.Rxb200Error) as e:
            obj.full_demod(x[:, 2 * 3000:2 * 3000 + 2 * 1004], 2 * 1000)
        assert e.value.code == _lib.EUNSUPPORTED
    assert g.levels().tolist() == lv.tolist()
    fh.same_as_single(g, d, "process", x[:, 2 * 3000:], 2 * 1000, "after the refusal")
    g.close()
    d.close()


def test_caller_device_is_kept():
    """A group whose members sit on another GPU leaves the caller's current device as it was, after every entry
    point."""
    if fh.n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    import torch
    p = fh.ROUTES["squelch_levels"][0]
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
