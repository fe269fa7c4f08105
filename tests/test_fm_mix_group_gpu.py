"""The channels of one capture spread over several GPUs through one mixing group handle (rxb200_fm_mix_group_*): the
group's PCM, n_pcm, chunk result lengths, squelch hits and -L levels equal those of ONE mixing handle with every channel,
after every call of sequences that mix process, process_read and reset, on every kernel route of the chain and with
members that own no channel.  The golden hashes of the reference hold through a group, the mixers' phases carry across
ragged reads and restart at reset, refused calls leave every member's phases and carries alone, and the caller's current
device stays.  Members repeat ordinal 0, so one H100 runs the whole group; the same cases run on distinct ordinals where
the box has that many GPUs."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_handles as fh
import fm_mix as fmx
from rx_tools_b200 import _lib, fm, sharding

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_mix_golden.json")
RATE = 2_400_000


def _offsets(k):
    """k channels on a 12.5 kHz raster around the capture's centre (up to +-200 kHz at k = 33)."""
    return [12500 * (j - k // 2) for j in range(k)]


def _members_match_shards(g):
    """Member i has a handle exactly when its shard of the channels is not empty; returns how many have one."""
    assert _lib.lib().rxb200_fm_mix_group_size(g._h) == g.n_dev
    owners = 0
    for i in range(g.n_dev):
        b, e = sharding.unit_range(i, g.n_dev, g.n_channels)
        assert (g.member(i) == 0) == (e == b), (g.n_channels, g.n_dev, i)
        owners += e > b
    assert g.member(g.n_dev) == 0 and g.member(-1) == 0
    return owners


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
@pytest.mark.parametrize("k", [1, 3, 5, 8, 33])
@pytest.mark.parametrize("name", sorted(fh.ROUTES))
def test_routes_match_one_mixing_handle(name, k, layout):
    """Every call of the route's sequence, a reset, and its first call again; every member's inner handle runs the
    kernel the single handle runs."""
    devices = fh.devices(layout)
    p, mode, chunk, lens, kind, make = fh.ROUTES[name]
    offs = _offsets(k)
    x = make(sum(lens) // 2, 50 + k)
    g = fm.FmMixGroup(p, RATE, offs, devices)
    owners = _members_match_shards(g)
    mx = fm.FmMix(p, RATE, offs)
    seq = list(fac.seq_bounds(x.size, lens))
    for c, step in enumerate(seq + ["reset"] + seq[:1]):
        if step == "reset":
            g.reset()
            mx.reset()
            continue
        pos, n = step
        fh.same_as_single(g, mx, mode, x[pos:pos + n], chunk, (name, k, c))
        assert mx.stats()["kernel_kind"] == kind, (name, k, c, mx.stats())
        kinds = fh.kernel_kinds(map(g.inner, range(g.n_dev)))
        assert len(kinds) == owners and kinds == [kind] * len(kinds), (name, k, c, kinds)
    g.close()
    mx.close()


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
def test_mixed_call_sequence_then_reset(layout):
    """process and process_read calls of several lengths on one group, reset, and the sequence again: chunk result
    lengths, squelch hits and levels after every call."""
    devices = fh.devices(layout)
    p = fh.ROUTES["squelch_levels"][0]
    offs = _offsets(7)
    calls = [("process", 2 * 2003, 2 * 3 * 2003), ("read", 0, 2 * 1777), ("process", 2 * 4096, 2 * 8 * 4096),
             ("read", 0, 2 * 5003), ("process", 2 * 999, 2 * (5 * 999 + 431)), ("read", 0, 2 * 257)]
    x = fac.loud_quiet(sum(n for _, _, n in calls) // 2, 300)
    g = fm.FmMixGroup(p, RATE, offs, devices)
    mx = fm.FmMix(p, RATE, offs)
    for rnd in range(2):
        pos = 0
        for c, (mode, chunk, n) in enumerate(calls):
            fh.same_as_single(g, mx, mode, x[pos:pos + n], chunk, (rnd, c, mode))
            pos += n
        g.reset()
        mx.reset()
        assert g.squelch_hits().tolist() == mx.squelch_hits().tolist()
    g.close()
    mx.close()


def test_golden_through_a_group_of_three():
    """Every shape of tests/golden/fm_mix_golden.json read by read through a group of 3 members on ordinal 0: the
    reference's result lengths, its hashes for the integer shapes, and the single handle's bytes for every shape."""
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fmx.SHAPES)
    for name in sorted(fmx.SHAPES):
        p, rate, offs, x = fmx.case_input(name)
        gd = gold[name]
        assert gd["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        g = fm.FmMixGroup(p, rate, offs, [0, 0, 0])
        got, counts = fh.reads(g, x, gd["lens_int16"])
        mx = fm.FmMix(p, rate, offs)
        want, _ = fh.reads(mx, x, gd["lens_int16"])
        assert got.tobytes() == want.tobytes(), name
        for j, c in enumerate(gd["channels"]):
            assert c["offset_hz"] == offs[j]
            assert counts == c["result_len"], (name, j)
            if fac.INTEGER(p):
                assert hashlib.sha256(got[j].tobytes()).hexdigest() == c["sha256"], (name, j)
        g.close()
        mx.close()


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
def test_phases_across_ragged_reads_and_reset(layout):
    """Ragged reads (1021:333:4093) over part of the capture, a reset, the whole read sequence, then chunk calls that
    end off a chunk: the phases run on across every call and restart at the reset, as in the single handle."""
    devices = fh.devices(layout)
    p, rate, offs, x = fmx.case_input("fm5a_lut_d100", seed=6)
    offs = offs + [-50000, 62500, 100000]                 # 7 channels: every member of 4 owns some
    g = fm.FmMixGroup(p, rate, offs, devices)
    mx = fm.FmMix(p, rate, offs)
    bounds = list(fac.seq_bounds(x.size, fmx.READS))
    for c, (pos, n) in enumerate(bounds[:len(bounds) // 2]):
        fh.same_as_single(g, mx, "read", x[pos:pos + n], 0, ("first half", c))
    g.reset()
    mx.reset()
    parts = []
    for c, (pos, n) in enumerate(bounds):
        parts.append(fh.same_as_single(g, mx, "read", x[pos:pos + n], 0, ("after reset", c)))
    c16 = 2 * 1021
    cuts = [0, 3 * c16, 4 * c16 + 2 * 17, 11 * c16, x.size]
    for a, b in zip(cuts, cuts[1:]):
        fh.same_as_single(g, mx, "process", x[a:b], c16, ("chunks", a))
    g.close()
    mx.close()
    # the reads after the reset are those of a fresh single handle
    fresh = fm.FmMix(p, rate, offs)
    want, _ = fh.reads(fresh, x, fmx.READS)
    assert np.concatenate(parts, axis=1).tobytes() == want.tobytes()
    fresh.close()


def _refused(g, mx, call, code):
    for obj in (g, mx):
        with pytest.raises(_lib.Rxb200Error) as e:
            call(obj)
        assert e.value.code == code, (obj, e.value)


@pytest.mark.parametrize("layout", fh.LAYOUTS, ids=fh.LAYOUT_IDS)
def test_refusals_leave_every_member_alone(layout):
    devices = fh.devices(layout)
    # fifth_order passes (fm2b shape), 5 channels: chunk 8 rows
    p, rate, _, kw = fmx.SHAPES["fm2b_f9"]
    offs = [-600000, -300000, 0, 450000, 900000]
    chunk = 8 * 2048
    x = fmx.capture(7 * chunk // 2, rate, offs, 11, **kw)
    g = fm.FmMixGroup(p, rate, offs, devices)
    mx = fm.FmMix(p, rate, offs)
    pos = chunk
    fh.same_as_single(g, mx, "process", x[:pos], chunk, "first")
    rest = np.ascontiguousarray(x[pos:pos + chunk])
    refusals = [
        (lambda o: o.full_demod(rest[:2 * 1001], 2 * 1001), _lib.EUNSUPPORTED),      # a chunk off the passes' granule
        (lambda o: o.process_read(rest[:31]), _lib.EUNSUPPORTED),                    # half a complex sample
    ]
    for c, (call, code) in enumerate(refusals):
        _refused(g, mx, call, code)
        fh.same_as_single(g, mx, "process", x[pos:pos + chunk], chunk, ("after refusal", c))
        pos += chunk
    for c, (stride, pcm, code) in enumerate(((1, True, _lib.ECAPACITY), (1 << 16, False, _lib.EINVAL))):
        assert fh.raw_process(g, rest, chunk, stride, pcm) == code
        assert fh.raw_process(mx, rest, chunk, stride, pcm) == code
        fh.same_as_single(g, mx, "process", x[pos:pos + chunk], chunk, ("after raw refusal", c))
        pos += chunk
    assert _lib.lib().rxb200_fm_mix_group_process(g._h, None, rest.size, chunk, rest.ctypes.data, 1 << 16, None,
                                                  None) == _lib.EINVAL
    fh.same_as_single(g, mx, "process", x[pos:pos + chunk], chunk, "after a null capture")
    g.close()
    mx.close()
    # per-chunk reduction stages: a last chunk of 4 complex samples makes no decimated sample, so the call is refused
    # before any member starts; levels, squelch carries and phases stay
    q = fm.FmParams.from_any(fmx.SHAPES["fm_lut_d42_squelch"][0])
    q.report_levels = 1
    rate, offs = 1_008_000, [-40000, -20000, 0, 20000, 40000]
    x = fmx.capture(6000, rate, offs, 9, quiet_half=True)
    g = fm.FmMixGroup(q, rate, offs, devices)
    mx = fm.FmMix(q, rate, offs)
    fh.same_as_single(g, mx, "process", x[:2 * 3000], 2 * 1000, "first")
    lv = g.levels()
    _refused(g, mx, lambda o: o.full_demod(x[2 * 3000:2 * 3000 + 2 * 1004], 2 * 1000), _lib.EUNSUPPORTED)
    assert g.levels().tolist() == lv.tolist()
    fh.same_as_single(g, mx, "process", x[2 * 3000:], 2 * 1000, "after the refusal")
    g.close()
    mx.close()


def test_caller_device_is_kept():
    """A group whose members sit on another GPU leaves the caller's current device as it was, after every entry
    point."""
    if fh.n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    import torch
    p = fh.ROUTES["squelch_levels"][0]
    offs = _offsets(3)
    x = fac.loud_quiet(4000, 600)
    for caller, members in ((0, [1, 1]), (1, [0, 0, 0])):
        torch.cuda.set_device(caller)
        g = fm.FmMixGroup(p, RATE, offs, members)
        assert torch.cuda.current_device() == caller
        g.full_demod(x, 2 * 1000)
        assert torch.cuda.current_device() == caller
        g.process_read(x[:2 * 999])
        assert torch.cuda.current_device() == caller
        g.squelch_hits()
        g.levels()
        g.reset()
        assert torch.cuda.current_device() == caller
        with pytest.raises(_lib.Rxb200Error):
            g.full_demod(x[:2 * 1004], 2 * 1000)
        assert torch.cuda.current_device() == caller
        g.close()
        assert torch.cuda.current_device() == caller
