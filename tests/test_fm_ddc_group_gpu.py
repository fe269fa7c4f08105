"""Decimating mixing groups (rxb200_fm_mix_group_create_ddc) against one decimating handle with every channel: groups of
2, 3 and 4 members on repeated ordinals, K = 5 and 33, over mixed process / process_read / reset sequences with reads
that are not multiples of M (and reads with no output), and refusals that start no member."""
import numpy as np
import pytest

import fm_ddc as fdd
import fm_mix as fmx
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu


def _ops(M, tiny):
    """tiny: a read of 7 samples (no output at M = 64); a chain with per-chunk stages refuses reads below one boxcar"""
    return [("read", 2 * 9001), ("chunk", 2 * M * 120 + 2 * (45 * M + 3), 2 * M * 60)] + [("read", 2 * 7)] * tiny + [
        ("reset",), ("read", 2 * 5003), ("chunk", 2 * M * 64, 2 * M * 64), ("read", 2 * 12011)]


def _run(obj, x, ops, levels):
    out, at = [], 0
    for op in ops:
        if op[0] == "reset":
            obj.reset()
            at = 0
            continue
        part = x[at:at + op[1]]
        if op[0] == "read":
            r = obj.process_read(part)
            out.append((r.tobytes(), r.shape))
        else:
            r, rl = obj.full_demod(part, op[2], True)
            out.append((r.tobytes(), rl.tolist()))
        out.append(obj.squelch_hits().tolist())
        if levels:
            out.append(obj.levels().tolist())
        at += op[1]
    return out


@pytest.mark.parametrize("n_dev", [2, 3, 4])
@pytest.mark.parametrize("k", [5, 33])
@pytest.mark.parametrize("name", ["nbfm_m64_t257", "fm_lut_squelch_m4", "raw_wide_m3"])
def test_group_equals_one_handle(name, k, n_dev):
    p, rate, _, ddc, _, _ = fdd.SHAPES[name]
    p = fm.FmParams.from_any(p)
    p.report_levels = 1 if p.squelch_level else 0
    M = ddc[0]
    offs = [int(rate // 200) * (j - k // 2) for j in range(k)]
    ops = _ops(M, not p.squelch_level)
    r = ops.index(("reset",))
    n = max(sum(op[1] for op in ops[:r]), sum(op[1] for op in ops[r + 1:]))
    x = fmx.capture(n // 2 + 16, rate, offs[::4], 70 + k, quiet_half=bool(p.squelch_level))
    one = fm.FmMix(p, rate, offs, ddc=ddc)
    grp = fm.FmMixGroup(p, rate, offs, devices=[0] * n_dev, ddc=ddc)
    assert _run(grp, x, ops, p.report_levels) == _run(one, x, ops, p.report_levels)
    one.close()
    grp.close()


def test_refused_call_starts_no_member():
    p, rate, offs, ddc, x, _ = fdd.case_input("fm2b_f9_m8", seed=4)
    offs = offs + [1_200_000, -2_400_000]
    one = fm.FmMix(p, rate, offs, ddc=ddc)
    grp = fm.FmMixGroup(p, rate, offs, devices=[0, 0, 0], ddc=ddc)
    assert grp.process_read(x[:2 * 20011]).tobytes() == one.process_read(x[:2 * 20011]).tobytes()
    rest = x[2 * 20011:]
    for call in (lambda g: g.full_demod(rest[:2 * 8 * 1024], 2 * 1001),     # not a multiple of 2M
                 lambda g: g.process_read(rest[:2 * 60])):                 # 7 outputs: fewer than 2^3
        for obj in (grp, one):
            with pytest.raises(_lib.Rxb200Error) as e:
                call(obj)
            assert e.value.code == _lib.EUNSUPPORTED
    assert grp.process_read(rest[:2 * 6007]).tobytes() == one.process_read(rest[:2 * 6007]).tobytes()
    one.close()
    grp.close()
