"""The discriminators' device code alone (rxb200_fm_disc_device, the very __device__ functions the kernels inline) against
the port on every operand class of fm_disc.py within each form's domain: the integer forms, the row and stream front
ends' FP32 forms and the AM envelope byte for byte; the libm-backed std forms (disc_std_f32, disc_std, disc_std_lean)
byte for byte too, except that a pair whose std value lies within 2^-30 of an integer (the port's near flag: the only
place where CUDA's atan2 and glibc's may truncate differently) may differ by 1.  And -A lut through every kernel route
at D >= 17 on a capture whose decimated samples carry the pairs the reference crashes on, against the port byte for
byte, each of them at +-8192."""

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_disc as fd
import fm_handles as fh
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu


def _device(form, q):
    torch = fh.torch()
    dq = torch.from_numpy(np.ascontiguousarray(q, dtype=np.int32)).cuda()
    out = fm.disc_device(form, dq)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _check(port, form, q, what):
    """the device form against the port on q's quads in the form's domain; returns (pairs compared, near pairs met,
    near pairs that differed)"""
    q = fd.domain(form, q)
    if q.shape[0] == 0:
        return 0, 0, 0
    got = _device(form, q)
    want, near = port.disc_many(form, q, want_near=form in fd.STD_FORMS)
    diff = got.astype(np.int64) - want
    if form in fd.STD_FORMS:
        bad = np.flatnonzero((diff != 0) & ~near)
        assert np.abs(diff[near]).max(initial=0) <= 1, (what, fd.FORM_NAMES[form])
        n_near, n_flip = int(near.sum()), int(np.count_nonzero(diff[near]))
    else:
        bad = np.flatnonzero(diff)
        n_near = n_flip = 0
    assert bad.size == 0, (what, fd.FORM_NAMES[form], bad.size, q[bad[:4]], got[bad[:4]], want[bad[:4]])
    return q.shape[0], n_near, n_flip


@pytest.mark.parametrize("form", range(9), ids=fd.FORM_NAMES)
def test_form_equals_port(form, port):
    sets = [("small", q) for q in fd.small_slices()]
    sets += sorted(fd.random_classes().items()) + sorted(fd.edges().items()) + [("stream", fd.stream_class())]
    total = near = flips = 0
    for name, q in sets:
        n, k, f = _check(port, form, q, name)
        total, near, flips = total + n, near + k, flips + f
    print(f"disc form {fd.FORM_NAMES[form]}: {total} pairs, {near} near an integer, {flips} of them 1 LSB apart")
    assert total > 1_000_000
    if form in fd.STD_FORMS:
        assert near < 1000                                    # the edge fixture's libm buckets and a few strays


def test_disc_device_refusals():
    torch = fh.torch()
    q = torch.zeros((4, 4), dtype=torch.int32, device="cuda")
    for form in (-1, 9):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.disc_device(form, q)
        assert e.value.code == _lib.EINVAL
    out = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert _lib.lib().rxb200_fm_disc_device(0, q.data_ptr() + 4, 2, out.data_ptr(), None) == _lib.EINVAL   # unaligned
    assert _lib.lib().rxb200_fm_disc_device(0, q.data_ptr(), 0, out.data_ptr(), None) == _lib.OK


# -A lut routes at D >= 17: name -> (parameters, chunk in complex samples, rotation undone per chunk, handle kind)
LUT_ROUTES = {
    "spec3": (fac.FM5A, 25000, True, "demod"),                                      # the fused SPEC 3 kernel
    "spec0": (fac.with_(fac.FM24K_LUT, offset_tuning=1), 21000, False, "demod"),   # the fused SPEC 0 kernel
    "any": (fac.with_(fac.FM24K_LUT, offset_tuning=1), 2003, False, "demod"),      # the any-length kernel
    "mix": (fac.FM5A, 25000, True, "mix"),                                          # a mixing handle, offset 0
}


@pytest.mark.parametrize("route", sorted(LUT_ROUTES))
def test_lut_crash_pairs_through_chain(route, port):
    p, chunk_c, rot, kind = LUT_ROUTES[route]
    D = p.downsample
    n_dec = 40 * (chunk_c // D + 1)
    dec, placed = fd.crash_sequence(D, n_dec, chunk_c / D)
    x = fd.crafted_capture(port, D, dec, chunk_complex=chunk_c if rot else None)
    want, lens, _ = port.fm_run(p, x, 2 * chunk_c, return_chunks=True)
    if kind == "mix":
        obj = fm.FmMix(p, 2_400_000, [0])
        got = obj.full_demod(x, 2 * chunk_c)[0]
        member = int(_lib.lib().rxb200_fm_mix_member(obj._h) or 0)
        kinds = fh.kernel_kinds([member])
    else:
        obj = fm.FmDemod(p)
        got = obj.full_demod(x, 2 * chunk_c)
        kinds = [obj.stats()["kernel_kind"]]
    obj.close()
    assert kinds == [0], (route, kinds)
    assert got.tobytes() == want.tobytes(), (route, np.flatnonzero(got != want)[:5])
    starts = set(np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist())
    checked = 0
    for n, pos in placed:
        if n not in starts:
            assert int(got[n]) == (8192 if pos else -8192), (route, n)
            checked += 1
    assert checked >= 16, route
