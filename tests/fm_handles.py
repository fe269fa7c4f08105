"""Helpers the GPU tests of the rx_fm handle kinds share (FmDemod, FmGroup, FmMix with and without a DDC, FmMixGroup):
every int16 value as a capture, reads over a read sequence, the port on each channel of one capture, the comparison of
PCM against the port, the group layouts, one call of a handle and the same call on a group, a raw process call for
refusals, and the one table of kernel routes.
"""
import ctypes as C

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import fm_read as frd
from rx_tools_b200 import _lib, fm


def torch():
    import torch
    return torch


def every_int16(seed):
    """65 536 complex samples whose I and Q each take every int16 value once."""
    rng = np.random.default_rng(seed)
    x = np.empty(2 * 65536, dtype=np.int16)
    x[0::2] = rng.permutation(np.arange(-32768, 32768)).astype(np.int16)
    x[1::2] = rng.permutation(np.arange(-32768, 32768)).astype(np.int16)
    return x


def reads(obj, x, lens16):
    """process_read over the read sequence: (pcm per channel, PCM count per read)."""
    parts, counts = [], []
    for pos, n in fac.seq_bounds(x.size, lens16):
        r = obj.process_read(x[pos:pos + n])
        parts.append(r)
        counts.append(r.shape[-1])
    return np.concatenate(parts, axis=-1), counts


def port_channels(port, p, rate, offs, x, lens16, ddc=None):
    """The port on each channel of a capture, read by read over lens16: [(pcm, result_len, hits)].  Without ddc the
    channel is the model's mixed stream; with ddc it is the model's decimated stream, one chain read per capture read
    with output."""
    out = []
    for f in offs:
        if ddc is None:
            y, lens = fmx.mix_model(x, fm.mix_table(rate, f)), lens16
        else:
            y, lens = fdd.nonempty(fdd.decimated_reads(x, fm.mix_table(rate, f), ddc, lens16))
        out.append(fac.port_run_seq(port, p, y, lens, return_chunks=True))
    return out


def compare(p, got, want, what):
    """PCM against the port: exact for the integer discriminators, else at most a few samples 1 LSB apart."""
    assert got.size == want.size, (what, got.size, want.size)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    if fac.INTEGER(p):
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    else:
        # fp64 atan2 on every sample (CUDA libm against glibc): a last-ulp difference may move a sample by 1 LSB
        assert np.count_nonzero(diff) <= max(2, int(1e-4 * diff.size)), (what, np.flatnonzero(diff)[:5])
        assert diff.max(initial=0) <= 1, what


def with_levels(p):
    q = fm.FmParams.from_any(p)
    q.report_levels = 1
    return q


# name -> (parameters, "process" or "read", chunk int16, the calls' lengths in int16, kernel_kind every handle reports,
# input of one channel)
ROUTES = {
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
    "squelch_levels": (with_levels(fac.with_(fac.FM24K_LUT, squelch_level=60)), "process", 2 * 2003,
                       [2 * 4 * 2003, 2 * (2003 + 457)], 0, fac.loud_quiet),
}

# the kernel routes alone, without the input column: (parameters, process or read, chunk, call lengths, kernel_kind)
KERNEL_ROUTES = {name: r[:5] for name, r in ROUTES.items() if name != "squelch_levels"}


def n_gpus():
    return int(_lib.lib().rxb200_device_count())


LAYOUTS = [("same", [0, 0]), ("same", [0, 0, 0]), ("same", [0, 0, 0, 0]),
           ("distinct", [0, 1]), ("distinct", [0, 1, 2]), ("distinct", [0, 1, 2, 3])]
LAYOUT_IDS = [f"{k}-{len(d)}" for k, d in LAYOUTS]


def devices(layout):
    """The layout's member ordinals; skips when the box has too few GPUs."""
    kind, devs = layout
    if n_gpus() < max(devs) + 1:
        pytest.skip(f"needs {max(devs) + 1} GPUs")
    return devs


def kernel_kinds(handles):
    """kernel_kind of the last call of every rxb200_fm handle given as an integer (0: no handle, skipped)."""
    kinds = []
    for h in handles:
        if h:
            s = _lib.FmStatsC()
            _lib.check(_lib.lib().rxb200_fm_last_stats(C.c_void_p(h), C.byref(s)))
            kinds.append(s.kernel_kind)
    return kinds


def call(obj, mode, x, chunk):
    """One call on any handle: (pcm, chunk result lengths or None)."""
    if mode == "read":
        return obj.process_read(x), None
    return obj.full_demod(x, chunk, return_chunks=True)


def same_as_single(g, one, mode, x, chunk, what):
    """One call on a group and on the single handle of the same kind; everything the group reports equals the single
    handle's."""
    got, gl = call(g, mode, x, chunk)
    want, wl = call(one, mode, x, chunk)
    assert got.shape == want.shape and got.tobytes() == want.tobytes(), what
    if wl is not None:
        assert gl.tolist() == wl.tolist(), what
    assert g.squelch_hits().tolist() == one.squelch_hits().tolist(), what
    if g.params.report_levels:
        assert g.levels().tolist() == one.levels().tolist(), what
    return got


def raw_process(obj, x, chunk, stride, pcm=True):
    """<prefix>_process of any handle straight through ctypes, so that a refusal returns its code."""
    out = np.zeros((obj.n_channels, max(stride, 1)), dtype=np.int16)
    n_pcm = C.c_size_t(0)
    return getattr(_lib.lib(), obj._prefix + "_process")(obj._h, x.ctypes.data, x.shape[-1], chunk,
                                                         out.ctypes.data if pcm else None, stride, C.byref(n_pcm),
                                                         None)
