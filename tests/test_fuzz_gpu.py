"""Randomised parity: random demod_state configurations, chunk lengths, stream lengths (ragged last chunk), call
splits and input statistics (loud, quiet, silent stretches) — CUDA path vs the port oracle, bit-exact (integer
discriminators, and atan2 unless the port met a value within 2^-30 of an integer) or within 1 LSB on isolated samples
(atan2 when it did)."""
import numpy as np
import pytest

import fm_disc as fd
import oracle
from rx_tools_b200 import _lib, fm

pytestmark = pytest.mark.gpu


def _random_case(rng):
    mode = int(rng.choice([0, 0, 0, 1, 2, 3, 4]))
    use_passes = rng.random() < 0.5
    P = int(rng.integers(1, 7)) if use_passes else 0
    D = (1 << P) if P else int(rng.choice([1, 2, 3, 6, 8, 10, 42, 100, 257]))
    gran = max(16, 2 << P)                      # int16 granularity the library accepts
    p = dict(mode=mode, downsample=D, downsample_passes=P,
             comp_fir_size=int(rng.choice([0, 9])) if P else 0,
             custom_atan=int(rng.integers(0, 4)), output_scale=int(rng.choice([1, 4, 64])),
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
    # chunk: a few decimated samples at least, multiple of the granularity (and of -o when used)
    dec_per_chunk = int(rng.integers(8, 400))
    post = 1
    if rng.random() < 0.15 and mode != 4 and (P or True):
        post = int(rng.choice([2, 4]))
        dec_per_chunk = ((dec_per_chunk + post - 1) // post) * post
    chunk_c = dec_per_chunk * D
    chunk_c = ((2 * chunk_c + gran - 1) // gran) * gran // 2
    if post > 1:
        # -o needs every chunk to decimate to a multiple of it: keep chunk an exact multiple of D*post
        m = D * post
        lcm = np.lcm(m, gran // 2)
        chunk_c = int(((chunk_c + lcm - 1) // lcm) * lcm)
        p["post_downsample"] = post
    chunk_c = min(chunk_c, 131072)
    chunk_c -= chunk_c % (gran // 2)
    if post > 1 and chunk_c % (D * post) != 0:
        p["post_downsample"] = 1
    n_chunks = int(rng.integers(2, 9))
    n_c = chunk_c * n_chunks
    if rng.random() < 0.4 and not p.get("post_downsample", 1) > 1:
        # ragged last chunk: without passes or a per-chunk stage as short as one block, which may complete no boxcar;
        # otherwise still long enough to produce output (a per-chunk stage refuses a chunk that decimates to nothing)
        short = P == 0 and not (p.get("squelch_level") or p.get("dc_block_raw") or p.get("dc_block_audio"))
        tail = int(rng.integers(1 if short else max(1, 4 * D * 2 // gran + 1), max(2, chunk_c * 2 // gran))) * (gran // 2)
        n_c = n_c - chunk_c + (min(tail, chunk_c) if short else
                               max(min(tail, chunk_c), gran // 2 * ((4 * D) // (gran // 2) + 1)))
        n_c = min(n_c, chunk_c * n_chunks)
    return p, chunk_c, n_c


def _random_input(rng, n_c):
    amp = float(rng.choice([20, 300, 3000, 12000, 32767]))
    kind = rng.random()
    if kind < 0.35:
        x = rng.integers(-int(amp), int(amp) + 1, size=2 * n_c, dtype=np.int32)
    else:
        t = np.arange(n_c)
        ph = 2 * np.pi * (0.02 + 0.2 * rng.random()) * t + 3.0 * np.sin(2 * np.pi * 0.0007 * t)
        x = np.empty(2 * n_c, dtype=np.int32)
        nz = max(1, int(amp / 50))
        x[0::2] = np.rint(amp * np.cos(ph)) + rng.integers(-nz, nz + 1, size=n_c)
        x[1::2] = np.rint(amp * np.sin(ph)) + rng.integers(-nz, nz + 1, size=n_c)
    if rng.random() < 0.4:      # a silent stretch (squelched / muted input): de-emphasis dead zone
        a, b = sorted(rng.integers(0, n_c, size=2))
        x[2 * a:2 * b] = int(rng.choice([0, 0, 7]))
    return np.clip(x, -32768, 32767).astype(np.int16)


@pytest.mark.parametrize("seed", range(60))
def test_random_configuration(seed, port):
    rng = np.random.default_rng(1000 + seed)
    pd, chunk_c, n_c = _random_case(rng)
    params = oracle.FmParams(**pd)
    x = _random_input(rng, n_c)
    chunk16 = 2 * chunk_c
    try:
        d = fm.FmDemod(params)
    except _lib.Rxb200Error as e:
        pytest.skip(f"rejected at create: {e}")
    if rng.random() < 0.5:
        d.tune(segment_len=int(rng.choice([0, 64, 256, 1024])))
    want, lw, hw = port.fm_run(params, x, chunk16, return_chunks=True)
    try:
        if rng.random() < 0.5:
            got, lg = d.full_demod(x, chunk16, return_chunks=True)
            assert np.array_equal(lg, lw)
        else:       # split into calls on chunk boundaries: carry across calls
            cuts = sorted(set(int(c) * chunk16 for c in rng.integers(1, max(2, x.size // chunk16 + 1), size=2)))
            parts, pos = [], 0
            for c in cuts + [x.size]:
                if c > pos:
                    parts.append(d.full_demod(x[pos:c], chunk16))
                    pos = c
            got = np.concatenate(parts) if parts else np.zeros(0, np.int16)
    except _lib.Rxb200Error as e:
        if e.code == _lib.EUNSUPPORTED:
            pytest.skip(f"shape not supported: {e}")
        raise
    assert got.size == want.size, (pd, chunk_c, n_c)
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    if params.mode == 0 and params.custom_atan == 0 and fd.port_met_near_integer():
        # the port met an fp64 atan2 value within 2^-30 of an integer, where CUDA's libm and glibc's may truncate
        # differently: that sample may be 1 LSB off, and downstream IIR / resampler stages can smear the flip
        assert np.count_nonzero(diff) <= max(2, int(1e-4 * diff.size)), (pd, np.flatnonzero(diff)[:5])
        if not params.deemph and params.rate_out2 <= 0 and not params.dc_block_audio:
            assert diff.max(initial=0) <= 1
    else:
        # integer paths, and -A std wherever no atan2 value came near an integer: bit-exact
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (pd, chunk_c, n_c, bad[:5], got[bad[:5]], want[bad[:5]])
    if params.squelch_level:
        hits = np.zeros(1, dtype=np.int32)
        import ctypes as C
        _lib.check(_lib.lib().rxb200_fm_squelch_hits(d._h, hits.ctypes.data_as(C.POINTER(C.c_int))))
        assert int(hits[0]) == int(hw[-1])
    d.close()
