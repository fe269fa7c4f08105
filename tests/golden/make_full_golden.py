"""Mint tests/golden/full_golden.json (+ full_std_vectors.npz): the UNMODIFIED reference (oracle/_ref) run over the
BASELINE.json full-size inputs of tests/full_inputs.py -- 1 GiB rx_fm streams (2 048 chunks), cfg1 at 2^20 samples,
cfg5A's 256 channels x 2.4 M, cfg4's 871 hops x 36 sweeps (every row), cfg3's 610 hop buffers -- and over the fp64
atan2 cases (stored as vectors, not hashes: the GPU path must reproduce them byte for byte unless the port, run over the
same input, meets an atan2 value within 2^-30 of an integer, where CUDA's libm and glibc's may truncate differently;
then it may differ by 1 LSB on <= 1e-5 of them).

Run in the authoring container only (needs /root/reference):  python tests/golden/make_full_golden.py   (~2 min)"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle  # noqa: E402
import full_inputs as FI  # noqa: E402
from cases import fm_cases  # noqa: E402
from rx_tools_b200.synth import digest  # noqa: E402


def main():
    oracle.build()
    assert oracle.have_ref(), "needs /root/reference"
    rf, rp, port = oracle.RefFm(), oracle.RefPower(), oracle.port()
    out, vec = {}, {}
    t0 = time.time()
    # ---- rx_fm, 1 GiB (2 048 chunks of 131 072)
    period = FI.fm_one_gib_period()
    x = np.tile(period, FI.FM_TILES)
    for name, cli in (("fm2b", dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9)),
                      ("fm2a", dict(wbfm=1, rate_s=2400000, rate_r=48000))):
        p = rf.derive(**cli)[0]
        y, lens, _ = rf.run(p, x, FI.CHUNK16, return_chunks=True)
        out[name] = dict(params=p.__dict__, period_sha256=digest(period), n_in_int16=int(x.size), n_out=int(y.size),
                         output_sha256=digest(y), chunk_result_len_sha256=digest(lens.astype(np.int32)),
                         chunk_result_len_head=[int(v) for v in lens[:8]], head=[int(v) for v in y[:8]], tail=[int(v) for v in y[-8:]])
        print(name, y.size, "pcm", round(time.time() - t0, 1), "s", flush=True)
    del x
    # ---- cfg1 at 2^20 samples: std (vector), fast, lut
    x1 = FI.cfg1_input()
    for atan, nm in ((0, "std"), (1, "fast"), (2, "lut")):
        p = rf.derive(rate_s=1024000, rate_r=24000, custom_atan=atan)[0]
        y = rf.run(p, x1, FI.CHUNK16)
        out[f"cfg1_{nm}"] = dict(params=p.__dict__, input_sha256=digest(x1), n_out=int(y.size), output_sha256=digest(y))
        if atan == 0:
            vec["cfg1_std_full"] = y
        assert y.size == 24576
    # ---- the fp64 atan2 cases of tests/cases.py, as vectors
    for c in fm_cases():
        if not c.exact:
            vec["case_" + c.name] = rf.run(c.params, c.make_input(), c.chunk_int16)
    # ---- cfg5A: 256 channels x 2.4 M complex, chunk 131 072 (ragged last chunk)
    p5 = oracle.FmParams(downsample=100, custom_atan=2, rate_out=24000)
    shas, n5 = [], None
    h = __import__("hashlib").sha256()
    for ch in range(FI.CFG5_CHANNELS):
        y = rf.run(p5, FI.cfg5_channel(ch), FI.CHUNK16)
        n5 = int(y.size)
        h.update(np.ascontiguousarray(y).tobytes())
        if ch in (0, 1, 255):
            shas.append((ch, digest(y)))
    out["cfg5A"] = dict(params=p5.__dict__, channels=FI.CFG5_CHANNELS, n_out_per_channel=n5, all_channels_sha256=h.hexdigest(),
                        channel_sha256={str(c): s for c, s in shas})
    print("cfg5A", n5, "pcm/channel", round(time.time() - t0, 1), "s", flush=True)
    # ---- cfg4: 871 hops x 36 sweeps, hamming
    plan = rp.setup("24M:1766M:1k", 0.285, 1, 0, 0, "hamming")
    assert plan.tune_count == 871
    hb = FI.cfg4_hops(plan.tune_count, plan.buf_len)
    avg, smp = rp.scan(hb, FI.CFG4_PASSES)
    out["cfg4"] = dict(tune_count=plan.tune_count, bin_e=plan.bin_e, passes=FI.CFG4_PASSES, input_sha256=digest(hb),
                       avg_sha256=digest(avg), samples=int(smp[0]), samples_all_equal=bool(np.all(smp == smp[0])),
                       row_sha256={str(i): digest(avg[i]) for i in (0, 1, 435, 870)},
                       csv_sha256=digest(np.frombuffer(rp.csv("/tmp/_full_golden.csv").encode(), dtype=np.uint8)))
    del hb
    print("cfg4", round(time.time() - t0, 1), "s", flush=True)
    # ---- cfg3: 610 hop buffers, host-built Hann table (SURVEY F4)
    hann = port.window_table("hann", 1024)
    plan = rp.setup("100M:101M:1k", 0.0, 1, 0, 0, "rectangle", hann)
    hb = FI.cfg3_hops(plan.buf_len)
    avg, smp = rp.scan(hb, FI.CFG3_BUFFERS)
    assert int(smp[0]) == 4880
    out["cfg3"] = dict(buffers=FI.CFG3_BUFFERS, input_sha256=digest(hb), avg_sha256=digest(avg), samples=int(smp[0]),
                       avg_head=[int(v) for v in avg.reshape(-1)[:8]])
    with open(os.path.join(HERE, "full_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "full_std_vectors.npz"), **vec)
    print("wrote full_golden.json:", sorted(out), "and", sorted(vec), round(time.time() - t0, 1), "s")


if __name__ == "__main__":
    main()
