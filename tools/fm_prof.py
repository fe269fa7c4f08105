#!/usr/bin/env python3
"""Where an item's cycles go in the split rx_fm kernel, per warp and per SMSP (sub-partition).

Needs a scratch build with -DRXB_PROF (tools/build_variants.sh prof="-DRXB_PROF"), selected with RXB200_LIB: the kernel
then sums clock64() intervals per warp into a device array (fm_kernels.cu, PF_*).  Runs bench.py's fm2b stream (1 GiB
CS16, chunk 131072) once to warm up and once measured, and prints per warp slot of the CTA: its %warpid % 4 over all
CTAs (the SMSP it issues on), and per item the cycles of each phase.
  RXB200_LIB=rx_tools_b200/variants/librxb200_prof.so python tools/fm_prof.py [--size-mib 1024]
--timeline: instead, PROF_CALLS back-to-back calls of that stream (sync=False, one output buffer, as bench.py makes
them) and, per call, from each CTA's %globaltimer stamps: how long the back end waits for its first item (fill), how
long the front-end warps sit idle after the sentinel ticket (drain), how long the CTA's SM slot stays empty before the
grid ends (tail), and the gap from the end of one call to the first CTA of the next (negative: the calls overlap)."""
import argparse
import collections
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PROF_CTAS, PROF_SLOTS = 1024, 16
(PF_WARPID, PF_SMID, PF_TOTAL, PF_ITEMS, PF_ROWS, PF_FRONT, PF_BAR_FE, PF_EMPTY, PF_RING, PF_PUBLISH,
 PF_FULL, PF_COLLECT, PF_PASS1, PF_CHAIN, PF_PASS2) = range(15)
FE_COLS = [("rows", PF_ROWS), ("front_rows", PF_FRONT), ("ring wait", PF_RING), ("BAR_FE", PF_BAR_FE),
           ("empty", PF_EMPTY), ("publish", PF_PUBLISH)]
BE_COLS = [("full", PF_FULL), ("collect", PF_COLLECT), ("pass 1", PF_PASS1), ("chain", PF_CHAIN), ("pass 2", PF_PASS2)]
PROF_CALLS, TS_N = 4, 8
TS_ENTRY, TS_FIRST_FULL, TS_SENTINEL, TS_LAST_END, TS_EXIT = range(5)


def timeline(lib, d, x, out, cap):
    """per-call fill / drain / tail / gap of PROF_CALLS chained calls (microseconds and shares of the call's span)"""
    import torch
    import bench
    from rx_tools_b200 import _lib
    lib.rxb200_fm_prof_timeline.argtypes = [C.c_void_p, C.c_size_t, C.c_int]

    def step():
        d.process_device(x.data_ptr(), x.numel(), bench.CHUNK, out.data_ptr(), cap, sync=False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    _lib.check(lib.rxb200_fm_prof_timeline(None, 0, 1))
    for _ in range(PROF_CALLS):
        step()
    torch.cuda.synchronize()
    buf = np.zeros(PROF_CALLS * PROF_CTAS * TS_N, dtype=np.uint64)
    _lib.check(lib.rxb200_fm_prof_timeline(buf.ctypes.data, buf.size, 0))
    ts = buf.reshape(PROF_CALLS, PROF_CTAS, TS_N).astype(np.int64)
    n = int((ts[0, :, TS_ENTRY] > 0).sum())
    ts = (ts[:, :n] - ts[0, :n, TS_ENTRY].min()) / 1e3        # microseconds from the first call's first CTA
    print(f"{n} CTAs per call; times in us from the first CTA of call 0")
    print("call   start     end    span   period    gap | fill mean/max   drain mean/max   tail mean/max |"
          "  fill%  drain%  tail%  gap%")
    prev_end = prev_start = None
    for c in range(PROF_CALLS):
        t = ts[c]
        start, end = t[:, TS_ENTRY].min(), t[:, TS_EXIT].max()
        span = end - start
        fill = t[:, TS_FIRST_FULL] - t[:, TS_ENTRY]
        drain = t[:, TS_EXIT] - t[:, TS_SENTINEL]
        tail = end - t[:, TS_EXIT]
        gap = start - prev_end if prev_end is not None else float("nan")
        period = start - prev_start if prev_start is not None else float("nan")
        print(f"{c:4d} {start:7.1f} {end:7.1f} {span:7.1f} {period:8.1f} {gap:6.1f} | {fill.mean():6.1f} {fill.max():6.1f}"
              f"    {drain.mean():6.1f} {drain.max():6.1f}   {tail.mean():6.1f} {tail.max():6.1f} |"
              f" {100 * fill.mean() / span:6.1f} {100 * drain.mean() / span:6.1f} {100 * tail.mean() / span:6.1f}"
              f" {100 * gap / span:5.1f}")
        prev_end, prev_start = end, start


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--timeline", action="store_true")
    args = ap.parse_args()
    import torch
    import bench
    from rx_tools_b200 import _lib, fm, synth
    lib = _lib.lib()
    if not hasattr(lib, "rxb200_fm_prof_read"):
        sys.exit("this librxb200.so was built without -DRXB_PROF")
    lib.rxb200_fm_prof_read.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    n_per = (args.size_mib << 20) // 4
    period = min(n_per, 1 << 24)
    x = torch.from_numpy(synth.cfg2_iq(period)).cuda().repeat(n_per // period).contiguous()
    n_int16 = x.numel()
    d = fm.FmDemod(bench.fm_params("fm2b"))
    cap = d.max_output(n_int16, bench.CHUNK) + 8
    out = torch.empty(cap, dtype=torch.int16, device="cuda")
    if args.timeline:
        timeline(lib, d, x, out, cap)
        d.close()
        return
    d.process_device(x.data_ptr(), n_int16, bench.CHUNK, out.data_ptr(), cap, sync=True)
    _lib.check(lib.rxb200_fm_prof_read(None, 0, 1))
    d.process_device(x.data_ptr(), n_int16, bench.CHUNK, out.data_ptr(), cap, sync=True)
    st = d.stats()
    buf = np.zeros(PROF_CTAS * 32 * PROF_SLOTS, dtype=np.uint64)
    _lib.check(lib.rxb200_fm_prof_read(buf.ctypes.data, buf.size, 0))
    a = buf.reshape(PROF_CTAS, 32, PROF_SLOTS).astype(np.float64)
    ctas = int((a[:, :, PF_ITEMS].sum(axis=1) > 0).sum())
    a = a[:ctas]
    warps = int((a[:, :, PF_ITEMS].sum(axis=0) > 0).sum())
    print(f"kernel_kind {st['kernel_kind']}, item {st['segment_len'] // 1024} rows, {ctas} CTAs x {warps} warps, "
          f"kernel {d.kernel_ms():.3f} ms")
    items = a[:, :, PF_ITEMS]
    be = [w for w in range(warps) if a[:, w, PF_ROWS].sum() == 0 and a[:, w, PF_FULL].sum() > 0]
    print("warp  %warpid%4 over CTAs          items  cycles/item  " + "  ".join(f"{n:>10}" for n, _ in FE_COLS + BE_COLS)
          + "  cycles/row")
    per_smsp = collections.defaultdict(lambda: [0.0, 0.0])
    for w in range(warps):
        sm = collections.Counter((a[:, w, PF_WARPID].astype(np.int64) % 4).tolist())
        smsp = ",".join(f"{k}:{v}" for k, v in sorted(sm.items()))
        it = items[:, w].sum()
        cols = [a[:, w, s].sum() / it for _, s in FE_COLS + BE_COLS]
        rows = a[:, w, PF_ROWS].sum()
        cpr = (a[:, w, PF_FRONT].sum() - a[:, w, PF_RING].sum()) / rows if rows else float("nan")
        if rows:
            s0 = sm.most_common(1)[0][0]
            per_smsp[s0][0] += a[:, w, PF_FRONT].sum() - a[:, w, PF_RING].sum()
            per_smsp[s0][1] += rows
        print(f"{w:4d}{' BE' if w in be else '   '} {smsp:<24} {it / ctas:6.1f} {a[:, w, PF_TOTAL].sum() / it:12.0f}  "
              + "  ".join(f"{c:10.1f}" if i == 0 else f"{c:10.0f}" for i, c in enumerate(cols)) + f"  {cpr:10.0f}")
    for s in sorted(per_smsp):
        print(f"SMSP {s}: front-end cycles per row (ring wait excluded) {per_smsp[s][0] / per_smsp[s][1]:.0f}")
    wid = a[:, :warps, PF_WARPID].astype(np.int64)
    print("warp slot = %warpid - 8 * (CTA's SM slot):", bool(((wid % 8) == np.arange(warps) % 8).all()) if warps <= 8 else
          bool(((wid % 16) == np.arange(warps)).all()))
    d.close()


if __name__ == "__main__":
    main()
