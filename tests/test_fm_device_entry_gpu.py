"""rxb200_fm_process_device -- the entry point bench.py times -- against the port: caller-chosen output strides around
a canary-filled buffer, an input that is 32-byte but not 256-byte aligned, bench's loop of sync = 0 calls on one
handle, refusals that must leave the stream's carry alone, and calls that alternate with the host entry point.  Plus
rx_power's device entry point from a 16-byte aligned tensor."""
import numpy as np
import pytest
import torch

import fm_paths
import oracle
from rx_tools_b200 import _lib, fm, power, synth

pytestmark = pytest.mark.gpu

CANARY = -21555                     # 0xabcd
CHUNK = 262144
N_CH = 3

# one handle per kernel: (params, int16 per channel and call -- a whole number of chunks, so that calls end on chunk
# boundaries --, chunk, kernel_kind)
HANDLES = {
    "rows": (fm.FmParams(downsample=8, downsample_passes=3, comp_fir_size=9, custom_atan=fm.ATAN_FAST, deemph=1,
                         deemph_a=23, rate_out=300_000, rate_out2=48_000), 64 * fm_paths.ROW_I16, 16 * fm_paths.ROW_I16, 1),
    "stream": (fm.FmParams(downsample=1, custom_atan=fm.ATAN_FAST, deemph=1, deemph_a=181, rate_out=2_400_000,
                           rate_out2=48_000), 2 * 65536, 32768, 3),
    "spec3": (fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24_000), 2 * 100_000, 20_000, 0),
    "spec2_squelch": (fm.FmParams(downsample=8, downsample_passes=3, comp_fir_size=9, custom_atan=fm.ATAN_FAST, deemph=1,
                                  deemph_a=23, rate_out=300_000, rate_out2=48_000, squelch_level=60), 2 * 60_000, 8000, 0),
    "spec0": (fm.FmParams(downsample=6, custom_atan=fm.ATAN_ALE, deemph=1, deemph_a=13, rate_out=170_000,
                          rate_out2=32_000, offset_tuning=1), 2 * 60_000, 12_000, 0),
}


def _op(p):
    return oracle.FmParams(**p.reference_fields())


def _inputs(n16, seed, n_ch=N_CH):
    rng = np.random.default_rng(seed)
    xs = [fm_paths.channel_input(rng, k, n16 // 2, s) for k, s in (("loud", False), ("quiet", True), ("loud", True))]
    xs[n_ch - 1][n16 // 3:n16 // 2] = 0
    return np.stack(xs[:n_ch])


def _device_input(x, offset_bytes):
    """x (int16 [n_ch][n]) on the device, offset_bytes into a larger allocation."""
    off = offset_bytes // 2
    buf = torch.zeros(x.size + off + 64, dtype=torch.int16, device="cuda")
    buf[off:off + x.size] = torch.from_numpy(x.reshape(-1)).cuda()
    view = buf[off:off + x.size]
    assert view.data_ptr() % 256 == offset_bytes % 256
    return buf, view


def _port(port, p, x, chunk):
    return np.stack([port.fm_run(_op(p), x[c], chunk) for c in range(x.shape[0])])


@pytest.mark.parametrize("name", sorted(HANDLES))
def test_strides_canary_and_alignment(name, port):
    """pcm_stride of total, total + 1 (odd), total + 13 and max_output + 8 around a canary-filled buffer; the input 32
    bytes into its allocation."""
    p, n16, chunk, kind = HANDLES[name]
    x = _inputs(n16, 1)
    want = _port(port, p, x, chunk)
    total = want.shape[1]
    d = fm.FmDemod(p, n_channels=N_CH)
    _, dx = _device_input(x, 32)
    for stride in (total, total + 1, total + 13, d.max_output(n16, chunk) + 8):
        d.reset()
        out = torch.full((N_CH * stride + 97,), CANARY, dtype=torch.int16, device="cuda")
        assert d.process_device(dx.data_ptr(), n16, chunk, out.data_ptr(), stride, sync=True) == total
        assert d.stats()["kernel_kind"] == kind
        h = out.cpu().numpy()
        mask = np.ones(h.size, dtype=bool)
        for c in range(N_CH):
            assert np.array_equal(h[c * stride:c * stride + total], want[c]), (name, stride, c)
            mask[c * stride:c * stride + total] = False
        assert np.all(h[mask] == CANARY), (name, stride, np.flatnonzero(h[mask] != CANARY)[:5])
    d.close()


@pytest.mark.parametrize("workload", ["fm2b", "fm5a"])
def test_bench_loop_of_async_calls(workload, port):
    """bench.py's timed loop: K = 4 calls with sync = 0 on one input into four outputs, one synchronize at the end."""
    if workload == "fm2b":
        p = fm.derive_params(wbfm=1, rate_s=300_000, rate_r=48_000, use_F=1, comp_fir_size=9).params
        n_ch, n = 1, 8 << 20                             # 32 MiB
        x = synth.cfg2_iq(n).reshape(1, -1)
        kind = 1
    else:
        p = fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24_000)
        n_ch, n = 8, 9 * CHUNK // 2                      # 8 x 4.7 MB, whole chunks: calls end on chunk boundaries
        x = np.stack([synth.cfg5_iq(n, c) for c in range(n_ch)])
        kind = 0
    n16 = x.shape[1]
    d = fm.FmDemod(p, n_channels=n_ch)
    cap = d.max_output(n16, CHUNK) + 8
    dx = torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).cuda()
    outs = [torch.empty(n_ch * cap, dtype=torch.int16, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    counts = [d.process_device(dx.data_ptr(), n16, CHUNK, o.data_ptr(), cap, sync=False) for o in outs]
    torch.cuda.synchronize()
    assert d.stats()["kernel_kind"] == kind
    for c in range(n_ch):
        want = port.fm_run(_op(p), np.tile(x[c], 4), CHUNK)
        got = np.concatenate([o.view(n_ch, cap)[c, :k].cpu().numpy() for o, k in zip(outs, counts)])
        assert got.size == want.size and np.array_equal(got, want), (workload, c, np.flatnonzero(got != want)[:5])
    d.close()


@pytest.mark.parametrize("name", sorted(HANDLES))
def test_refusals_leave_the_stream_alone(name, port):
    p, n16, chunk, kind = HANDLES[name]
    x = np.concatenate([_inputs(n16, 3), _inputs(n16, 4)], axis=1)
    want = _port(port, p, x, chunk)
    d = fm.FmDemod(p, n_channels=N_CH)
    cap = d.max_output(n16, chunk) + 8
    parts = []
    for i in range(2):
        buf, dx = _device_input(np.ascontiguousarray(x[:, i * n16:(i + 1) * n16]), 32)
        out = torch.empty(N_CH * cap, dtype=torch.int16, device="cuda")
        k = d.process_device(dx.data_ptr(), n16, chunk, out.data_ptr(), cap, sync=True)
        parts.append(out.view(N_CH, cap)[:, :k].cpu().numpy())
        if i == 0:
            _, bad = _device_input(np.ascontiguousarray(x[:, n16:]), 16)
            with pytest.raises(_lib.Rxb200Error) as e:
                d.process_device(bad.data_ptr(), n16, chunk, out.data_ptr(), cap, sync=True)
            assert e.value.code == _lib.EINVAL
            with pytest.raises(_lib.Rxb200Error) as e:
                d.process_device(dx.data_ptr(), n16, chunk, out.data_ptr(), k - 1, sync=True)
            assert e.value.code == _lib.ECAPACITY
    got = np.concatenate(parts, axis=1)
    assert np.array_equal(got, want), name
    d.close()


@pytest.mark.parametrize("name", ["rows", "stream", "spec3"])
def test_device_and_host_calls_alternate(name, port):
    p, n16, chunk, kind = HANDLES[name]
    x = np.concatenate([_inputs(n16, 5 + i) for i in range(4)], axis=1)
    want = _port(port, p, x, chunk)
    d = fm.FmDemod(p, n_channels=N_CH)
    cap = d.max_output(n16, chunk) + 8
    parts = []
    for i in range(4):
        part = np.ascontiguousarray(x[:, i * n16:(i + 1) * n16])
        if i % 2 == 0:
            dx = torch.from_numpy(part.reshape(-1)).cuda()
            out = torch.empty(N_CH * cap, dtype=torch.int16, device="cuda")
            k = d.process_device(dx.data_ptr(), n16, chunk, out.data_ptr(), cap, sync=False)
            torch.cuda.synchronize()
            parts.append(out.view(N_CH, cap)[:, :k].cpu().numpy())
        else:
            parts.append(d.full_demod(part, chunk))
        assert d.stats()["kernel_kind"] == kind
    assert np.array_equal(np.concatenate(parts, axis=1), want), name
    d.close()


def test_power_scanner_device_offset_input(port):
    """PowerScanner.scanner_device from a tensor 16 bytes into its allocation, sync = 0, over two hop sub-ranges."""
    plan = power.plan_range("24M:60M:1k", 0.285)
    assert plan.n_hops > 3
    win = power.window_table("hamming", 1 << plan.bin_e)
    n_pass = 3
    x = synth.power_hops(n_pass, plan.n_hops, plan.buf_len, seed=91)
    pp = oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len, downsample=plan.downsample,
                            downsample_passes=plan.downsample_passes, comp_fir_size=plan.comp_fir_size,
                            boxcar=plan.boxcar, peak_hold=plan.peak_hold)
    want, wsmp = port.power_scan(pp, win, x, n_pass, plan.n_hops)
    sc = power.PowerScanner(plan, win)
    split = plan.n_hops // 3
    keep = []
    for a, b in [(0, split), (split, plan.n_hops)]:
        buf, dx = _device_input(np.ascontiguousarray(x[:, a:b]), 16)
        keep.append(buf)
        sc.scanner_device(dx.data_ptr(), n_pass, a, b, sync=False)
    torch.cuda.synchronize()
    avg, smp = sc.read()
    assert np.array_equal(smp, wsmp) and np.array_equal(avg, want)
    sc.close()
