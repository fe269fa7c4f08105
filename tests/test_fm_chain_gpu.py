"""Back-to-back calls on one handle: the split kernel of a call may start while the previous call on the handle drains
(programmatic dependent launch), and its ticket, publish and margin words are reused by call parity without being
cleared.  Every case makes its calls through the device entry points with sync=False, one after the other, and holds
the outputs to the same calls made with a synchronise after each one, and to the port over the same chunk sequence."""
import numpy as np
import pytest

from cases import fm_cases
from fm_any_chunk import port_run_seq
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

CHUNK = 16384                    # int16 per chunk: 8 rows of the row front end


def _case(name):
    return next(c for c in fm_cases() if c.name == name)


def _plan(calls, chunk):
    """calls: ("p", n_int16) for process_device with `chunk`, ("r", n_int16) for one read.  Returns the chunk lengths
    (int16) of the whole sequence, for the port."""
    lens = []
    for kind, n in calls:
        lens += [n] if kind == "r" else [min(chunk, n - p) for p in range(0, n, chunk)]
    return lens


class _Run:
    """One handle's calls: inputs staged per call (so every call's input is aligned), outputs per call or one reused."""

    def __init__(self, torch, params, xs, calls, chunk, tune=0, reuse_out=False):
        self.n_ch = xs.shape[0]
        self.d = fm.FmDemod(params, device=0, n_channels=self.n_ch)
        if tune:
            self.d.tune(segment_len=tune)
        self.calls, self.chunk, self.reuse = calls, chunk, reuse_out
        self.ins, pos = [], 0
        for _, n in calls:
            self.ins.append(torch.from_numpy(np.ascontiguousarray(xs[:, pos:pos + n])).cuda())
            pos += n
        self.caps = [self.d.max_output(n, n if kind == "r" else chunk) + 8 for kind, n in calls]
        cap = max(self.caps)
        n_out = 1 if reuse_out else len(calls)
        self.outs = [torch.zeros(self.n_ch * cap, dtype=torch.int16, device="cuda") for _ in range(n_out)]
        self.cap = cap
        self.n_pcm, self.fixups, self.kinds = [], [], []
        torch.cuda.synchronize()

    def call(self, i, sync):
        kind, n = self.calls[i]
        out = self.outs[0 if self.reuse else i]
        if kind == "r":
            k = self.d.process_read_device(self.ins[i].data_ptr(), n, out.data_ptr(), self.cap, sync=sync)
        else:
            k = self.d.process_device(self.ins[i].data_ptr(), n, self.chunk, out.data_ptr(), self.cap, sync=sync)
        self.n_pcm.append(k)
        if sync:
            st = self.d.stats()
            self.fixups.append(st["fixup_segments"])
            self.kinds.append(st["kernel_kind"])

    def pcm(self, i):
        """channel-major PCM of call i (after the run has synchronised)"""
        out = self.outs[0 if self.reuse else i].view(self.n_ch, self.cap)
        return out[:, :self.n_pcm[i]].cpu().numpy()

    def all_pcm(self):
        return np.concatenate([self.pcm(i) for i in range(len(self.calls))], axis=1)

    def close(self):
        self.d.close()


def _both(torch, params, xs, calls, chunk, tune=0, reuse_out=False):
    """the calls chained (sync=False throughout), then the same calls with a synchronise after each"""
    a = _Run(torch, params, xs, calls, chunk, tune, reuse_out)
    for i in range(len(calls)):
        a.call(i, False)
    torch.cuda.synchronize()
    b = _Run(torch, params, xs, calls, chunk, tune, reuse_out)
    for i in range(len(calls)):
        b.call(i, True)
    return a, b


def _inputs(name, n_ch, total):
    x = _case(name).make_input()
    reps = -(-total // x.size)
    x = np.tile(x, reps)
    return np.stack([np.roll(x, 2 * 977 * c)[:total] for c in range(n_ch)])


def _check_port(port, params, xs, calls, chunk, got):
    lens = _plan(calls, chunk)
    for c in range(xs.shape[0]):
        want = port_run_seq(port, params, xs[c, :sum(n for _, n in calls)], lens)
        assert np.array_equal(got[c], want), f"channel {c}: {np.count_nonzero(got[c] != want)} samples differ"


@pytest.fixture(scope="module")
def torch():
    import torch as t
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


@pytest.mark.parametrize("reuse_out", [False, True], ids=["own_outputs", "one_output"])
@pytest.mark.parametrize("tune", [0, 4096], ids=["planned_items", "short_items"])
def test_chain_matches_synced_and_port(torch, port, tune, reuse_out):
    """fm2b's shape, back to back, as bench.py calls it (one output buffer every call) and with an output per call.
    Short items (4 rows) give each call many items, so the look-back and the margin hand-over run in every call."""
    case = _case("cfg2B")
    calls = [("p", 4 * CHUNK)] * 14
    xs = _inputs("cfg2B", 1, sum(n for _, n in calls))
    a, b = _both(torch, case.params, xs, calls, CHUNK, tune, reuse_out)
    assert all(k == 1 for k in b.kinds), b.kinds
    if reuse_out:
        last = a.pcm(len(calls) - 1)
        assert np.array_equal(last, b.pcm(len(calls) - 1))
        want = port_run_seq(port, case.params, xs[0], _plan(calls, CHUNK))
        assert np.array_equal(last[0], want[want.size - last.shape[1]:])
    else:
        assert np.array_equal(a.all_pcm(), b.all_pcm())
        _check_port(port, case.params, xs, calls, CHUNK, a.all_pcm())
    a.close(); b.close()


def test_chain_long_calls(torch, port):
    """bench.py's chunk (131072 complex) and one chunk per call, planned items, one reused output"""
    case = _case("cfg2B")
    calls = [("p", 262144)] * 6
    xs = _inputs("cfg2B", 1, sum(n for _, n in calls))
    a, b = _both(torch, case.params, xs, calls, 262144, reuse_out=True)
    assert all(k == 1 for k in b.kinds), b.kinds
    assert np.array_equal(a.pcm(5), b.pcm(5))
    c = _Run(torch, case.params, xs, calls, 262144)           # every call's output, chained
    for i in range(len(calls)):
        c.call(i, False)
    torch.cuda.synchronize()
    _check_port(port, case.params, xs, calls, 262144, c.all_pcm())
    assert 0.0 < c.d.kernel_ms() < 100.0          # the split kernel's own stamps: the last call's device time
    a.close(); b.close(); c.close()


def test_chain_quiet_input_fixups(torch, port):
    """burst then silence: de-emphasis brackets stay open, so the look-back, the serial fix-up and fix_count run in
    chained calls; the last call's fix-up count is that call's alone"""
    case = _case("burst_then_silence")
    calls = [("p", 4 * CHUNK)] * 14
    xs = _inputs("burst_then_silence", 1, sum(n for _, n in calls))
    a, b = _both(torch, case.params, xs, calls, CHUNK, tune=4096)
    assert all(k == 1 for k in b.kinds), b.kinds
    assert max(b.fixups) > 0, b.fixups
    assert a.d.stats()["fixup_segments"] == b.fixups[-1]
    assert np.array_equal(a.all_pcm(), b.all_pcm())
    _check_port(port, case.params, xs, calls, CHUNK, a.all_pcm())
    a.close(); b.close()


def test_chain_channels(torch, port):
    """three channels per call"""
    case = _case("cfg2B")
    calls = [("p", 4 * CHUNK)] * 10
    xs = _inputs("cfg2B", 3, sum(n for _, n in calls))
    a, b = _both(torch, case.params, xs, calls, CHUNK, tune=4096)
    assert all(k == 1 for k in b.kinds), b.kinds
    assert np.array_equal(a.all_pcm(), b.all_pcm())
    _check_port(port, case.params, xs, calls, CHUNK, a.all_pcm())
    a.close(); b.close()


def test_chain_across_kernel_kinds(torch, port):
    """split-kernel calls between calls on the fused kernel (one chunk: fewer than 16 rows) and on the any-length
    kernel (a read off the pass granule): the parity and the call tags carry across the other kernels"""
    case = _case("cfg2B")
    pattern = [("p", 4 * CHUNK), ("p", CHUNK), ("p", 4 * CHUNK), ("p", 4 * CHUNK), ("r", 2002), ("p", 4 * CHUNK),
               ("r", 4 * CHUNK), ("p", 4 * CHUNK)]
    calls = pattern * 3
    xs = _inputs("cfg2B", 1, sum(n for _, n in calls))
    a, b = _both(torch, case.params, xs, calls, CHUNK, tune=4096)
    want_kinds = {("p", 4 * CHUNK): 1, ("p", CHUNK): 0, ("r", 2002): 0, ("r", 4 * CHUNK): 1}
    assert b.kinds == [want_kinds[c] for c in calls], b.kinds
    assert np.array_equal(a.all_pcm(), b.all_pcm())
    _check_port(port, case.params, xs, calls, CHUNK, a.all_pcm())
    a.close(); b.close()


def test_chain_two_handles(torch, port):
    """two handles called in turn, each with its own stream and sync words"""
    case = _case("cfg2B")
    calls = [("p", 4 * CHUNK)] * 10
    total = sum(n for _, n in calls)
    x1 = _inputs("cfg2B", 1, total)
    x2 = _inputs("burst_then_silence", 1, total)
    r1 = _Run(torch, case.params, x1, calls, CHUNK, tune=4096)
    r2 = _Run(torch, case.params, x2, calls, CHUNK, tune=4096)
    for i in range(len(calls)):
        r1.call(i, False)
        r2.call(i, False)
    torch.cuda.synchronize()
    _check_port(port, case.params, x1, calls, CHUNK, r1.all_pcm())
    _check_port(port, case.params, x2, calls, CHUNK, r2.all_pcm())
    r1.close(); r2.close()
