"""The launch rules of fm_mix.cu restated, so that a test can say which regime of a kernel it reaches and assert it, and a
DDC model that scales to captures too long to mix in full in numpy.

mix_launch caps fm_mix_kernel's grid at n_sm * per_sm / groups CTAs per grid row (blockIdx.y, 256 channels each), and
every CTA strides over the capture; per_sm <= 2048 / MIX_THREADS = 8, so a lower bound on the trips every CTA makes
needs no occupancy query.  ddc_launch picks U outputs per CTA as the least of the staging room (DDC_SPAN samples), the
reach of the mixer's table offsets (DDC_REACH samples) and an even share of the outputs over 2 * n_sm / groups CTAs;
ddc_regime is that rule line for line, and names the term that wins.

ddc_sparse computes fm_ddc.ddc_model's outputs bit for bit but mixes only the samples the windows at the emission points
cover, gathered with torch indexing on whatever device holds the capture.
"""
import numpy as np

MIX_THREADS = 256
MIX_UNIT = 8                     # complex samples per thread and trip
MIX_GROUP = 256                  # channels per grid row
MIX_SMEM_MAX = 96 * 1024         # the largest table range a CTA stages in shared memory
MAX_THREADS_PER_SM = 2048
DDC_SPAN = 8192
DDC_REACH = 1 << 20


def groups(n_ch):
    """Grid rows of a call on n_ch channels (both kernels)."""
    return -(-n_ch // MIX_GROUP)


def mix_trips_at_least(n, n_groups, n_sm):
    """The fewest grid-stride trips any CTA of any grid row of fm_mix_kernel makes on n complex samples, at any
    occupancy: the grid row has bx <= n_sm * 8 / groups CTAs of 256 threads, one MIX_UNIT per thread and trip, and its
    last CTA starts (bx - 1) * 256 units in."""
    units = -(-n // MIX_UNIT)
    bx = max(1, n_sm * (MAX_THREADS_PER_SM // MIX_THREADS) // n_groups)
    return max(1, -(-(units - (bx - 1) * MIX_THREADS) // (bx * MIX_THREADS)))


def mix_uses_smem(periods):
    """Whether mix_launch stages the tables in shared memory: the largest grid row's table range (its channels' periods,
    concatenated in channel order) fits MIX_SMEM_MAX bytes of (c, s) int32 pairs."""
    periods = list(periods)
    rows = [sum(periods[g:g + MIX_GROUP]) for g in range(0, len(periods), MIX_GROUP)]
    return max(rows) * 8 <= MIX_SMEM_MAX


def ddc_span(M, T):
    """The most outputs one CTA's DDC_SPAN staged samples hold: windows of T samples, staged M apart when T >= M, else
    T apart."""
    ws = M if T >= M else T
    return (DDC_SPAN - T) // ws + 1


def ddc_lanes(T):
    """Lanes per output: the least power of two >= T, at most 32."""
    lanes = 1
    while lanes < 32 and lanes < T:
        lanes <<= 1
    return lanes


def ddc_regime(n_out, M, T, n_ch, n_sm, rows=None):
    """ddc_launch's outputs per CTA for n_out > 0 outputs per channel: (U, which), which is "span" (the staging room),
    "reach" (the table offsets) or "n_out" (the even share of the outputs) -- the term that sets U.  rows: the grid rows
    of a policy that plans its own (ddc_launch's rows; None: one per MIX_GROUP channels)."""
    span = ddc_span(M, T)
    reach = (DDC_REACH - T) // M + 1
    ctas = ddc_ctas(n_ch, n_sm, rows)
    share = (n_out + ctas - 1) // ctas
    bound = min(span, reach)
    U = max(1, min(bound, share))
    if share < bound:
        return U, "n_out"
    return U, "span" if span <= reach else "reach"


def ddc_ctas(n_ch, n_sm, rows=None):
    """CTAs per grid row ddc_launch shares the outputs over (rows as ddc_regime)."""
    g = rows if rows else groups(n_ch)
    return max(1, (2 * n_sm + g - 1) // g)


def device_sms():
    """The SM count the launch rules use: cudaDevAttrMultiProcessorCount of device 0."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wrap16(v):
    return ((v + 32768) & 0xffff) - 32768


def ddc_sparse(x, table, taps, decim, shift, pos=0, hist=None, table_phase=None, block=1 << 21):
    """fm_ddc.ddc_model over one call, computing only the windows at the emission points: x is the call's capture as
    int16[2c] (a numpy array or a torch tensor on any device), the rest as ddc_model.  Returns (int16[2 * n_out] numpy,
    the new history as int16[2(T - 1)] numpy)."""
    import torch
    xt = torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x).reshape(-1, 2)
    dev = xt.device
    taps = np.asarray(taps, dtype=np.int64).reshape(-1)
    T, M, H = taps.size, int(decim), taps.size - 1
    h = (torch.zeros((H, 2), dtype=torch.int16, device=dev) if hist is None
         else torch.as_tensor(np.asarray(hist, dtype=np.int16)).reshape(-1, 2).to(dev))
    assert h.shape[0] == H
    tp = pos if table_phase is None else table_phase
    tab = torch.as_tensor(np.asarray(table, dtype=np.int64)).to(dev)
    L = tab.shape[0]
    c = xt.shape[0]
    m0, m1 = pos // M, (pos + c) // M
    e = torch.arange(m0, m1, dtype=torch.int64, device=dev) * M + (M - 1 - pos)      # local emission points
    hr = torch.as_tensor(taps[::-1].copy()).to(dev)
    span = torch.arange(T, dtype=torch.int64, device=dev) - H
    out = torch.empty((e.numel(), 2), dtype=torch.int64, device=dev)
    per = max(1, block // T)
    for a in range(0, e.numel(), per):
        j = e[a:a + per, None] + span                                  # capture index of each window sample, >= -H
        raw = xt[j.clamp(min=0)].to(torch.int64)
        if H:
            raw = torch.where((j >= 0)[..., None], raw, h[(j + H).clamp(max=H - 1)].to(torch.int64))
        k = torch.remainder(tp + j, L)
        cc, ss = tab[k, 0], tab[k, 1]
        zi = _wrap16((raw[..., 0] * cc - raw[..., 1] * ss + (1 << 14)) >> 15)
        zq = _wrap16((raw[..., 0] * ss + raw[..., 1] * cc + (1 << 14)) >> 15)
        out[a:a + per, 0] = (zi * hr).sum(-1)
        out[a:a + per, 1] = (zq * hr).sum(-1)
    y = out if shift == 0 else (out + (1 << (shift - 1))) >> shift
    y = y.clamp(-32768, 32767).to(torch.int16).reshape(-1).cpu().numpy()
    if H == 0:
        return y, np.zeros(0, np.int16)
    tail = torch.cat([h, xt[max(0, c - H):]])[-H:]
    return y, tail.reshape(-1).cpu().numpy()


def sparse_reads(x, table, ddc, lens16, table_phase=0):
    """The decimated stream of each read of a read sequence over a capture from create or reset (zero history), in
    order: the outputs of the whole capture at once, split by the emission points each read holds.  x as ddc_sparse."""
    import fm_any_chunk as fac
    import fm_ddc as fdd
    decim, taps, shift = ddc
    n16 = int(x.numel() if hasattr(x, "numel") else np.asarray(x).size)
    y, _ = ddc_sparse(x, table, taps, decim, shift, table_phase=table_phase)
    out, pos, at = [], 0, 0
    for _, n in fac.seq_bounds(n16, lens16):
        d = fdd.decimated_len(pos, n, decim)
        out.append(y[at:at + d])
        at += d
        pos += n // 2
    assert at == y.size
    return out
