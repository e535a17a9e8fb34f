"""bench.py's device-resident duplex schedule (measure -> run_device, the non-serial branch), written once for the GPU tests that
tie it to the oracle and for tools/schedule_bench.py.

Each group is an encoder-only and a decoder-only context of m streams, installed on CUDA streams of their own at priorities
-1 / 0, over rows [g*m, (g+1)*m) of shared input, packet and output buffers.  Hop i uses slot i % 8: its encode waits until
the slot's previous packets have been decoded, its decode waits for its packets through an event, and nothing synchronises
the host.  The decode_plc workload runs decode_plc_device on the decoder contexts alone, over caller-supplied packets and
received masks.  With `dtx` the encoders run encode_dtx_device into a flag buffer per slot, and the decoders take a DTX hop as a
lost packet: received = 1 - flag, computed on the decoder's CUDA stream.  With `mask` every context reads the active mask of
hop i from pattern i % len(mask) (lyra_b200_set_active_mask): a stream that sits out a hop is neither encoded nor decoded.
"""
import numpy as np
import torch

from lyra_b200 import _capi

NBUF = 8


def _row(t, g, m):
    """Device address of row g * m of a contiguous tensor."""
    return t.data_ptr() + g * m * t.stride(0) * t.element_size()


class Schedule:
    def __init__(self, slots, groups, split, mode, bits=64, rate=16000, stream_rates=None, masks=None, keep_hops=0, stream_bits=None,
                 dtx=None, mask=None, realign=0):
        """slots: NBUF host arrays of n rows, the input PCM (rate // 50 samples per row), or with `masks` (the decode_plc
        workload) the packets; masks: NBUF received masks of n entries.  stream_rates: the per-stream rates of every group's
        m streams; stream_bits: their per-stream bit counts (both roles, at most `bits`); dtx: their DTX settings (1 on, 0 off;
        None: no DTX, encode_device).  keep_hops: hop i < keep_hops writes its own output (and flag) buffer and keeps a copy of
        its packets (and DTX flags), and the schedule runs at most keep_hops hops; with 0 every hop writes one shared output.
        mask: active-mask patterns of n entries each (0 = the stream sits the hop out), hop i uses pattern i % len(mask) on both
        contexts of every group; realign > 0: every `realign` hops both contexts align every stream with the first stream of its
        tile (lyra_b200_align_streams), so tiles whose lanes sat out different hops are back on one hop counter."""
        n = len(slots[0])
        self.n, self.m, self.bits, self.keep_hops = n, n // groups, bits, keep_hops
        self.plc = masks is not None
        self.dtx = dtx is not None
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
        if self.plc:
            self.pks, self.masks = [dev(x) for x in slots], [dev(x) for x in masks]
        else:
            self.pcm = [dev(x) for x in slots]
            self.pks = [torch.zeros((n, _capi.packet_bytes(bits)), dtype=torch.uint8, device="cuda") for _ in range(NBUF)]
            self.kept_pks = [torch.zeros_like(self.pks[0]) for _ in range(keep_hops)]
        if self.dtx:                      # per slot: the encoders' DTX flags and the decoders' received masks made from them
            self.dtx_flags = [torch.zeros((n,), dtype=torch.uint8, device="cuda") for _ in range(NBUF)]
            self.received = [torch.ones((n,), dtype=torch.bool, device="cuda") for _ in range(NBUF)]     # one byte, 0 or 1
            self.kept_flags = [torch.zeros_like(self.dtx_flags[0]) for _ in range(keep_hops)]
        self.mask = None if mask is None else [dev(np.asarray(x, np.uint8)) for x in mask]
        self.realign = realign
        outs = max(keep_hops, 1)
        self.out = [torch.full((n, rate // 50), 0x5A5A, dtype=torch.int16, device="cuda") for _ in range(outs)]
        self.flags = [torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda") for _ in range(outs)] if self.plc else None
        self.groups = []
        for _ in range(groups):
            e_ = None if self.plc else _capi.Context(self.m, roles="encoder")
            d_ = _capi.Context(self.m, roles="decoder")
            gx, gy = torch.cuda.Stream(priority=-1), torch.cuda.Stream(priority=0)
            for c, prio, st in ((e_, -1, gx), (d_, 0, gy)):
                if c is None:
                    continue
                if rate != 16000:
                    c.set_sample_rate(rate)
                c.set_priority(prio)
                c.set_stream(st.cuda_stream)
                c.set_split(split)
                if stream_rates is not None:
                    c.set_stream_sample_rates(stream_rates)
                if stream_bits is not None:
                    c.set_stream_bits("encoder" if c is e_ else "decoder", stream_bits)
                if dtx is not None and c is e_:
                    c.set_stream_dtx(dtx)
            d_.set_decoder_mode(mode)
            self.groups.append((e_, d_, gx, gy))
        self.ev_pk = [[torch.cuda.Event() for _ in range(NBUF)] for _ in range(groups)]      # [group][slot] packets written
        self.ev_free = [[torch.cuda.Event() for _ in range(NBUF)] for _ in range(groups)]    # ... and consumed
        torch.cuda.synchronize()          # the buffers above were filled on the current stream, the settings on the groups'

    def hop(self, i):
        """Hop i of every group."""
        b, o, m, bits = i % NBUF, i if self.keep_hops else 0, self.m, self.bits
        for g, (e_, d_, gx, gy) in enumerate(self.groups):
            pk, out = _row(self.pks[b], g, m), _row(self.out[o], g, m)
            if self.plc:
                d_.decode_plc_device(m, pk, _row(self.masks[b], g, m), bits, out, _row(self.flags[o], g, m))
                continue
            if i >= NBUF:
                gx.wait_event(self.ev_free[g][b])
            rows = slice(g * m, (g + 1) * m)
            if self.mask is not None:
                p = _row(self.mask[i % len(self.mask)], g, m)
                e_.set_active_mask(p)
                d_.set_active_mask(p)
                if self.realign and i and i % self.realign == 0:
                    t = e_.tile_streams
                    ids = np.array([k for k in range(m) if k % t], np.int32)
                    for c in (e_, d_):
                        c.align_streams(ids, ids // t * t)
            if self.dtx:
                e_.encode_dtx_device(m, _row(self.pcm[b], g, m), bits, pk, _row(self.dtx_flags[b], g, m))
            else:
                e_.encode_device(m, _row(self.pcm[b], g, m), bits, pk)
            self.ev_pk[g][b].record(gx)
            gy.wait_event(self.ev_pk[g][b])
            rec = 0
            if self.dtx:
                with torch.cuda.stream(gy):                # a DTX hop reaches the decoder as a lost packet
                    torch.eq(self.dtx_flags[b][rows], 0, out=self.received[b][rows])
                rec = _row(self.received[b], g, m)
            d_.decode_device(m, pk, rec, bits, out)
            if self.keep_hops:
                with torch.cuda.stream(gy):                # before the slot is reused
                    self.kept_pks[i][rows].copy_(self.pks[b][rows])
                    if self.dtx:
                        self.kept_flags[i][rows].copy_(self.dtx_flags[b][rows])
            self.ev_free[g][b].record(gy)

    def close(self):
        for e_, d_, _, _ in self.groups:
            for c in (e_, d_):
                if c is not None:
                    c.close()


def run(schedules, hops):
    """Hops 0 .. hops-1, the schedules interleaved hop by hop."""
    for i in range(hops):
        for s in schedules:
            s.hop(i)


def timed(schedules, hops):
    """Frames/s of run(schedules, hops), timed with CUDA events on a timer stream that every work stream forks from and joins
    into: nothing of the run starts before the first event, and the second waits for all of it."""
    timer = torch.cuda.Stream()
    work = [st for s in schedules for grp in s.groups for st in grp[2:]]
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(timer)
    for st in work:
        st.wait_stream(timer)
    run(schedules, hops)
    for st in work:
        timer.wait_stream(st)
    e1.record(timer)
    torch.cuda.synchronize()
    return sum(s.n for s in schedules) * hops / (e0.elapsed_time(e1) / 1e3)
