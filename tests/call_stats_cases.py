"""Cases for the per-stream call statistics of the fused codec calls (lyra_b200_set_stats / _read_stats / _read_stats_device),
shared by the CPU tier (emulated kernels) and the GPU tier.  `Model` restates the counting rules in numpy and is fed from what
each call returned: the input rows (encoders), the output PCM (decoders; levels are computed from the returned samples, so both
decoder modes are exact), packet_bytes / DTX flags, the received masks and, for decode_plc, the plan reconstructed from
plc_get_state before the hop and the received byte.  The library's statistics must equal the model's word for word."""
import math

import numpy as np

import active_mask_cases as am
import call_schedule_cases as cs
import mixed_rate_cases as mc
import rate_cases as rc
import stream_dtx_cases as dc
from parity_cases import Guarded

EINVAL = -1
KINDS = am.KINDS
W = 8                                        # LYRA_B200_STATS_WORDS
HOPS, SAT_OUT, ENERGY, LEVEL, EMPTY, BITS, RECEIVED, CN_HOPS, EVENTS = 0, 1, 2, 3, 4, 5, 4, 5, 6
COUNTERS = [HOPS, SAT_OUT, ENERGY, 4, 5, 6]  # what clear zeroes
# RFC 6464 thresholds, as the library computes them on the host (the same libm)
THRESHOLDS = np.array([2.0 ** 30 * math.pow(10.0, -(k + 0.5) / 10.0) for k in range(127)])
PLC_CONCEAL, PLC_FADE = 1280, 640


def level_energy(row):
    """(RFC 6464 level, floor(sum of squares / samples)) of one hop"""
    sq = int(np.sum(np.asarray(row, np.int64) ** 2))
    msq = sq / len(row)
    return int(np.count_nonzero(THRESHOLDS > msq)), sq // len(row)


def plc_plan(state, rec):
    """(received, comfort noise in the output) of a decode_plc hop from the stream's control state before it (PlcPlanKernel)"""
    cp, fp, d = (int(v) for v in state)
    if rec and cp > 0:
        cp = 0
    got = bool(rec) and cp == 0
    if got:
        d = -1
    elif cp == PLC_CONCEAL:
        d = 1
    return got, not (d == -1 and fp == 0)


class Model:
    """The statistics of one role of one context, by stream id"""

    def __init__(self, max_streams):
        self.w = np.zeros((max_streams, W), np.uint64)
        self.w[:, LEVEL] = 127
        self.prev = np.ones(max_streams, bool)      # the private word: the last run hop was received

    def _run(self, s, row):
        lv, en = level_energy(row)
        self.w[s, HOPS] += 1
        self.w[s, ENERGY] += np.uint64(en)
        self.w[s, LEVEL] = lv

    def encode(self, s, row, empty, bits):
        self._run(s, row)
        if empty:
            self.w[s, EMPTY] += 1
        else:
            self.w[s, BITS] += np.uint64(bits)

    def decode(self, s, row, received, cn=False):
        self._run(s, row)
        self.w[s, RECEIVED] += int(received)
        self.w[s, CN_HOPS] += int(cn)
        if not received and self.prev[s]:
            self.w[s, EVENTS] += 1
        self.prev[s] = received

    def sat_out(self, s):
        self.w[s, SAT_OUT] += 1

    def read(self, ids, clear=False):
        out = self.w[ids].copy()
        if clear:
            for k in np.unique(ids):
                self.w[k, COUNTERS] = 0
        return out

    def copy(self, src, dst):
        for s, d in zip(src, dst):
            if s < 0:
                self.w[d] = 0
                self.w[d, LEVEL] = 127
                self.prev[d] = True
            else:
                self.w[d], self.prev[d] = self.w[s], self.prev[s]


def _same(got, want, what):
    got = np.asarray(got).view(np.uint64) if np.asarray(got).dtype == np.int64 else np.asarray(got)
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)[:6]
        raise AssertionError("%s: statistics differ from the model at (row, word) %s: got %s, want %s" % (
            what, bad.tolist(), [int(got[tuple(b)]) for b in bad], [int(want[tuple(b)]) for b in bad]))


def _extreme_rows(x, row_rate, f):
    """digital silence in stream 0 on even hops and a full-scale square wave in stream 1 on odd hops (levels 127 and 0)"""
    if len(x) > 1:
        k = f % 2
        h = int(row_rate[k]) // 50
        x[k, :h] = 0 if k == 0 else np.where(np.arange(h) % 2 == 0, 32767, -32768)
    return x


class Runner:
    """One context (and its models) driving one codec kind hop by hop through its host-buffer call (ids: None = dense, else the
    sparse ids of each hop) or its device twin (device = True; mask: the active mask of each hop or None)"""

    def __init__(self, Context, api, mem, kind, *, max_streams, n, bits=64, ctx_rate=16000, rates=None, bit_set=None, dtx=None,
                 split=None, mode="exact", stats=True, ctx=None):
        """rates, bit_set: interleaved over every stream (mixed_rate_cases.interleaved); dtx: the DTX setting of streams 0..n-1;
        ctx: run on this context (already set up) instead of a new one"""
        self.kind, self.n, self.bits = kind, n, bits
        self.encoder = kind.startswith("encode")
        every = np.arange(max_streams, dtype=np.int32)
        self.srate = mc.interleaved(max_streams, rates) if rates else np.full(max_streams, ctx_rate, np.int32)
        self.sbits = mc.interleaved(max_streams, bit_set) if bit_set else None
        self.c = ctx
        if ctx is None:
            self.c = mc._make(Context, api, max_streams, ctx_rate, mode, am.CNG_SEED, split, mem.stream)
            if rates:
                self.c.set_stream_sample_rates(self.srate, every)
            if bit_set:
                for role in ("encoder", "decoder"):
                    self.c.set_stream_bits(role, self.sbits, every)
            if dtx is not None:
                self.c.set_stream_dtx(np.asarray(dtx, np.int32), every[:n])
            if stats:
                self.c.set_stats(1)
        self.mem, self.H, self.P = mem, rc.hop_of(ctx_rate), int(dc.pbytes(bits))
        self.role = "encoder" if self.encoder else "decoder"
        self.model = Model(max_streams)
        self.d = None

    def own_bits(self, s):
        return int(self.sbits[s]) if self.sbits is not None else self.bits

    def _dev(self, rows):
        if self.d is None or self.d[0] != rows:
            m = self.mem
            self.d = (rows, Guarded(m, rows, (self.H,) if self.encoder else (self.P,), np.int16 if self.encoder else np.uint8, 0x3C),
                      Guarded(m, rows, (), np.uint8, 0x77), Guarded(m, rows, (self.P,) if self.encoder else (self.H,),
                                                                     np.uint8 if self.encoder else np.int16, 0xA5),
                      Guarded(m, rows, (), np.uint8, 0xEE), Guarded(m, rows, (), np.uint8, 0x5A))
        return self.d[1:]

    def hop(self, x, rec, ids=None, device=False, mask=None, update=True):
        """one call over x (encoder rows or packets) with received bytes rec; -> output rows; updates the model"""
        c, kind, bits = self.c, self.kind, self.bits
        rows = len(x)
        sids = np.arange(rows, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
        plan = None
        if kind == "decode_plc":
            st = c.plc_state(stream_ids=sids)
            plan = [plc_plan(st[k], rec[k]) for k in range(rows)]
        run = np.ones(rows, bool) if mask is None else mask != 0
        if device:
            d_in, d_rec, d_out, d_flags, d_mask = self._dev(rows)
            if mask is not None:
                # rows that sit out are poisoned: full-scale input, lost-packet bytes; none of them may be read
                x = x.copy()
                if self.encoder:
                    x[~run] = 32767
                d_mask.put(mask)
                c.set_active_mask(d_mask.ptr)
            d_in.put(x)
            d_rec.put(np.where(run, rec, 0))
            d_out.fill()
            d_flags.fill()
            if kind == "encode":
                c.encode_device(rows, d_in.ptr, bits, d_out.ptr)
            elif kind == "encode_dtx":
                c.encode_dtx_device(rows, d_in.ptr, bits, d_out.ptr, d_flags.ptr)
            elif kind == "decode":
                c.decode_device(rows, d_in.ptr, d_rec.ptr, bits, d_out.ptr)
            elif kind == "decode_track_noise":
                c.decode_track_noise_device(rows, d_in.ptr, d_rec.ptr, bits, d_out.ptr, d_flags.ptr)
            else:
                c.decode_plc_device(rows, d_in.ptr, d_rec.ptr, bits, d_out.ptr, d_flags.ptr)
            out, flags = d_out.get("output"), d_flags.get("flags")
            if mask is not None:
                c.set_active_mask(None)
            empty = flags.astype(bool) if kind == "encode_dtx" else np.zeros(rows, bool)
        else:
            assert mask is None
            if kind == "encode":
                out = c.encode(x, bits, stream_ids=ids)
                empty = np.zeros(rows, bool)
            elif kind == "encode_dtx":
                out, sizes = c.encode_dtx(x, bits, stream_ids=ids)
                empty = sizes == 0
            elif kind == "decode":
                out = c.decode(x, bits, stream_ids=ids, received=rec)
            elif kind == "decode_track_noise":
                out, _ = c.decode_track_noise(x, bits, stream_ids=ids, received=rec)
            else:
                out, _ = c.decode_plc(x, bits, stream_ids=ids, received=rec)
        if not update:
            return out
        for k in range(rows):
            s = int(sids[k])
            if not run[k]:
                self.model.sat_out(s)
                continue
            h = int(self.srate[s]) // 50
            if self.encoder:
                self.model.encode(s, x[k, :h], bool(empty[k]), self.own_bits(s))
            elif kind == "decode_plc":
                self.model.decode(s, out[k, :h], *plan[k])
            else:
                self.model.decode(s, out[k, :h], bool(rec[k]))
        return out

    def inputs(self, f, rng, hops, rows, sids, wavs):
        if self.encoder:
            x = dc.quiet_rows(wavs, self.srate[sids], sids, f, self.H, rng, hops)
            return _extreme_rows(x, self.srate[sids], f), np.ones(rows, np.uint8)
        x = rng.integers(0, 256, size=(rows, self.P)).astype(np.uint8)
        return x, am._received(self.kind, f, rows, rng)

    def check(self, what, ids=None):
        ids = np.arange(self.n, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
        _same(self.c.stats(self.role, stream_ids=ids), self.model.read(ids), what)

    def close(self):
        self.c.close()


def run_kind(Context, api, mem, wavs, kind, *, n, hops, max_streams=None, sparse=False, device=False, masked=False, split=None,
             mode="exact", ctx_rate=16000, rates=None, bits=64, bit_set=None, dtx=None, seed=1):
    """kind over streams 0..n-1 (dense host buffers, sparse ids in no particular order, or the device twin, with an active mask
    that changes every hop when masked) against the model, after every hop.  Also checks that the extreme rows gave levels 127
    and 0, that the DTX streams produced empty packets and that the loss bursts of decode_plc reached comfort noise."""
    max_streams = max_streams or n + 3
    R = Runner(Context, api, mem, kind, max_streams=max_streams, n=n, bits=bits, ctx_rate=ctx_rate, rates=rates, bit_set=bit_set,
               dtx=dtx, split=split, mode=mode)
    rng = np.random.default_rng(seed)
    # sparse: a shuffled subset of the streams, the same every hop (so the loss bursts of decode_plc stay on their streams)
    chosen = rng.permutation(rng.choice(max_streams, size=max(2, n // 2), replace=False)).astype(np.int32)
    for f in range(hops):
        ids = chosen if sparse else None
        sids = np.arange(n, dtype=np.int32) if ids is None else ids
        x, rec = R.inputs(f, rng, hops, len(sids), sids, wavs)
        mask = am.hop_mask(f, len(sids), rng) if masked else None
        R.hop(x, rec, ids=ids, device=device, mask=mask)
        R.check("%s hop %d" % (kind, f), ids=np.arange(max_streams, dtype=np.int32))
    w = R.model.w
    if R.encoder and not masked and not sparse:
        assert w[0, LEVEL] == 127 or w[1, LEVEL] == 0, "the extreme rows did not reach levels 127 / 0"
    if kind == "encode_dtx" and (dtx is None or any(dtx)):
        assert w[:, EMPTY].sum() > 0, "no empty DTX packet"
    if kind == "decode_plc":
        assert w[:, CN_HOPS].sum() > 0 and w[:, EVENTS].sum() > 0, "the loss bursts did not reach comfort noise"
    if masked:
        assert w[:, SAT_OUT].sum() > 0
    R.close()
    return w


def run_levels(Context, api, *, n=4):
    """Levels of known hops: silence 127, a full-scale square wave 0, and constant rows at the threshold boundaries"""
    c = Context(n, capi=api)
    c.set_stats(1)
    model = Model(n)
    rows = np.zeros((n, 320), np.int16)
    rows[1] = np.where(np.arange(320) % 2 == 0, 32767, -32768)
    rows[2] = 1                                # msq 1: -90.3 dBov, level 90
    rows[3] = 3277                             # about -20 dBov
    c.encode(rows, 64)
    for k in range(n):
        model.encode(k, rows[k], False, 64)
    got = c.stats("encoder", n=n)
    _same(got, model.read(np.arange(n)), "known levels")
    assert list(got[:2, LEVEL]) == [127, 0], got[:, LEVEL]
    assert list(got[2:, LEVEL]) == [90, 20], got[:, LEVEL]
    c.close()


def run_split_independence(Context, api, mem, wav16, *, n, hops, splits=(1, 2, 3), mode="exact"):
    """The device twins over n streams at every split give the same statistics (and the model's); decode_plc runs 16 hops so
    that its loss bursts reach comfort noise"""
    res = {}
    for kind in KINDS:
        for split in splits:
            res[(kind, split)] = run_kind(Context, api, mem, {16000: wav16}, kind, n=n, hops=16 if kind == "decode_plc" else hops,
                                          device=True, split=split, mode=mode, max_streams=n)
        for split in splits[1:]:
            assert np.array_equal(res[(kind, split)], res[(kind, splits[0])]), "%s: statistics depend on the split" % kind


def run_clear(Context, api, mem, wavs, kind, *, n, hops, seed=3):
    """A context polled every hop with clear (alternately read_stats and read_stats_device, into a guarded buffer) sums to the
    one read of a twin that is never cleared; the levels match hop by hop; clear keeps the event state."""
    A = Runner(Context, api, mem, kind, max_streams=n, n=n)
    B = Runner(Context, api, mem, kind, max_streams=n, n=n)
    rng = np.random.default_rng(seed)
    total = np.zeros((n, W), np.uint64)
    d_st = Guarded(mem, n, (W,), np.int64, 0x6B)
    role = A.role
    for f in range(hops):
        x, rec = A.inputs(f, rng, hops, n, np.arange(n, dtype=np.int32), wavs)
        A.hop(x, rec)
        B.hop(x, rec)
        if f % 2:
            got = A.c.stats(role, n=n, clear=True)
        else:
            d_st.fill()
            A.c.stats_device(role, n, d_st.ptr, clear=True)
            got = d_st.get("statistics").view(np.uint64)
        _same(got, A.model.read(np.arange(n), clear=True), "%s hop %d: a cleared poll" % (kind, f))
        assert np.array_equal(got[:, LEVEL], B.model.w[:n, LEVEL])
        for w in COUNTERS:
            total[:, w] += got[:, w]
    want = B.c.stats(role, n=n)
    _same(want, B.model.read(np.arange(n)), "%s: the twin that was never cleared" % kind)
    for w in COUNTERS:
        assert np.array_equal(total[:, w], want[:, w]), "%s: the cleared polls do not sum to one read (word %d)" % (kind, w)
    # repeated ids with clear: every listed stream is read before any is cleared
    ids = np.array([1, 0, 1, 1], np.int32)
    A.hop(*A.inputs(hops, rng, hops + 1, n, np.arange(n, dtype=np.int32), wavs))
    got = A.c.stats(role, stream_ids=ids, clear=True)
    _same(got, A.model.read(ids, clear=True), "%s: repeated ids with clear" % kind)
    A.check("%s: after a clear of repeated ids" % kind)
    A.close()
    B.close()


def _stats_offsets(c):
    """byte offsets of the encoder and decoder statistics entries in a record of a context with both roles: the per-stream words
    (DTX, encoder bits, decoder bits, rate) follow them"""
    rb = c.stream_state_bytes()
    return rb - 16 - 2 * W * 8, rb - 16 - W * 8


def run_travel(Context, api, mem, wav16, *, max_streams=16, hops=6, seed=5):
    """copy_streams, export -> import into a second context, further hops, reset, copy from -1; records with a LEVEL of 128 or
    an event state of 2 are refused with nothing changed"""
    rng = np.random.default_rng(seed)
    wavs = {16000: wav16}
    enc = Runner(Context, api, mem, "encode_dtx", max_streams=max_streams, n=max_streams)
    dec = Runner(Context, api, mem, "decode_plc", max_streams=max_streams, n=max_streams, ctx=enc.c)   # the same streams
    ids = np.arange(6, dtype=np.int32)
    for f in range(hops):
        for R in (enc, dec):
            x, rec = R.inputs(f, rng, hops, len(ids), ids, wavs)
            R.hop(x, rec, ids=ids)
    src, dst = np.array([0, 3, -1], np.int32), np.array([9, 12, 4], np.int32)
    enc.c.copy_streams(src, dst)
    for R in (enc, dec):
        R.model.copy(src, dst)
        R.check("after copy_streams", ids=np.arange(max_streams))
    other = mc._make(Context, api, max_streams, 16000, "exact", am.CNG_SEED, None, mem.stream)
    other.set_stats(1)
    recs = enc.c.export_streams(stream_ids=np.array([1, 2, 9], np.int32))
    other.import_streams(recs, stream_ids=np.array([5, 6, 7], np.int32))
    moved = {"encoder": Model(max_streams), "decoder": Model(max_streams)}
    for role, R in (("encoder", enc), ("decoder", dec)):
        m = moved[role]
        for s, d in zip((1, 2, 9), (5, 6, 7)):
            m.w[d], m.prev[d] = R.model.w[s], R.model.prev[s]
        _same(other.stats(role, n=max_streams), m.read(np.arange(max_streams)), "%s after import" % role)
    # the moved streams continue in the second context as they would have in the first
    oenc = Runner(Context, api, mem, "encode_dtx", max_streams=max_streams, n=max_streams, ctx=other)
    odec = Runner(Context, api, mem, "decode_plc", max_streams=max_streams, n=max_streams, ctx=other)
    oenc.model, odec.model = moved["encoder"], moved["decoder"]
    for f in range(hops, hops + 3):
        for R in (oenc, odec):
            x, rec = R.inputs(f, rng, hops + 3, 3, np.array([5, 6, 7], np.int32), wavs)
            R.hop(x, rec, ids=np.array([5, 6, 7], np.int32))
        for role, R in (("encoder", oenc), ("decoder", odec)):
            R.check("%s hop %d after import" % (role, f), ids=np.arange(max_streams))
    # bad records: nothing changes
    e_off, d_off = _stats_offsets(other)
    before = other.export_streams()
    for off, word, value in ((e_off, LEVEL, 128), (d_off, LEVEL, 128), (d_off, 7, 2)):
        bad = recs.copy()
        bad[1, off + 8 * word:off + 8 * word + 8] = np.frombuffer(np.uint64(value).tobytes(), np.uint8)
        rcode = api.lib.lyra_b200_import_streams(other.h, np.array([5, 6, 7], np.int32).ctypes.data, 3, bad.ctypes.data)
        assert rcode == EINVAL, "a record with word %d = %d was accepted" % (word, value)
        assert np.array_equal(other.export_streams(), before), "a refused import changed a stream"
    # reset and copy from -1 restore the initial image
    other.reset(stream_ids=[5])
    other.copy_streams([-1], [6])
    init = Model(max_streams).read(np.arange(2))
    for role in ("encoder", "decoder"):
        _same(other.stats(role, stream_ids=[5, 6]), init, "%s after reset / copy from -1" % role)
    enc.c.reset()
    for role in ("encoder", "decoder"):
        _same(enc.c.stats(role, n=max_streams), Model(max_streams).read(np.arange(max_streams)), "%s after reset" % role)
    other.close()
    enc.close()


def run_off_and_launches(Context, api, mem, wav16, *, n, hops=3, split=None, seed=7):
    """Statistics never enabled: launches equal call_schedule_cases.expected_launches, outputs equal a twin with statistics on,
    and the statistics read back as the initial image.  On adds exactly one launch per part (dense host-buffer, device and
    sparse calls).  Enabled after the first hop, the counts start there."""
    parts = 1 if split is None else split
    wavs = {16000: wav16}
    rng = np.random.default_rng(seed)
    sids = np.array([n - 1, 0], np.int32)
    for kind in KINDS:
        off = Runner(Context, api, mem, kind, max_streams=n, n=n, split=split, stats=False)
        on = Runner(Context, api, mem, kind, max_streams=n, n=n, split=split)
        late = Runner(Context, api, mem, kind, max_streams=n, n=n, split=split, stats=False)
        for f in range(hops):
            if f == 1:
                late.c.set_stats(1)
            x, rec = off.inputs(f, rng, hops, n, np.arange(n, dtype=np.int32), wavs)
            for call in ("host", "device", "sparse"):
                counts, outs = [], []
                for R in (off, on, late):
                    l0 = R.c.launch_count
                    update = R is on or (R is late and f >= 1)
                    if call == "sparse":
                        outs.append(R.hop(x[:2], rec[:2], ids=sids, update=update))
                    else:
                        outs.append(R.hop(x, rec, device=call == "device", update=update))
                    counts.append(R.c.launch_count - l0)
                for o in outs[1:]:
                    assert np.array_equal(o, outs[0]), "%s hop %d (%s): statistics changed an output" % (kind, f, call)
                want = cs.expected_launches(kind, 1 if call == "sparse" else parts, False)
                assert counts[0] == want, "%s (%s): %d launches with statistics off, expected %d" % (kind, call, counts[0], want)
                added = counts[1] - want
                assert added == (1 if call == "sparse" else parts), "%s (%s): statistics on added %d launches" % (kind, call, added)
        _same(off.c.stats(off.role, n=n), Model(n).read(np.arange(n)), "%s: statistics never enabled" % kind)
        on.check("%s: statistics on" % kind)
        late.check("%s: statistics enabled mid-run" % kind)
        for R in (off, on, late):
            R.close()


def run_unaligned(Context, api, mem, wavs, *, n, hops=3, seed=11):
    """The device twins on row buffers that start 0..7 samples past a 16-byte boundary (slices of a larger buffer: the ABI
    promises 2-byte alignment only), at a 48 kHz row rate with 8 / 16 / 48 kHz streams, so each row has an unaligned head, a
    vector body and a tail: encode_device reads such rows, decode_device writes them"""
    rng = np.random.default_rng(seed)
    for kind in ("encode", "decode"):
        R = Runner(Context, api, mem, kind, max_streams=n, n=n, ctx_rate=48000, rates=(8000, 16000, 48000))
        H, P = R.H, R.P
        big = mem.zeros((n * H + 8,), np.int16)
        d_pk = mem.zeros((n, P), np.uint8)
        for f in range(hops):
            for off in range(8):
                x, rec = R.inputs(f * 8 + off, rng, hops * 8, n, np.arange(n, dtype=np.int32), wavs)
                ptr = mem.ptr(big) + 2 * off
                if kind == "encode":
                    flat = np.zeros(n * H + 8, np.int16)
                    flat[off:off + n * H] = x.reshape(-1)
                    mem.put(big, flat)
                    R.c.encode_device(n, ptr, R.bits, mem.ptr(d_pk))
                    for k in range(n):
                        R.model.encode(k, x[k, :int(R.srate[k]) // 50], False, R.bits)
                else:
                    mem.put(d_pk, x)
                    R.c.decode_device(n, mem.ptr(d_pk), 0, R.bits, ptr)
                    out = mem.get(big)[off:off + n * H].reshape(n, H)
                    for k in range(n):
                        R.model.decode(k, out[k, :int(R.srate[k]) // 50], True)
                R.check("%s with rows %d samples past a 16-byte boundary" % (kind, off))
        R.close()


def run_argument_errors(Context, api, mem):
    """Bad role, n or ids, NULL buffers: EINVAL and no launch; a context without the role refuses it"""
    lib = api.lib
    c = Context(8, capi=api)
    out = np.zeros((8, W), np.uint64)
    d_out = mem.zeros((8, W), np.int64)
    ok_ids = np.arange(4, dtype=np.int32)
    bad_ids = np.array([0, 8], np.int32)
    neg_ids = np.array([-1], np.int32)
    l0 = c.launch_count
    assert lib.lyra_b200_set_stats(None, 1) == EINVAL
    cases = [
        lambda: lib.lyra_b200_read_stats(c.h, 0, None, 4, out.ctypes.data, 0),
        lambda: lib.lyra_b200_read_stats(c.h, 3, None, 4, out.ctypes.data, 0),
        lambda: lib.lyra_b200_read_stats(c.h, 1, None, 0, out.ctypes.data, 0),
        lambda: lib.lyra_b200_read_stats(c.h, 1, None, 9, out.ctypes.data, 0),
        lambda: lib.lyra_b200_read_stats(c.h, 2, bad_ids.ctypes.data, 2, out.ctypes.data, 1),
        lambda: lib.lyra_b200_read_stats(c.h, 2, neg_ids.ctypes.data, 1, out.ctypes.data, 1),
        lambda: lib.lyra_b200_read_stats(c.h, 1, ok_ids.ctypes.data, 4, None, 0),
        lambda: lib.lyra_b200_read_stats(None, 1, None, 4, out.ctypes.data, 0),
        lambda: lib.lyra_b200_read_stats_device(c.h, 0, 4, mem.ptr(d_out), 0),
        lambda: lib.lyra_b200_read_stats_device(c.h, 3, 4, mem.ptr(d_out), 0),
        lambda: lib.lyra_b200_read_stats_device(c.h, 1, 0, mem.ptr(d_out), 0),
        lambda: lib.lyra_b200_read_stats_device(c.h, 2, 9, mem.ptr(d_out), 1),
        lambda: lib.lyra_b200_read_stats_device(c.h, 2, 4, None, 1),
        lambda: lib.lyra_b200_read_stats_device(None, 2, 4, mem.ptr(d_out), 1),
    ]
    for i, fn in enumerate(cases):
        assert fn() == EINVAL, "case %d was accepted" % i
        assert c.launch_count == l0, "case %d launched" % i
    for roles, missing in (("encoder", 2), ("decoder", 1)):
        r = Context(8, capi=api, roles=roles)
        l1 = r.launch_count
        assert lib.lyra_b200_read_stats(r.h, missing, None, 4, out.ctypes.data, 0) == EINVAL
        assert lib.lyra_b200_read_stats_device(r.h, missing, 4, mem.ptr(d_out), 0) == EINVAL
        assert r.launch_count == l1
        _same(r.stats(3 - missing, n=8), Model(8).read(np.arange(8)), "%s-only context" % roles)
        r.close()
    c.close()
