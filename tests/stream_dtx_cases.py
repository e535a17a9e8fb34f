"""Cases for per-stream DTX (lyra_b200_set_stream_dtx), shared by the CPU tier (emulated kernels) and the GPU tier.  A stream with
DTX off must behave in encode_dtx exactly like LyraEncoder created with enable_dtx = false: every hop encoded, flag 0,
packet_bytes ceil(b / 8).  A stream with DTX on behaves as before.  Checked against the oracle (rate_cases.OracleEncoder with the
stream's setting) and against a pair of twin contexts: encode_dtx for the streams with DTX on, encode for the others."""
import numpy as np

import mixed_rate_cases as mc
import rate_cases as rc
from parity_cases import Guarded

EINVAL = -1


def pbytes(bits):
    return (np.asarray(bits) + 7) // 8


def _make(Context, api, max_streams, ctx_rate, ids, srate, sbits, split=None, stream=None):
    """a context at row rate ctx_rate with the streams' own rates and encoder bit counts (None: the context's / the call's)"""
    c = Context(max_streams, capi=api)
    c.set_sample_rate(ctx_rate)
    if split is not None:
        c.set_split(split)
    if stream is not None:
        c.set_stream(stream)
    if srate is not None:
        c.set_stream_sample_rates(srate, ids)
    if sbits is not None:
        c.set_stream_bits("encoder", sbits, ids)
    return c


def quiet_rows(wavs, srate, ids, f, H, rng, frames):
    """hop f of speech rows (mixed_rate_cases.mixed_rows), with stretches the DTX estimators classify as noise: every third
    stream silent in the second half, every fifth at a low noise level from hop frames // 3 on"""
    n = len(ids)
    silent = (np.arange(n) % 3 == 0) & (f >= frames // 2)
    pcm, _ = mc.mixed_rows(wavs, srate, ids, f, H, rng, silent)
    low = (np.arange(n) % 5 == 1) & (f >= frames // 3)
    for k in np.nonzero(low)[0]:
        h = rc.hop_of(int(srate[k]))
        pcm[k, :h] = rng.integers(-12, 13, size=h)
    return pcm


def run_mixed_parity(Context, api, O, wavs, *, max_streams, stream_ids=None, n=None, frames=12, oracle_rows=None, bits=64,
                     ctx_rate=16000, rates=None, bit_set=None, split=None, mem=None, seed=1):
    """encode_dtx with DTX on for even rows and off for odd rows of one context, hop by hop: against the oracle (oracle_rows, None:
    every row) and against two twin contexts with the same rates and bit counts, one running encode_dtx over the DTX-on rows and
    one running encode over the DTX-off rows.  Packets and packet_bytes are bit-exact, so the later hops' equality also shows that
    the state of every stream carried on right.  mem None: host-buffer calls (stream_ids None = dense streams 0..n-1); otherwise
    encode_dtx_device over streams 0..n-1 with guarded caller buffers, its flags against the twins' packet_bytes."""
    ids = np.arange(n, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    device = mem is not None
    assert not (device and stream_ids is not None), "the device calls serve streams 0..n-1"
    call_ids = None if stream_ids is None else ids
    enable = (np.arange(n) % 2 == 0).astype(np.int32)
    on, off = np.nonzero(enable)[0], np.nonzero(enable == 0)[0]
    srate = mc.interleaved(n, rates) if rates else None
    sbits = mc.interleaved(n, bit_set) if bit_set else None
    row_rate = srate if srate is not None else np.full(n, ctx_rate, np.int32)
    row_bits = sbits if sbits is not None else np.full(n, bits, np.int32)
    P, H = int(pbytes(bits)), rc.hop_of(ctx_rate)
    ctx = _make(Context, api, max_streams, ctx_rate, ids, srate, sbits, split, mem.stream if device else None)
    ctx.set_stream_dtx(enable, ids)
    assert np.array_equal(ctx.stream_dtx(ids), enable)
    tw_on, tw_off = (_make(Context, api, max_streams, ctx_rate, ids, srate, sbits) for _ in range(2))
    rows = range(n) if oracle_rows is None else oracle_rows
    orc = {k: rc.OracleEncoder(O, int(row_rate[k]), dtx=bool(enable[k])) for k in rows}
    if device:
        d_pcm = Guarded(mem, n, (H,), np.int16, 0x3C)
        d_flags = Guarded(mem, n, (), np.uint8, 0xAA)
    rng = np.random.default_rng(seed)
    seen = set()
    for f in range(frames):
        pcm = quiet_rows(wavs, row_rate, ids, f, H, rng, frames)
        if device:
            d_pcm.put(pcm)
            d_pk = Guarded(mem, n, (P,), np.uint8, 0xFF)
            d_flags.fill()
            ctx.encode_dtx_device(n, d_pcm.ptr, bits, d_pk.ptr, d_flags.ptr)
            pk, flags = d_pk.get("packets"), d_flags.get("flags")
            assert set(np.unique(flags)) <= {0, 1}, "hop %d: a flag is not 0 or 1" % f
            sizes = np.where(flags != 0, 0, pbytes(row_bits))
            d_pcm.get("input PCM")
        else:
            pk, sizes = ctx.encode_dtx(pcm, bits, stream_ids=call_ids)
        w_pk, w_sizes = tw_on.encode_dtx(pcm[on], bits, stream_ids=ids[on])
        assert np.array_equal(pk[on], w_pk) and np.array_equal(sizes[on], w_sizes), "hop %d: DTX-on streams differ from encode_dtx" % f
        w_pk = tw_off.encode(pcm[off], bits, stream_ids=ids[off])
        assert np.array_equal(pk[off], w_pk), "hop %d: DTX-off streams differ from encode" % f
        assert np.array_equal(sizes[off], pbytes(row_bits[off])), "hop %d: a DTX-off stream's packet_bytes" % f
        for k, o in orc.items():
            want = o.encode(pcm[k, :rc.hop_of(int(row_rate[k]))], int(row_bits[k]))
            assert sizes[k] == len(want) and bytes(pk[k][:sizes[k]]) == want and not pk[k][sizes[k]:].any(), \
                "encode_dtx != oracle (DTX %s), hop %d stream %d: %d bytes, oracle %d" % ("on" if enable[k] else "off", f, ids[k],
                                                                                          sizes[k], len(want))
        seen |= set(int(s == 0) for s in sizes[on])
    assert seen == {0, 1}, "the DTX-on streams must produce both empty and encoded hops"
    for c in (ctx, tw_on, tw_off):
        c.close()


class ToggledOracle:
    """rate_cases.OracleEncoder whose DTX is switched between hops: on builds a fresh NoiseEstimator, the encoder carries on"""

    def __init__(self, O, rate, dtx):
        self.O, self.rate = O, rate
        self.o = rc.OracleEncoder(O, rate, dtx=dtx)

    def set_dtx(self, on):
        self.o.est = self.O.NoiseEstimator(self.rate, 320, 640, 160) if on else None

    def encode(self, pcm, bits):
        return self.o.encode(pcm, bits)


def run_toggle(Context, api, O, wav16, *, max_streams=16, stream_ids=(1, 4, 9), hops=24, speech=4, bits=64):
    """set_stream_dtx between hops against the oracle, over speech followed by silence: stream 0 goes on -> off -> on,
    stream 1 starts off and goes on, stream 2 stays on and is set on again; each turn on restarts the estimator (a fresh
    NoiseEstimator), the encoder carries on.  Setting the value a stream has launches nothing and changes nothing."""
    ids = np.asarray(stream_ids, np.int32)
    n = len(ids)
    sched = {0: (1, 0, 1), 10: (1, 1, 1), 14: (0, 1, 1), 16: (0, 1, 1), 18: (1, 1, 1)}
    ctx = Context(max_streams, capi=api)
    orc = [ToggledOracle(O, 16000, True) for _ in range(n)]
    seen = [set() for _ in range(n)]
    state = np.ones(n, np.int32)
    for f in range(hops):
        if f in sched:
            new = np.asarray(sched[f], np.int32)
            rec0 = ctx.export_streams(ids)
            l0 = ctx.launch_count
            ctx.set_stream_dtx(new, ids)
            if np.array_equal(new, state):
                assert ctx.launch_count == l0, "hop %d: setting the values the streams have launched kernels" % f
                assert np.array_equal(ctx.export_streams(ids), rec0), "hop %d: setting the values the streams have changed them" % f
            for k in range(n):
                if new[k] != state[k]:
                    orc[k].set_dtx(bool(new[k]))
            state = new
            assert np.array_equal(ctx.stream_dtx(ids), state)
        x = rc.speech_rows(wav16, 16000, ids, f)
        if f >= speech:
            x[:] = 0
        pk, sizes = ctx.encode_dtx(x, bits, stream_ids=ids)
        for k in range(n):
            want = orc[k].encode(x[k], bits)
            assert sizes[k] == len(want) and bytes(pk[k][:sizes[k]]) == want, "hop %d stream %d (DTX %d): %d bytes, oracle %d" % (
                f, ids[k], state[k], sizes[k], len(want))
            seen[k].add((int(state[k]), int(sizes[k] == 0)))
    assert (1, 1) in seen[0] and (1, 1) in seen[2] and (0, 0) in seen[0] and (0, 0) in seen[1], \
        "the toggles must meet empty and encoded hops: %s" % seen
    ctx.close()


def run_moves(Context, api, wav16, LyraB200Error, *, max_streams=16, ids=(2, 5, 6), enable=(0, 1, 0), copy_to=(10, 13, 14),
              import_to=(7, 0, 1), hops=8, after=3, bits=64):
    """Copy, export and import carry the DTX word and the streams continue bit for bit like an unmoved twin; reset and copy from
    -1 turn DTX back on (in the host mirror too: setting 1 again then launches nothing).  A record whose DTX word is not 0 or 1
    fails the whole import and changes nothing.  In an encoder-only record the word sits just before the encoder bits word."""
    ids, copy_to, import_to, en = (np.asarray(x, np.int32) for x in (ids, copy_to, import_to, enable))
    A, T, B = (Context(max_streams, capi=api) for _ in range(3))
    for c in (A, T):
        c.set_stream_dtx(en, ids)

    def hop(c, f, where):
        x = rc.speech_rows(wav16, 16000, ids, f)
        if f >= hops // 2:
            x[:] = 0
        return c.encode_dtx(x, bits, stream_ids=where)
    seen = set()
    for f in range(hops):
        pk, sizes = hop(A, f, ids)
        hop(T, f, ids)
        seen |= set(int(s == 0) for s in sizes[en == 1])
        assert (sizes[en == 0] > 0).all()
    assert seen == {0, 1}, "the history must produce both empty and encoded hops"
    A.copy_streams(ids, copy_to)
    B.import_streams(T.export_streams(ids), import_to)
    for c, where in ((A, copy_to), (B, import_to)):
        assert np.array_equal(c.stream_dtx(where), en), "the move did not carry the DTX word"
    for f in range(hops, hops + after):
        want = hop(T, f, ids)
        for c, where in ((A, copy_to), (B, import_to)):
            got = hop(c, f, where)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), "moved stream differs, hop %d" % f
    A.reset(copy_to[:1])
    A.copy_streams([-1, -1], copy_to[1:])
    assert np.array_equal(A.stream_dtx(copy_to), [1, 1, 1]), "reset / copy from -1 must turn DTX on"
    l0 = A.launch_count
    A.set_stream_dtx([1, 1, 1], copy_to)
    assert A.launch_count == l0, "the host mirror missed the reset / copy from -1"
    assert np.array_equal(A.stream_dtx(ids), en), "the sources keep their words"
    # a damaged DTX word fails the whole import; the word is the fourth word from the end (DTX, encoder bits, decoder bits, rate)
    rec = T.export_streams(ids)
    assert np.array_equal(rec.view(np.uint32)[:, -4], 1 - en), "DTX word not where expected"
    before, words = B.export_streams(), B.stream_dtx()
    for bad in (2, 0xFFFFFFFF):
        r = rec.copy()
        r.view(np.uint32)[1, -4] = bad
        assert mc._fails_einval(lambda: B.import_streams(r, [3, 4, 8]), LyraB200Error), "accepted DTX word %d" % bad
    assert np.array_equal(B.export_streams(), before) and np.array_equal(B.stream_dtx(), words), "a refused import changed a stream"
    E = Context(max_streams, capi=api, roles="encoder")
    E.set_stream_dtx([0], [3])
    w = E.export_streams([2, 3]).view(np.uint32)
    assert list(w[:, -3]) == [0, 1] and not w[:, -2].any() and not w[:, -1].any(), "encoder-only record: DTX, encoder bits, rate"
    for c in (A, T, B, E):
        c.close()


def run_validation(Context, api, LyraB200Error, *, max_streams=16):
    """Every refused call returns EINVAL and queues or changes nothing: words, exported state and launch count stay."""
    ctx = Context(max_streams, capi=api)
    ctx.set_stream_dtx([0, 0], [3, 8])
    dec = Context(max_streams, capi=api, roles="decoder")
    fails = lambda fn: mc._fails_einval(fn, LyraB200Error)     # noqa: E731
    lib = api.lib
    before, words, l0 = ctx.export_streams(), ctx.stream_dtx(), ctx.launch_count
    one = np.ones(1, np.int32)
    for what, call in {
        "enable NULL": lambda: ctx._check(lib.lyra_b200_set_stream_dtx(ctx.h, None, 1, None)),
        "value 2": lambda: ctx.set_stream_dtx([1, 2], [3, 4]),
        "value -1": lambda: ctx.set_stream_dtx([-1], [3]),
        "an id out of range": lambda: ctx.set_stream_dtx([1], [max_streams]),
        "a negative id": lambda: ctx.set_stream_dtx([1], [-1]),
        "repeated ids": lambda: ctx.set_stream_dtx([1, 1], [3, 3]),
        "a decoder-only context": lambda: dec.set_stream_dtx([0], [1]),
        "the getter in a decoder-only context": lambda: dec.stream_dtx(),
        "the getter with enable NULL": lambda: ctx._check(lib.lyra_b200_stream_dtx(ctx.h, None, 1, None)),
        "n = 0": lambda: ctx._check(lib.lyra_b200_set_stream_dtx(ctx.h, None, 0, one.ctypes.data)),
    }.items():
        assert fails(call), "accepted %s" % what
    assert ctx.launch_count == l0, "a refused call launched kernels"
    assert np.array_equal(ctx.export_streams(), before) and np.array_equal(ctx.stream_dtx(), words), "a refused call changed a stream"
    for c in (ctx, dec):
        c.close()


def run_unchanged_when_unused(Context, api, wav16, *, max_streams=16, stream_ids=(0, 3, 9), hops=2, seed=3):
    """A context that never called the setter and one that turned DTX off and on again before its first hop issue the same
    launches per call with the same outputs, for all five fused calls; a context with DTX-off streams issues the same launches
    in encode_dtx."""
    ids = np.asarray(stream_ids, np.int32)
    n = len(ids)
    c, d, e = (Context(max_streams, capi=api) for _ in range(3))
    d.set_stream_dtx([0, 0], [3, 9])
    d.set_stream_dtx(np.ones(max_streams, np.int32))
    e.set_stream_dtx([0, 0], ids[1:])
    rng = np.random.default_rng(seed)

    def calls(ctx, f, r):
        x = rc.speech_rows(wav16, 16000, ids, f)
        rec = (r.random(n) >= 0.3).astype(np.uint8)
        res, counts = [], []
        for fn in (lambda: [ctx.encode(x, 64, stream_ids=ids)], lambda: [ctx.decode(np.zeros((n, 8), np.uint8), 64, stream_ids=ids, received=rec)],
                   lambda: [ctx.encode(np.zeros((max_streams, 320), np.int16), 64)], lambda: [ctx.decode(np.zeros((max_streams, 8), np.uint8), 64)],
                   lambda: ctx.decode_track_noise(np.zeros((n, 8), np.uint8), 64, stream_ids=ids, received=rec),
                   lambda: ctx.decode_plc(np.zeros((n, 8), np.uint8), 64, stream_ids=ids), lambda: ctx.encode_dtx(x, 64, stream_ids=ids),
                   lambda: ctx.encode_dtx(np.zeros((max_streams, 320), np.int16), 64)):
            l0 = ctx.launch_count
            res += list(fn())
            counts.append(ctx.launch_count - l0)
        return res, counts
    for f in range(hops):
        rs = rng.bit_generator.state
        out = {}
        for name, ctx in (("c", c), ("d", d), ("e", e)):
            rng.bit_generator.state = rs
            out[name] = calls(ctx, f, rng)
        assert out["c"][1] == out["d"][1] == out["e"][1], "launches per call differ: %s" % {k: v[1] for k, v in out.items()}
        for u, v in zip(out["c"][0], out["d"][0]):
            assert np.array_equal(u, v), "hop %d: turning DTX off and on again before the first hop changed an output" % f
    for x in (c, d, e):
        x.close()
