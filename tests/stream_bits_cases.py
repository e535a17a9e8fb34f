"""Cases for per-stream bit counts (lyra_b200_set_stream_bits), shared by the CPU tier (emulated kernels) and the GPU tier.  A
stream with its own count b in a call at num_bits must behave exactly like the same stream id in a twin context called at b
bits with the same rows: its packet in the first ceil(b / 8) bytes of its row and zeros after them, the same packet_bytes,
flags, control state and PCM.  Decoders get packets whose row tails hold random bytes, which they must ignore.  A sample of
streams is also checked against the oracle at that stream's bit count."""
import numpy as np

import mixed_rate_cases as mc
import rate_cases as rc
from parity_cases import TENSOR_PCM_TOL_LSB, Guarded

EINVAL = -1
CALLS = mc.CALLS
COMMON = (64, 120, 184)          # 3.2, 6.0 and 9.2 kbps
ODD = (4, 60, 100, 180)          # odd stage counts: the last byte holds one stage and a zero low nibble


def pbytes(bits):
    return (np.asarray(bits) + 7) // 8


def _make(Context, api, max_streams, rate, mode, cng_seed, split=None, stream=None, srate=None, ids=None):
    c = mc._make(Context, api, max_streams, rate, mode, cng_seed, split, stream)
    if srate is not None:
        c.set_stream_sample_rates(srate, ids)
    return c


def _set_bits(c, sbits, ids):
    for role in ("encoder", "decoder"):
        c.set_stream_bits(role, sbits, ids)
        assert np.array_equal(c.stream_bits(role, ids), sbits)


def _check_packets(got, want, sel, b, what):
    """rows `sel` of `got` hold `want` in their first ceil(b / 8) bytes and zeros after them"""
    p = int(pbytes(b))
    assert np.array_equal(got[sel, :p], want), "%s: packets at %d bits differ from the twin" % (what, b)
    assert not got[sel, p:].any(), "%s: a packet row tail at %d bits is not 0" % (what, b)


def run_mixed_parity(Context, api, O, wavs, *, bit_set, max_streams, stream_ids=None, n=None, frames=10, oracle_rows=(),
                     decoder_mode="exact", split=None, mem=None, ctx_rate=16000, rates=None, cng_seed=7, seed=1):
    """Every fused call with streams at bit counts bit_set interleaved (both roles) in contexts called at max(bit_set), hop by hop,
    against twin contexts (same ids, same rows) called at each stream's count.  rates: per-stream sample rates interleaved too,
    in the mixed and the twin contexts alike.  mem None: the host-buffer calls (stream_ids None = dense streams 0..n-1);
    otherwise the *_device twins over streams 0..n-1 with guarded caller buffers.  Inputs: speech, every third stream silent in
    the second half (DTX), random losses for decode / decode_track_noise, bursts of 7 (into comfort noise and back) or 2 for
    decode_plc.  oracle_rows: rows also checked against the oracle at their count and rate."""
    ids = np.arange(n, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    device = mem is not None
    assert not (device and stream_ids is not None), "the device calls serve streams 0..n-1"
    call_ids = None if stream_ids is None else ids
    sbits = mc.interleaved(n, bit_set)
    srate = mc.interleaved(n, rates) if rates else np.full(n, ctx_rate, np.int32)
    bits = int(max(bit_set))
    P = int(pbytes(bits))
    H = rc.hop_of(ctx_rate)
    stream = mem.stream if device else None
    sr = srate if rates else None
    mixed = {k: _make(Context, api, max_streams, ctx_rate, decoder_mode, cng_seed, split, stream, sr, ids) for k in CALLS}
    for c in mixed.values():
        _set_bits(c, sbits, ids)
    present = sorted(set(int(b) for b in sbits))
    sel = {b: np.nonzero(sbits == b)[0] for b in present}
    twins = {b: {k: _make(Context, api, max_streams, ctx_rate, decoder_mode, cng_seed, None, None, sr, ids) for k in CALLS}
             for b in present}
    tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    orc = {k: dict(codec=rc.OracleCodec(O, int(srate[k])), dtx=rc.OracleEncoder(O, int(srate[k]), dtx=True)) for k in oracle_rows}
    if device:
        G = lambda row, dtype, s: Guarded(mem, n, row, dtype, s)     # noqa: E731
        d_pcm, d_pk_in, d_rec, d_plc_rec = G((H,), np.int16, 0x3C), G((P,), np.uint8, 0x3C), G((), np.uint8, 0xC3), G((), np.uint8, 0xC3)
        d_out, d_trk, d_plc = G((H,), np.int16, 0x5A), G((H,), np.int16, 0x5A), G((H,), np.int16, 0x5A)
        d_trk_flags, d_cn, d_dtx_flags = (G((), np.uint8, 0xAA) for _ in range(3))
    rng = np.random.default_rng(seed)
    burst = [(1 + k % 3, 7 if k % 2 == 0 else 2) for k in range(n)]
    seen = dict(cn=False, dtx=set(), loss=False)
    tail = (np.arange(P)[None, :] >= pbytes(sbits)[:, None])
    for f in range(frames):
        silent = (np.arange(n) % 3 == 0) & (f >= frames // 2)
        pcm, _ = mc.mixed_rows(wavs, srate, ids, f, H, rng, silent)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        rec_trk = (rng.random(n) >= 0.25).astype(np.uint8)
        rec_plc = np.array([0 if b0 <= f < b0 + bl else 1 for b0, bl in burst], dtype=np.uint8)
        noise = rng.integers(0, 256, size=(n, P), dtype=np.uint8)
        if device:
            d_pcm.put(pcm)
            d_rec.put(rec)
            d_plc_rec.put(rec_plc)
            d_pk, d_dtx_pk = G((P,), np.uint8, 0xA5), G((P,), np.uint8, 0xFF)
            for buf in (d_out, d_trk, d_plc, d_trk_flags, d_cn, d_dtx_flags):
                buf.fill()
            mixed["codec"].encode_device(n, d_pcm.ptr, bits, d_pk.ptr)
            pk = d_pk.get("packets")
            d_pk_in.put(np.where(tail, noise, pk))
            mixed["codec"].decode_device(n, d_pk_in.ptr, d_rec.ptr, bits, d_out.ptr)
            d_rec.put(rec_trk)
            mixed["track"].decode_track_noise_device(n, d_pk_in.ptr, d_rec.ptr, bits, d_trk.ptr, d_trk_flags.ptr)
            mixed["plc"].decode_plc_device(n, d_pk_in.ptr, d_plc_rec.ptr, bits, d_plc.ptr, d_cn.ptr)
            mixed["dtx"].encode_dtx_device(n, d_pcm.ptr, bits, d_dtx_pk.ptr, d_dtx_flags.ptr)
            out = d_out.get("PCM")
            t_out, t_flags = d_trk.get("PCM"), d_trk_flags.get("flags").astype(bool)
            p_out, p_cn = d_plc.get("PCM"), d_cn.get("flags").astype(bool)
            x_pk, x_sizes = d_dtx_pk.get("packets"), np.where(d_dtx_flags.get("flags") != 0, 0, pbytes(sbits))
            d_pcm.get("input PCM")
            d_pk_in.get("input packets")
        else:
            pk = mixed["codec"].encode(pcm, bits, stream_ids=call_ids)
            pk_in = np.where(tail, noise, pk)
            out = mixed["codec"].decode(pk_in, bits, stream_ids=call_ids, received=rec)
            t_out, t_flags = mixed["track"].decode_track_noise(pk_in, bits, stream_ids=call_ids, received=rec_trk)
            p_out, p_cn = mixed["plc"].decode_plc(pk_in, bits, stream_ids=call_ids, received=rec_plc)
            x_pk, x_sizes = mixed["dtx"].encode_dtx(pcm, bits, stream_ids=call_ids)
        p_state = mixed["plc"].plc_state(stream_ids=ids)
        for b in present:
            s, tw = sel[b], twins[b]
            what = "hop %d, streams at %d bits in a call at %d" % (f, b, bits)
            tpk = tw["codec"].encode(pcm[s], b, stream_ids=ids[s])
            _check_packets(pk, tpk, s, b, "encode, " + what)
            assert np.array_equal(out[s], tw["codec"].decode(tpk, b, stream_ids=ids[s], received=rec[s])), "decode, " + what
            w_out, w_flags = tw["track"].decode_track_noise(tpk, b, stream_ids=ids[s], received=rec_trk[s])
            assert np.array_equal(t_out[s], w_out) and np.array_equal(t_flags[s], w_flags), "decode_track_noise, " + what
            w_out, w_cn = tw["plc"].decode_plc(tpk, b, stream_ids=ids[s], received=rec_plc[s])
            assert np.array_equal(p_out[s], w_out) and np.array_equal(p_cn[s], w_cn), "decode_plc, " + what
            assert np.array_equal(p_state[s], tw["plc"].plc_state(stream_ids=ids[s])), "control state, " + what
            w_pk, w_sizes = tw["dtx"].encode_dtx(pcm[s], b, stream_ids=ids[s])
            assert np.array_equal(x_sizes[s], w_sizes), "encode_dtx packet_bytes, " + what
            _check_packets(x_pk, w_pk, s, b, "encode_dtx, " + what)
        for k, o in orc.items():
            b, h = int(sbits[k]), rc.hop_of(int(srate[k]))
            x = pcm[k, :h]
            opkt = o["codec"].encode(x, b)
            assert bytes(pk[k][:len(opkt)]) == opkt, "encode != oracle at %d bits, hop %d stream %d" % (b, f, ids[k])
            d = rc._pcm_diff(out[k, :h], o["codec"].decode(opkt if rec[k] else None, b))
            assert d <= tol, "decode != oracle at %d bits, hop %d stream %d: %d" % (b, f, ids[k], d)
            want = o["dtx"].encode(x, b)
            assert x_sizes[k] == len(want) and bytes(x_pk[k][:x_sizes[k]]) == want, "encode_dtx != oracle, hop %d stream %d" % (f, ids[k])
        seen["loss"] |= not rec.all()
        seen["cn"] |= bool(p_cn.any())
        seen["dtx"] |= set(int(v == 0) for v in x_sizes)
    assert seen["loss"] and seen["cn"], "the case must lose packets and reach comfort noise"
    assert seen["dtx"] == {0, 1}, "the case must produce both DTX and encoded hops"
    for c in list(mixed.values()) + [c for tw in twins.values() for c in tw.values()]:
        c.close()


def run_bits_change(Context, api, wav16, *, max_streams=16, stream_ids=(1, 4, 9), hops=12, seed=3, cng_seed=5):
    """set_bitrate between hops: the encoder counts of the streams change every 3 hops and equal a twin that switches the call's
    num_bits at that hop (one twin per stream); the decoder counts change in the middle of a loss burst, against a twin decoder
    that switches num_bits there.  The calls run at 184 bits."""
    ids = np.asarray(stream_ids, np.int32)
    n = len(ids)
    enc_sched = [(64, 120, 184), (120, 184, 64), (4, 60, 184), (184, 64, 100)]
    a = Context(max_streams, capi=api)
    a.set_cng_seed(cng_seed)
    tw = [Context(max_streams, capi=api) for _ in range(n)]
    for t in tw:
        t.set_cng_seed(cng_seed)
    rng = np.random.default_rng(seed)
    for f in range(hops):
        eb = np.asarray(enc_sched[(f // 3) % len(enc_sched)], np.int32)
        db = np.asarray((64, 64, 120) if f < hops // 2 else (184, 120, 64), np.int32)
        a.set_stream_bits("encoder", eb, ids)
        a.set_stream_bits("decoder", db, ids)
        pcm = rc.speech_rows(wav16, 16000, ids, f)
        lost = np.array([hops // 2 - 2 <= f < hops // 2 + 2 and k != 1 for k in range(n)], bool)
        pk = a.encode(pcm, 184, stream_ids=ids)
        out, cn = a.decode_plc(pk, 184, stream_ids=ids, received=(~lost).astype(np.uint8))
        for k in range(n):
            p = int(pbytes(eb[k]))
            want = tw[k].encode(pcm[k:k + 1], int(eb[k]), stream_ids=ids[k:k + 1])
            assert np.array_equal(pk[k:k + 1, :p], want) and not pk[k, p:].any(), "encoder count change, hop %d stream %d" % (f, ids[k])
            w_out, w_cn = tw[k].decode_plc(pk[k:k + 1, :int(pbytes(db[k]))], int(db[k]), stream_ids=ids[k:k + 1],
                                           received=(~lost[k:k + 1]).astype(np.uint8))
            assert np.array_equal(out[k], w_out[0]) and cn[k] == w_cn[0], "decoder count change, hop %d stream %d" % (f, ids[k])
    for c in [a] + tw:
        c.close()


def run_validation(Context, api, wav16, LyraB200Error, *, max_streams=16, ids=(2, 5, 11), bits=(120, 64, 184)):
    """Every refused setter call and every refused codec call returns EINVAL and changes nothing: the words, the exported state
    and the following calls equal a twin that never saw the refused calls."""
    ids, sb = np.asarray(ids, np.int32), np.asarray(bits, np.int32)
    ctx, twin = Context(max_streams, capi=api), Context(max_streams, capi=api)
    for c in (ctx, twin):
        _set_bits(c, sb, ids)
    enc_only = Context(max_streams, capi=api, roles="encoder")
    fails = lambda fn: mc._fails_einval(fn, LyraB200Error)     # noqa: E731
    before, words = ctx.export_streams(), {r: ctx.stream_bits(r) for r in ("encoder", "decoder")}
    for what, call in {
        "count 3": lambda: ctx.set_stream_bits("encoder", [3], [1]),
        "count 188": lambda: ctx.set_stream_bits("decoder", [64, 188], [1, 3]),
        "count -4": lambda: ctx.set_stream_bits("encoder", [-4], [1]),
        "role 0": lambda: ctx.set_stream_bits(0, [64], [1]),
        "role both": lambda: ctx.set_stream_bits("both", [64], [1]),
        "a role the context lacks": lambda: enc_only.set_stream_bits("decoder", [64], [1]),
        "an id out of range": lambda: ctx.set_stream_bits("encoder", [64], [max_streams]),
        "repeated ids": lambda: ctx.set_stream_bits("encoder", [64, 120], [6, 6]),
        "a getter for a role the context lacks": lambda: enc_only.stream_bits("decoder"),
    }.items():
        assert fails(call), "accepted %s" % what
    assert np.array_equal(ctx.export_streams(), before), "a refused setter call changed a stream"
    for r, w in words.items():
        assert np.array_equal(ctx.stream_bits(r), w)
    # a call below a listed stream's own count is refused and queues nothing
    rng = np.random.default_rng(4)
    pcm = rng.integers(-8000, 8000, size=(len(ids), 320), dtype=np.int16)
    l0 = ctx.launch_count
    assert fails(lambda: ctx.encode(pcm, 120, stream_ids=ids)), "encode at 120 bits with a stream at 184"
    assert fails(lambda: ctx.encode_dtx(pcm, 64, stream_ids=ids))
    assert fails(lambda: ctx.decode(np.zeros((len(ids), 15), np.uint8), 120, stream_ids=ids))
    assert fails(lambda: ctx.decode_plc(np.zeros((len(ids), 8), np.uint8), 64, stream_ids=ids))
    assert fails(lambda: ctx.decode_track_noise(np.zeros((len(ids), 8), np.uint8), 64, stream_ids=ids))
    assert fails(lambda: ctx.encode(np.zeros((max_streams, 320), np.int16), 120)), "a dense call lists stream 11 at 184"
    assert ctx.launch_count == l0, "a refused call launched kernels"
    for f in range(2):
        x = rc.speech_rows(wav16, 16000, ids, f)
        got = [ctx.encode(x, 184, stream_ids=ids)]
        got.append(ctx.decode_plc(got[0], 184, stream_ids=ids)[0])
        want = [twin.encode(x, 184, stream_ids=ids)]
        want.append(twin.decode_plc(want[0], 184, stream_ids=ids)[0])
        for u, v in zip(got, want):
            assert np.array_equal(u, v), "a refused call changed the following calls, hop %d" % f
    # a stream the call does not list does not constrain it
    ctx.encode(rc.speech_rows(wav16, 16000, [5, 7], 0), 64, stream_ids=[5, 7])
    # the words in a record: encoder, decoder, then the sample rate last; a damaged bits word is refused
    rec = ctx.export_streams(ids)
    w = rec.view(np.uint32)
    assert w[0, 1] == 3, "record format version"
    assert np.array_equal(w[:, -3], sb) and np.array_equal(w[:, -2], sb), "bits words not where expected"
    for bad in (3, 188, 0xFFFFFFFC):
        for col in (-3, -2):
            r = rec.copy()
            r.view(np.uint32)[0, col] = bad
            assert fails(lambda: ctx.import_streams(r, ids)), "accepted a record with bits word %d" % bad
    assert enc_only.export_streams([1]).view(np.uint32)[0, -2] == 0, "an encoder-only record holds the encoder word before the rate"
    for c in (ctx, twin, enc_only):
        c.close()


def run_moves(Context, api, wav16, *, max_streams=16, ids=(2, 5), enc_bits=(120, 60), dec_bits=(184, 64), copy_to=(10, 13),
              import_to=(7, 0), hops=10, after=3, cng_seed=5):
    """Streams with their own counts in both roles, after a history that reaches comfort noise and DTX: moved with copy_streams
    and with export / import into a second context, they carry both words and continue bit for bit like an unmoved twin; the
    calls then refuse a num_bits below the moved words.  reset and copy_streams from -1 clear both words."""
    ids, copy_to, import_to = (np.asarray(x, np.int32) for x in (ids, copy_to, import_to))
    eb, db = np.asarray(enc_bits, np.int32), np.asarray(dec_bits, np.int32)
    A, T, B = (Context(max_streams, capi=api) for _ in range(3))
    for c in (A, T, B):
        c.set_cng_seed(cng_seed)
    for c in (A, T):
        c.set_stream_bits("encoder", eb, ids)
        c.set_stream_bits("decoder", db, ids)

    def hop(c, f, where):
        x = rc.speech_rows(wav16, 16000, ids, f)
        if f >= 6:
            x[0] = 0
        lost = np.array([2 <= f <= 8, False])
        pk, sizes = c.encode_dtx(x, 184, stream_ids=where)
        out, cn = c.decode_plc(np.where(np.arange(23)[None, :] < pbytes(db)[:, None], pk, 0xEE), 184, stream_ids=where,
                               received=(~lost).astype(np.uint8))
        return {"pk": pk, "sizes": sizes, "pcm": out, "cn": cn, "state": c.plc_state(stream_ids=where)}
    seen_cn = seen_dtx = False
    for f in range(hops):
        o = hop(A, f, ids)
        hop(T, f, ids)
        seen_cn |= bool(o["cn"].any())
        seen_dtx |= bool((o["sizes"] == 0).any())
    assert seen_cn and seen_dtx, "the history must reach comfort noise and DTX"
    A.copy_streams(ids, copy_to)
    B.import_streams(T.export_streams(ids), import_to)
    for c, where in ((A, copy_to), (B, import_to)):
        assert np.array_equal(c.stream_bits("encoder", where), eb) and np.array_equal(c.stream_bits("decoder", where), db)
    for f in range(hops, hops + after):
        ot = hop(T, f, ids)
        for c, where in ((A, copy_to), (B, import_to)):
            o = hop(c, f, where)
            for name, v in o.items():
                assert np.array_equal(v, ot[name]), "%s of a moved stream differs, hop %d (%s)" % (name, f, "copy" if c is A else "import")
    A.reset(copy_to[:1])
    A.copy_streams([-1], copy_to[1:])
    for r in ("encoder", "decoder"):
        assert not A.stream_bits(r, copy_to).any(), "reset / copy from -1 must clear the words"
    assert np.array_equal(A.stream_bits("encoder", ids), eb), "the sources keep their words"
    A.encode(np.zeros((2, 320), np.int16), 4, stream_ids=copy_to)     # cleared in the host mirror too: any num_bits is accepted
    for c in (A, T, B):
        c.close()


def run_refused_after_move(Context, api, LyraB200Error, *, max_streams=16):
    """The host mirror follows copy, import and reset: a call below a moved stream's word is refused, after reset it is not."""
    A, B = Context(max_streams, capi=api), Context(max_streams, capi=api)
    A.set_stream_bits("encoder", [120], [3])
    A.copy_streams([3], [8])
    B.import_streams(A.export_streams([3]), [12])
    x = np.zeros((1, 320), np.int16)
    for c, s in ((A, 8), (B, 12)):
        assert mc._fails_einval(lambda: c.encode(x, 64, stream_ids=[s]), LyraB200Error), "the moved word was not checked"
        c.reset([s])
        c.encode(x, 64, stream_ids=[s])
    for c in (A, B):
        c.close()


def run_unchanged_when_unused(Context, api, wav16, *, max_streams=16, stream_ids=(0, 3, 9), hops=2, seed=3):
    """A context that never set a word issues the same launches per call as one that set words and cleared them all again, and
    the same as before it first set one; the outputs are equal too."""
    ids = np.asarray(stream_ids, np.int32)
    n = len(ids)
    c, d = Context(max_streams, capi=api), Context(max_streams, capi=api)
    rng = np.random.default_rng(seed)

    def calls(ctx, f):
        x = rc.speech_rows(wav16, 16000, ids, f)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        res, counts = [], []
        for fn in (lambda: [ctx.encode(x, 64, stream_ids=ids)], lambda: [ctx.decode(np.zeros((n, 8), np.uint8), 64, stream_ids=ids, received=rec)],
                   lambda: [ctx.encode(np.zeros((max_streams, 320), np.int16), 64)], lambda: [ctx.decode(np.zeros((max_streams, 8), np.uint8), 64)],
                   lambda: ctx.decode_track_noise(np.zeros((n, 8), np.uint8), 64, stream_ids=ids, received=rec),
                   lambda: ctx.decode_plc(np.zeros((n, 8), np.uint8), 64, stream_ids=ids), lambda: ctx.encode_dtx(x, 64, stream_ids=ids)):
            l0 = ctx.launch_count
            res += list(fn())
            counts.append(ctx.launch_count - l0)
        return res, counts
    f = 0
    for phase in range(2):
        if phase:
            c.set_stream_bits("encoder", [120, 184], [3, 9])
            c.set_stream_bits("decoder", [64], [0])
            c.encode(rc.speech_rows(wav16, 16000, ids, 0), 184, stream_ids=ids)
            d.encode(rc.speech_rows(wav16, 16000, ids, 0), 184, stream_ids=ids)
            c.set_stream_bits("encoder", [0, 0], [3, 9])
            c.set_stream_bits("decoder", np.zeros(max_streams, np.int32))
        for _ in range(hops):
            rs = rng.bit_generator.state
            rc_, cc = calls(c, f)
            rng.bit_generator.state = rs
            rd, cd = calls(d, f)
            assert cc == cd, "launches per call differ (%s): %s vs %s" % ("after clearing" if phase else "before setting", cc, cd)
            for u, v in zip(rc_, rd):
                assert np.array_equal(u, v)
            f += 1
    c.close()
    d.close()
