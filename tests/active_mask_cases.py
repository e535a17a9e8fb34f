"""Cases for the active mask of the *_device codec calls (lyra_b200_set_active_mask), shared by the CPU tier (emulated kernels)
and the GPU tier.  A stream whose mask byte is 0 must be exactly a LyraEncoder / LyraDecoder that is not called this hop: its
state does not change, its inputs are not read and its output rows are zeros (plus the flags the header specifies).  Checked
against a twin context driven by the sparse host-buffer calls over exactly the active ids, record for record after every hop,
and against per-stream oracle runs that skip the same hops."""
import numpy as np

import mixed_rate_cases as mc
import rate_cases as rc
import stream_dtx_cases as dc
from parity_cases import Guarded

KINDS = ("encode", "encode_dtx", "decode", "decode_track_noise", "decode_plc")
CNG_SEED = 9
PLC_FADE_SAMPLES = 640


def hop_mask(f, n, rng, p=0.6):
    """the mask of hop f: every seventh hop (from hop 3) sits every stream out, every seventh (from hop 5) runs all, the others
    are random"""
    if f % 7 == 3:
        return np.zeros(n, np.uint8)
    if f % 7 == 5:
        return np.ones(n, np.uint8)
    return (rng.random(n) < p).astype(np.uint8)


def _make(Context, api, max_streams, n, ctx_rate, mode, srate, sbits, dtx, split=None, stream=None):
    """a context at row rate ctx_rate whose streams 0..n-1 have the given own rates, bit counts (both roles) and DTX settings"""
    c = mc._make(Context, api, max_streams, ctx_rate, mode, CNG_SEED, split, stream)
    ids = np.arange(n, dtype=np.int32)
    if srate is not None:
        c.set_stream_sample_rates(srate, ids)
    if sbits is not None:
        c.set_stream_bits("encoder", sbits, ids)
        c.set_stream_bits("decoder", sbits, ids)
    if dtx is not None:
        c.set_stream_dtx(dtx, ids)
    return c


def _received(kind, f, n, rng):
    """decode_plc: a loss burst of 12 hops (4 concealed, then the fade into comfort noise, counted in the hops the stream runs)
    on every other stream, starting at a hop that depends on the stream; the plain decoders: random losses"""
    if kind == "decode_plc":
        k = np.arange(n)
        start = 2 + k % 4
        return np.where((k % 2 == 0) & (f >= start) & (f < start + 12), 0, 1).astype(np.uint8)
    return (rng.random(n) >= 0.2).astype(np.uint8)


def run_twin(Context, api, mem, wavs, kind, *, n, hops, tail=5, bits=64, split=None, mode="exact", ctx_rate=16000, rates=None,
             bit_set=None, dtx=None, seed=1):
    """kind's device twin over streams 0..n-1 with a mask that changes every hop (hop_mask), against a twin context that runs
    the host-buffer call over the active ids only.  The context has `tail` more streams than n and the mask buffer `tail` more
    rows, all 0: rows past n are not part of any call.  Every caller buffer is guarded (parity_cases.Guarded).  After every hop:
    active rows equal the twin's, the rows of streams that sat out are as specified, the exported records of every stream equal
    the twin's, and those of the streams that sat out equal their records before the hop."""
    max_streams = n + tail
    ids = np.arange(n, dtype=np.int32)
    srate = mc.interleaved(n, rates) if rates else None
    sbits = mc.interleaved(n, bit_set) if bit_set else None
    dtx_w = None if dtx is None else np.asarray(dtx, np.int32)
    row_rate = srate if srate is not None else np.full(n, ctx_rate, np.int32)
    row_bits = sbits if sbits is not None else np.full(n, bits, np.int32)
    P, H = int(dc.pbytes(bits)), rc.hop_of(ctx_rate)
    A = _make(Context, api, max_streams, n, ctx_rate, mode, srate, sbits, dtx_w, split, mem.stream)
    B = _make(Context, api, max_streams, n, ctx_rate, mode, srate, sbits, dtx_w)
    d_mask = Guarded(mem, n + tail, (), np.uint8, 0x5A)
    A.set_active_mask(d_mask.ptr)
    encoder = kind.startswith("encode")
    d_in = Guarded(mem, n, (H,) if encoder else (P,), np.int16 if encoder else np.uint8, 0x3C)
    d_rec = Guarded(mem, n, (), np.uint8, 0x77)
    d_out = Guarded(mem, n, (P,) if encoder else (H,), np.uint8 if encoder else np.int16, 0xA5)
    d_flags = Guarded(mem, n, (), np.uint8, 0xEE)
    rng = np.random.default_rng(seed)
    seen = set()
    for f in range(hops):
        m = hop_mask(f, n, rng)
        act = np.nonzero(m)[0].astype(np.int32)
        out = np.nonzero(m == 0)[0]
        d_mask.put(np.concatenate([m, np.zeros(tail, np.uint8)]))
        if encoder:
            x = dc.quiet_rows(wavs, row_rate, ids, f, H, rng, hops)
        else:
            x = rng.integers(0, 256, size=(n, P)).astype(np.uint8)
        rec = _received(kind, f, n, rng)
        d_in.put(x)
        d_rec.put(np.where(m != 0, rec, 0x77))     # the byte of a stream that sits out is not read
        d_out.fill()
        d_flags.fill()
        before = A.export_streams()
        if kind == "encode":
            A.encode_device(n, d_in.ptr, bits, d_out.ptr)
        elif kind == "encode_dtx":
            A.encode_dtx_device(n, d_in.ptr, bits, d_out.ptr, d_flags.ptr)
        elif kind == "decode":
            A.decode_device(n, d_in.ptr, d_rec.ptr, bits, d_out.ptr)
        elif kind == "decode_track_noise":
            A.decode_track_noise_device(n, d_in.ptr, d_rec.ptr, bits, d_out.ptr, d_flags.ptr)
        else:
            A.decode_plc_device(n, d_in.ptr, d_rec.ptr, bits, d_out.ptr, d_flags.ptr)
        got, flags = d_out.get("output"), d_flags.get("flags")
        d_in.get("input")
        d_rec.get("received")
        d_mask.get("mask")
        # the rows of the streams that sit out
        if len(out):
            assert not got[out].any(), "hop %d: a stream that sat out has a nonzero output row (%s)" % (f, kind)
            if kind == "encode_dtx":
                assert (flags[out] == 1).all(), "hop %d: the DTX flag of a stream that sat out is not 1" % f
            elif kind == "decode_track_noise":
                want = B.noise_estimate(stream_ids=out)[1]
                assert np.array_equal(flags[out], want.astype(np.uint8)), "hop %d: is_noise of a stream that sat out" % f
            elif kind == "decode_plc":
                want = B.plc_state(stream_ids=out)[:, 1] == PLC_FADE_SAMPLES
                assert np.array_equal(flags[out], want.astype(np.uint8)), "hop %d: is_comfort_noise of a stream that sat out" % f
        # the active rows against the twin's host-buffer call over exactly those ids
        if len(act):
            if kind == "encode":
                w = B.encode(x[act], bits, stream_ids=act)
                assert np.array_equal(got[act], w), "hop %d: encode_device != encode over the active ids" % f
            elif kind == "encode_dtx":
                w, sizes = B.encode_dtx(x[act], bits, stream_ids=act)
                assert np.array_equal(got[act], w), "hop %d: encode_dtx_device packets != encode_dtx" % f
                assert np.array_equal(flags[act], (sizes == 0).astype(np.uint8)), "hop %d: DTX flags != encode_dtx" % f
                seen |= set(int(s == 0) for s in sizes)
            elif kind == "decode":
                w = B.decode(x[act], bits, stream_ids=act, received=rec[act])
                assert np.array_equal(got[act], w), "hop %d: decode_device != decode over the active ids" % f
            elif kind == "decode_track_noise":
                w, wf = B.decode_track_noise(x[act], bits, stream_ids=act, received=rec[act])
                assert np.array_equal(got[act], w) and np.array_equal(flags[act], wf.astype(np.uint8)), \
                    "hop %d: decode_track_noise_device != decode_track_noise" % f
            else:
                w, wf = B.decode_plc(x[act], bits, stream_ids=act, received=rec[act])
                assert np.array_equal(got[act], w) and np.array_equal(flags[act], wf.astype(np.uint8)), \
                    "hop %d: decode_plc_device != decode_plc" % f
                seen |= set(int(v) for v in wf)
        after = A.export_streams()
        assert np.array_equal(after[out], before[out]), "hop %d: the state of a stream that sat out changed (%s)" % (f, kind)
        assert np.array_equal(after[n:], before[n:]), "hop %d: a stream past n changed" % f
        assert np.array_equal(after, B.export_streams()), "hop %d: stream records differ from the twin's (%s)" % (f, kind)
    if kind == "encode_dtx" and (dtx_w is None or dtx_w.any()):
        assert seen == {0, 1}, "the DTX-on streams must produce both empty and encoded hops: %s" % seen
    if kind == "decode_plc":
        assert seen == {0, 1}, "the loss bursts must reach comfort noise: %s" % seen
    A.set_active_mask(None)
    for c in (A, B):
        c.close()


def _device_calls(ctx, mem, n, H, P, bits, x, pk_in, rec):
    """the five device twins once each on one context; -> (outputs, launches per call)"""
    d_pcm = mem.zeros((n, H), np.int16)
    mem.put(d_pcm, x)
    d_pk = mem.zeros((n, P), np.uint8)
    mem.put(d_pk, pk_in)
    d_rec = mem.zeros((n,), np.uint8)
    mem.put(d_rec, rec)
    outs, counts = [], []
    for call in ("encode", "encode_dtx", "decode", "decode_track_noise", "decode_plc"):
        o = mem.zeros((n, P if call.startswith("encode") else H), np.uint8 if call.startswith("encode") else np.int16)
        fl = mem.zeros((n,), np.uint8)
        l0 = ctx.launch_count
        if call == "encode":
            ctx.encode_device(n, mem.ptr(d_pcm), bits, mem.ptr(o))
        elif call == "encode_dtx":
            ctx.encode_dtx_device(n, mem.ptr(d_pcm), bits, mem.ptr(o), mem.ptr(fl))
        elif call == "decode":
            ctx.decode_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(o))
        elif call == "decode_track_noise":
            ctx.decode_track_noise_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(o), mem.ptr(fl))
        else:
            ctx.decode_plc_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(o), mem.ptr(fl))
        counts.append(ctx.launch_count - l0)
        outs += [mem.get(o), mem.get(fl)]
    return outs, counts


def run_ones_zeros_and_launches(Context, api, mem, wav16, *, n, hops=4, bits=64, split=None, mode="exact", seed=2):
    """Four contexts run the five device twins hop by hop: no mask, an all-ones mask, a random mask and a mask that is installed
    and uninstalled again.  Launches per call are equal in all four; the all-ones and the uninstalled contexts are bit-identical
    to the one without a mask, outputs and records.  Then an all-zero mask: every call changes no stream, writes zero rows and
    the specified flags."""
    H, P = 320, int(dc.pbytes(bits))
    ctxs = [mc._make(Context, api, n, 16000, mode, CNG_SEED, split, mem.stream) for _ in range(4)]
    masks = [mem.zeros((n,), np.uint8) for _ in range(3)]
    mem.put(masks[0], np.ones(n, np.uint8))
    ctxs[1].set_active_mask(mem.ptr(masks[0]))
    ctxs[2].set_active_mask(mem.ptr(masks[1]))
    ctxs[3].set_active_mask(mem.ptr(masks[0]))
    ctxs[3].set_active_mask(None)
    rng = np.random.default_rng(seed)
    ids = np.arange(n)
    for f in range(hops):
        mem.put(masks[1], hop_mask(f, n, rng))
        x = dc.quiet_rows({16000: wav16}, np.full(n, 16000, np.int32), ids, f, H, rng, hops)
        pk = rng.integers(0, 256, size=(n, P)).astype(np.uint8)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        res = [_device_calls(c, mem, n, H, P, bits, x, pk, rec) for c in ctxs]
        assert res[0][1] == res[1][1] == res[2][1] == res[3][1], "hop %d: launches per call differ: %s" % (f, [r[1] for r in res])
        for k in (1, 3):
            for a, b in zip(res[0][0], res[k][0]):
                assert np.array_equal(a, b), "hop %d: context %d differs from the one without a mask" % (f, k)
            assert np.array_equal(ctxs[0].export_streams(), ctxs[k].export_streams()), "hop %d: records of context %d differ" % (f, k)
    # all zeros: nothing changes
    mem.put(masks[2], np.zeros(n, np.uint8))
    c = ctxs[2]
    c.set_active_mask(mem.ptr(masks[2]))
    before = c.export_streams()
    x = dc.quiet_rows({16000: wav16}, np.full(n, 16000, np.int32), ids, hops, H, rng, hops)
    outs, counts = _device_calls(c, mem, n, H, P, bits, x, np.full((n, P), 0x5B, np.uint8), np.ones(n, np.uint8))
    assert counts == res[0][1], "an all-zero mask changed the launch counts"
    assert np.array_equal(c.export_streams(), before), "an all-zero mask changed a stream"
    enc, enc_fl, dtx, dtx_fl, dec, _, dtn, dtn_fl, plc, plc_fl = outs
    assert not enc.any() and not dtx.any() and not dec.any() and not dtn.any() and not plc.any(), "an all-zero mask left a nonzero row"
    assert (dtx_fl == 1).all(), "an all-zero mask: encode_dtx_device flags must be 1"
    assert np.array_equal(dtn_fl, c.noise_estimate(n=n)[1].astype(np.uint8)), "an all-zero mask: is_noise must be the current flag"
    assert np.array_equal(plc_fl, (c.plc_state(n=n)[:, 1] == PLC_FADE_SAMPLES).astype(np.uint8)), "an all-zero mask: comfort-noise flag"
    for x_ in ctxs:
        x_.close()


def run_oracle_spot(Context, api, O, mem, wav16, *, n, hops, rows, bits=64, seed=4):
    """Exact mode, 16 kHz: encode_device and decode_device (of the packets just encoded) with a random mask every hop, against
    per-stream oracle codecs that skip the hops their stream sits out, on a sample of rows."""
    H, P = 320, int(dc.pbytes(bits))
    ctx = mc._make(Context, api, n, 16000, "exact", CNG_SEED, None, mem.stream)
    d_mask = Guarded(mem, n, (), np.uint8, 0x5A)
    ctx.set_active_mask(d_mask.ptr)
    d_pcm, d_pk, d_out = Guarded(mem, n, (H,), np.int16, 0x3C), Guarded(mem, n, (P,), np.uint8, 0xFF), Guarded(mem, n, (H,), np.int16, 0x3C)
    orc = {r: rc.OracleCodec(O, 16000) for r in rows}
    rng = np.random.default_rng(seed)
    skipped = set()
    for f in range(hops):
        m = hop_mask(f, n, rng, p=0.5)
        d_mask.put(m)
        x = rc.speech_rows(wav16, 16000, range(n), f)
        d_pcm.put(x)
        d_pk.fill()
        d_out.fill()
        ctx.encode_device(n, d_pcm.ptr, bits, d_pk.ptr)
        ctx.decode_device(n, d_pk.ptr, 0, bits, d_out.ptr)
        pk, pcm = d_pk.get("packets"), d_out.get("PCM")
        for r in rows:
            if not m[r]:
                assert not pk[r].any() and not pcm[r].any(), "hop %d row %d sat out: nonzero output" % (f, r)
                skipped.add(r)
                continue
            want = orc[r].encode(x[r], bits)
            assert bytes(pk[r]) == want, "hop %d row %d: packet != oracle" % (f, r)
            assert np.array_equal(pcm[r], orc[r].decode(want, bits)), "hop %d row %d: PCM != oracle" % (f, r)
    assert skipped, "no sampled row sat out"
    ctx.close()


def run_setter(Context, api, LyraB200Error):
    """NULL context -> EINVAL; any context, either role, accepts a pointer and NULL without launching anything"""
    assert api.lib.lyra_b200_set_active_mask(None, None) == mc.EINVAL
    for roles in ("both", "encoder", "decoder"):
        c = Context(8, capi=api, roles=roles)
        l0 = c.launch_count
        buf = np.ones(8, np.uint8)
        c.set_active_mask(buf.ctypes.data)
        c.set_active_mask(None)
        assert c.launch_count == l0
        c.close()
