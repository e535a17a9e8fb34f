"""Cases for per-stream sample rates (lyra_b200_set_stream_sample_rates), shared by the CPU tier (emulated kernels) and the GPU
tier.  A stream at rate r in a context of a higher row rate must behave exactly like the same stream id in a context whose rate
is r, fed the same first r / 50 samples of its rows: bit-exact packets, flags, packet_bytes, control state and PCM (the rest of a
decoder row is 0).  A sample of streams is also checked against the oracle composition of rate_cases.py."""
import numpy as np

import rate_cases as rc
from parity_cases import TENSOR_PCM_TOL_LSB, Guarded

EINVAL = -1
ALL_RATES = (8000, 16000, 32000, 48000)
CALLS = ("codec", "track", "plc", "dtx")


def interleaved(n, rates):
    """rates[k % len(rates)] for row k: with 4 rates (or 2) every tile of 8 streams mixes them"""
    return np.array([rates[k % len(rates)] for k in range(n)], dtype=np.int32)


def _fails_einval(fn, LyraB200Error):
    try:
        fn()
    except LyraB200Error as e:
        assert e.code == EINVAL, e
        return True
    return False


def mixed_rows(wavs, srate, ids, f, row, rng, silent=None):
    """Hop f of each id at its own rate: speech in the first rate / 50 samples of a `row`-sample row, random data after it (the
    encoders must ignore it).  silent[k]: the speech part of row k is 0.  -> (rows[n][row], {rate: rows[rows of that rate][rate / 50]})"""
    n = len(ids)
    out = rng.integers(-20000, 20000, size=(n, row)).astype(np.int16)
    by_rate = {}
    for r in sorted(set(int(x) for x in srate)):
        sel = np.nonzero(srate == r)[0]
        x = rc.speech_rows(wavs[r], r, ids[sel], f)
        if silent is not None:
            x[silent[sel]] = 0
        out[sel, :rc.hop_of(r)] = x
        by_rate[r] = x
    return out, by_rate


def _make(Context, api, max_streams, rate, mode, cng_seed, split=None, stream=None):
    c = Context(max_streams, capi=api)
    c.set_sample_rate(rate)
    c.set_decoder_mode(mode)
    c.set_cng_seed(cng_seed)
    if split is not None:
        c.set_split(split)
    if stream is not None:
        c.set_stream(stream)
    return c


def _check_rows(got, want, sel, r, what):
    """the first r / 50 samples of rows `sel` of `got` equal `want`, the rest of those rows is 0"""
    h = rc.hop_of(r)
    bad = np.nonzero((got[sel, :h] != want).any(axis=1))[0]
    assert bad.size == 0, "%s: rows %s at %d Hz differ from the single-rate twin" % (what, sel[bad[:8]], r)
    assert not got[sel, h:].any(), "%s: a row tail at %d Hz is not 0" % (what, r)


def run_mixed_parity(Context, api, O, wavs, *, ctx_rate, rates, max_streams, stream_ids=None, n=None, frames=10, oracle_rows=(),
                     decoder_mode="exact", split=None, mem=None, cng_seed=7, seed=1):
    """Every fused call with streams at interleaved rates in one context of row rate ctx_rate, hop by hop, against twin streams
    (same ids) in one single-rate context per rate fed the same rows.  mem None: the host-buffer calls (stream_ids None = dense
    streams 0..n-1); otherwise the *_device twins over streams 0..n-1 with guarded caller buffers.  Inputs: speech, every third
    stream silent in the second half (DTX, the estimators' noise branch), random row tails; decode / decode_track_noise lose random
    packets, decode_plc bursts of 7 (into comfort noise and back) or 2; the bit rate changes every fourth hop.  oracle_rows: rows
    also checked against the oracle composition at their rate."""
    ids = np.arange(n, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    device = mem is not None
    assert not (device and stream_ids is not None), "the device calls serve streams 0..n-1"
    call_ids = None if stream_ids is None else ids
    srate = interleaved(n, rates)
    H = rc.hop_of(ctx_rate)
    exact = decoder_mode == "exact"
    stream = mem.stream if device else None
    mixed = {k: _make(Context, api, max_streams, ctx_rate, decoder_mode, cng_seed, split, stream) for k in CALLS}
    for c in mixed.values():
        c.set_stream_sample_rates(srate, ids)
        assert np.array_equal(c.stream_sample_rates(ids), srate)
    present = sorted(set(int(r) for r in srate))
    sel = {r: np.nonzero(srate == r)[0] for r in present}
    twins = {r: {k: _make(Context, api, max_streams, r, decoder_mode, cng_seed) for k in CALLS} for r in present}
    tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    orc = {k: dict(codec=rc.OracleCodec(O, int(srate[k])), track=rc.OracleCodec(O, int(srate[k]), track=True),
                   plc=rc.OraclePlcDecoder(O, int(srate[k]), cng_seed + int(ids[k])), dtx=rc.OracleEncoder(O, int(srate[k]), dtx=True))
           for k in oracle_rows}
    if device:
        G = lambda row, dtype, s: Guarded(mem, n, row, dtype, s)     # noqa: E731
        d_pcm, d_rec, d_plc_rec = G((H,), np.int16, 0x3C), G((), np.uint8, 0xC3), G((), np.uint8, 0xC3)
        d_out, d_trk, d_plc = G((H,), np.int16, 0x5A), G((H,), np.int16, 0x5A), G((H,), np.int16, 0x5A)
        d_trk_flags, d_cn, d_dtx_flags = (G((), np.uint8, 0xAA) for _ in range(3))
    rng = np.random.default_rng(seed)
    burst = [(1 + k % 3, 7 if k % 2 == 0 else 2) for k in range(n)]
    seen = dict(cn=False, dtx=set(), loss=False)
    for f in range(frames):
        bits = (64, 120, 184)[(f // 4) % 3]
        P = (bits + 7) // 8
        silent = (np.arange(n) % 3 == 0) & (f >= frames // 2)
        pcm, pcm_r = mixed_rows(wavs, srate, ids, f, H, rng, silent)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        rec_trk = (rng.random(n) >= 0.25).astype(np.uint8)
        rec_plc = np.array([0 if b0 <= f < b0 + bl else 1 for b0, bl in burst], dtype=np.uint8)
        if device:
            d_pcm.put(pcm)
            d_rec.put(rec)
            d_plc_rec.put(rec_plc)
            d_pk, d_dtx_pk = G((P,), np.uint8, 0xA5), G((P,), np.uint8, 0xFF)
            for buf in (d_out, d_trk, d_plc, d_trk_flags, d_cn, d_dtx_flags):
                buf.fill()
            mixed["codec"].encode_device(n, d_pcm.ptr, bits, d_pk.ptr)
            pk = d_pk.get("packets")
            mixed["codec"].decode_device(n, d_pk.ptr, d_rec.ptr, bits, d_out.ptr)
            d_rec.put(rec_trk)
            mixed["track"].decode_track_noise_device(n, d_pk.ptr, d_rec.ptr, bits, d_trk.ptr, d_trk_flags.ptr)
            mixed["plc"].decode_plc_device(n, d_pk.ptr, d_plc_rec.ptr, bits, d_plc.ptr, d_cn.ptr)
            mixed["dtx"].encode_dtx_device(n, d_pcm.ptr, bits, d_dtx_pk.ptr, d_dtx_flags.ptr)
            out = d_out.get("PCM")
            t_out, t_flags = d_trk.get("PCM"), d_trk_flags.get("flags").astype(bool)
            p_out, p_cn = d_plc.get("PCM"), d_cn.get("flags").astype(bool)
            x_pk, x_sizes = d_dtx_pk.get("packets"), np.where(d_dtx_flags.get("flags") != 0, 0, P)
            d_pcm.get("input PCM")
        else:
            pk = mixed["codec"].encode(pcm, bits, stream_ids=call_ids)
            out = mixed["codec"].decode(pk, bits, stream_ids=call_ids, received=rec)
            t_out, t_flags = mixed["track"].decode_track_noise(pk, bits, stream_ids=call_ids, received=rec_trk)
            p_out, p_cn = mixed["plc"].decode_plc(pk, bits, stream_ids=call_ids, received=rec_plc)
            x_pk, x_sizes = mixed["dtx"].encode_dtx(pcm, bits, stream_ids=call_ids)
        assert out.shape == (n, H)
        p_state = mixed["plc"].plc_state(stream_ids=ids)
        for r in present:
            s, tw = sel[r], twins[r]
            what = "hop %d, %d Hz streams in a %d Hz context" % (f, r, ctx_rate)
            tpk = tw["codec"].encode(pcm_r[r], bits, stream_ids=ids[s])
            assert np.array_equal(pk[s], tpk), "encode: " + what
            _check_rows(out, tw["codec"].decode(tpk, bits, stream_ids=ids[s], received=rec[s]), s, r, "decode, " + what)
            w_out, w_flags = tw["track"].decode_track_noise(tpk, bits, stream_ids=ids[s], received=rec_trk[s])
            _check_rows(t_out, w_out, s, r, "decode_track_noise, " + what)
            assert np.array_equal(t_flags[s], w_flags), "decode_track_noise flags: " + what
            w_out, w_cn = tw["plc"].decode_plc(tpk, bits, stream_ids=ids[s], received=rec_plc[s])
            _check_rows(p_out, w_out, s, r, "decode_plc, " + what)
            assert np.array_equal(p_cn[s], w_cn), "comfort-noise flags: " + what
            assert np.array_equal(p_state[s], tw["plc"].plc_state(stream_ids=ids[s])), "control state: " + what
            w_pk, w_sizes = tw["dtx"].encode_dtx(pcm_r[r], bits, stream_ids=ids[s])
            assert np.array_equal(x_sizes[s], w_sizes) and np.array_equal(x_pk[s], w_pk), "encode_dtx: " + what
        for k, o in orc.items():
            r, h = int(srate[k]), rc.hop_of(int(srate[k]))
            x = pcm[k, :h]
            opkt = o["codec"].encode(x, bits)
            assert bytes(pk[k]) == opkt, "encode != oracle at %d Hz, hop %d stream %d" % (r, f, ids[k])
            d = rc._pcm_diff(out[k, :h], o["codec"].decode(opkt if rec[k] else None, bits))
            assert d <= tol, "decode != oracle at %d Hz, hop %d stream %d: %d" % (r, f, ids[k], d)
            d = rc._pcm_diff(t_out[k, :h], o["track"].decode(opkt if rec_trk[k] else None, bits))
            assert d <= tol, "decode_track_noise != oracle at %d Hz, hop %d stream %d: %d" % (r, f, ids[k], d)
            if exact:
                assert bool(t_flags[k]) == o["track"].est.is_noise, (f, k)
            d = rc._pcm_diff(p_out[k, :h], o["plc"].tick(opkt if rec_plc[k] else None))
            assert d <= tol, "decode_plc != oracle at %d Hz, hop %d stream %d: %d" % (r, f, ids[k], d)
            assert tuple(int(v) for v in p_state[k]) == o["plc"].dec.state, (f, k)
            want = o["dtx"].encode(x, bits)
            assert x_sizes[k] == len(want) and bytes(x_pk[k][:x_sizes[k]]) == want, "encode_dtx != oracle, hop %d stream %d" % (f, ids[k])
        seen["loss"] |= not rec.all()
        seen["cn"] |= bool(p_cn.any())
        seen["dtx"] |= set(int(v == 0) for v in x_sizes)
    assert seen["loss"] and seen["cn"], "the case must lose packets and reach comfort noise"
    assert seen["dtx"] == {0, 1}, "the case must produce both DTX and encoded hops"
    for c in list(mixed.values()) + [c for tw in twins.values() for c in tw.values()]:
        c.close()


def run_rate_change_mid_call(Context, api, O, wavs, *, ctx_rate=48000, max_streams=16, stream_ids=(1, 2, 5, 11),
                             schedule=((8000, 48000, 16000, 32000), (48000, 8000, 16000, 16000), (32000, 8000, 48000, 16000)),
                             hops=3, bits=64, seed=2):
    """The streams' rates change between calls (schedule[i] holds for `hops` hops): every hop equals the oracle composition whose
    converters restart fresh at each change while the codec state carries on; a stream whose rate stays keeps its converters.
    A twin context gets the same calls plus, before every hop, set_stream_sample_rates to the rates the streams already have: its
    outputs and the launch counts of its codec calls equal the first context's."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    a, b = Context(max_streams, capi=api), Context(max_streams, capi=api)
    for c in (a, b):
        c.set_sample_rate(ctx_rate)
    rng = np.random.default_rng(seed)
    H = rc.hop_of(ctx_rate)
    ref = {k: rc.OracleCodec(O, int(schedule[0][k])) for k in range(n)}
    f = 0
    for i, rates in enumerate(schedule):
        srate = np.asarray(rates, dtype=np.int32)
        for c in (a, b):
            c.set_stream_sample_rates(srate, ids)
        if i:
            for k in range(n):
                if srate[k] != schedule[i - 1][k]:
                    ref[k].set_rate(O, int(srate[k]))
        for _ in range(hops):
            b.set_stream_sample_rates(srate, ids)                # the rates the streams have: nothing changes
            pcm, _ = mixed_rows(wavs, srate, ids, f, H, rng)
            outs = []
            for c in (a, b):
                l0 = c.launch_count
                pk = c.encode(pcm, bits, stream_ids=ids)
                outs.append((pk, c.decode(pk, bits, stream_ids=ids), c.launch_count - l0))
            assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1]), \
                "setting the current rates changed an output, hop %d" % f
            assert outs[0][2] == outs[1][2], "setting the current rates changed the calls' launches, hop %d" % f
            pk, out = outs[0][0], outs[0][1]
            for k in range(n):
                h = rc.hop_of(int(srate[k]))
                opkt = ref[k].encode(pcm[k, :h], bits)
                assert bytes(pk[k]) == opkt, "encode after a rate change != oracle, hop %d stream %d" % (f, ids[k])
                assert np.array_equal(out[k, :h], ref[k].decode(opkt, bits)), "decode after a rate change, hop %d stream %d" % (f, ids[k])
                assert not out[k, h:].any()
            f += 1
    for c in (a, b):
        c.close()


def _every_call(c, f, ids, srate, wavs, H, bits, rng, keys=None):
    """one hop of encode_dtx, encode and decode_plc (packets lost on hops 2..9 for every other row) on ids at their rates; the
    audio of row k is that of stream keys[k] (default: ids[k]), so a moved stream can be fed what it had at its old id"""
    n = len(ids)
    pcm, _ = mixed_rows(wavs, srate, ids if keys is None else keys, f, H, rng, silent=(np.arange(n) % 2 == 0) & (f >= 6))
    pk, sizes = c.encode_dtx(pcm, bits, stream_ids=ids)
    lost = (np.arange(n) % 2 == 1) & (f >= 2) & (f <= 9)
    out, cn = c.decode_plc(c.encode(pcm, bits, stream_ids=ids), bits, stream_ids=ids, received=(~lost).astype(np.uint8))
    return {"dtx": pk, "dtx_bytes": sizes, "plc_pcm": out, "cn": cn, "plc_state": c.plc_state(stream_ids=ids)}


def run_moves(Context, api, wavs, *, max_streams=16, ctx_rate=48000, ids=(2, 5), rates=(8000, 48000), copy_to=(10, 13),
              import_to=(7, 0), hops=11, after=3, bits=64, cng_seed=5):
    """Streams at 8 and 48 kHz in a 48 kHz context, after a history that reaches comfort noise and DTX: moved with copy_streams in
    their context and with export / import into a second context (which reached 48 kHz through another rate), they continue bit
    for bit like a twin that was not moved, and carry their rates.  Then reset and copy_streams from -1 put a stream back at the
    context's rate, and set_sample_rate puts every stream at its rate."""
    ids, copy_to, import_to = (np.asarray(x, np.int32) for x in (ids, copy_to, import_to))
    srate = np.asarray(rates, np.int32)
    H = rc.hop_of(ctx_rate)

    def make(path):
        c = Context(max_streams, capi=api)
        c.set_cng_seed(cng_seed)
        for r in path:
            c.set_sample_rate(r)
        return c
    A, T, B = make([ctx_rate]), make([ctx_rate]), make([32000, ctx_rate])
    for c in (A, T):
        c.set_stream_sample_rates(srate, ids)
    seen_cn = seen_dtx = False
    for f in range(hops):
        oa = _every_call(A, f, ids, srate, wavs, H, bits, np.random.default_rng(f))
        _every_call(T, f, ids, srate, wavs, H, bits, np.random.default_rng(f))
        seen_cn |= bool(oa["cn"].any())
        seen_dtx |= bool((oa["dtx_bytes"] == 0).any())
    assert seen_cn and seen_dtx, "the history must reach comfort noise and DTX"
    A.copy_streams(ids, copy_to)
    B.import_streams(T.export_streams(ids), import_to)
    assert np.array_equal(A.stream_sample_rates(copy_to), srate) and np.array_equal(B.stream_sample_rates(import_to), srate)
    for f in range(hops, hops + after):
        ot = _every_call(T, f, ids, srate, wavs, H, bits, np.random.default_rng(f))
        for c, where in ((A, copy_to), (B, import_to)):
            o = _every_call(c, f, where, srate, wavs, H, bits, np.random.default_rng(f), keys=ids)
            for name, v in o.items():
                assert np.array_equal(v, ot[name]), "%s of a moved stream differs, hop %d (%s)" % (name, f, "copy" if c is A else "import")
    A.reset(copy_to[:1])
    A.copy_streams([-1], copy_to[1:])
    assert list(A.stream_sample_rates(copy_to)) == [ctx_rate] * len(copy_to), "reset / copy from -1 must restore the context rate"
    assert np.array_equal(A.stream_sample_rates(ids), srate), "the sources keep their rates"
    B.set_sample_rate(ctx_rate)
    assert set(B.stream_sample_rates().tolist()) == {ctx_rate}, "set_sample_rate must put every stream at the context's rate"
    T.set_sample_rate(32000)
    assert set(T.stream_sample_rates().tolist()) == {32000}
    for c in (A, T, B):
        c.close()


def run_validation(Context, api, wavs, LyraB200Error, *, max_streams=16, ctx_rate=32000, ids=(2, 5, 11, 12), bits=64):
    """Each refused call returns EINVAL and changes no stream: the following export and rates equal the ones before."""
    ids = np.asarray(ids, np.int32)
    srate = np.asarray((8000, 32000, 16000, 8000), np.int32)
    ctx = Context(max_streams, capi=api)
    ctx.set_sample_rate(ctx_rate)
    ctx.set_stream_sample_rates(srate, ids)
    rng = np.random.default_rng(9)
    for f in range(2):
        _every_call(ctx, f, ids, srate, wavs, rc.hop_of(ctx_rate), bits, rng)
    good = ctx.export_streams(ids)
    # the rate word is the last entry of the state list, so the last word of a record
    assert np.array_equal(good.view(np.uint32)[:, -1], np.where(srate == ctx_rate, 0, srate)), "rate word not where expected"
    before, rates_before = ctx.export_streams(), ctx.stream_sample_rates()

    def with_rate(word):
        r = good.copy()
        r.view(np.uint32)[1, -1] = word
        return r
    for what, call in {
        "an unsupported rate": lambda: ctx.set_stream_sample_rates([44100], [3]),
        "rate 0": lambda: ctx.set_stream_sample_rates([0], [3]),
        "rate 16001": lambda: ctx.set_stream_sample_rates([8000, 16001], [3, 4]),
        "a rate above the context's": lambda: ctx.set_stream_sample_rates([8000, 48000], [3, 4]),
        "repeated ids": lambda: ctx.set_stream_sample_rates([8000, 16000], [6, 6]),
        "an id out of range": lambda: ctx.set_stream_sample_rates([8000], [max_streams]),
        "a record with an unsupported rate word": lambda: ctx.import_streams(with_rate(44100), ids),
        "a record with a rate above the context's": lambda: ctx.import_streams(with_rate(48000), ids),
        "a record with rate word 16001": lambda: ctx.import_streams(with_rate(16001), ids),
    }.items():
        assert _fails_einval(call, LyraB200Error), "accepted %s" % what
    assert np.array_equal(ctx.export_streams(), before), "a refused call changed a stream"
    assert np.array_equal(ctx.stream_sample_rates(), rates_before)
    ctx.import_streams(with_rate(16000), ids)            # a supported rate below the context's is a valid record
    assert ctx.stream_sample_rates(ids)[1] == 16000
    ctx.close()


def run_16khz_unchanged(Context, api, wav16, *, max_streams=16, stream_ids=(0, 3, 9), hops=2, bits=64, seed=3):
    """A 16 kHz context given set_stream_sample_rates(..., 16000) equals one that never was, launch counts included, in every
    fused call: nothing new launches."""
    ids = np.asarray(stream_ids, np.int32)
    n = len(ids)
    c, d = Context(max_streams, capi=api), Context(max_streams, capi=api)
    c.set_stream_sample_rates(np.full(n, 16000, np.int32), ids)
    c.set_stream_sample_rates(np.full(max_streams, 16000, np.int32))
    rng = np.random.default_rng(seed)
    for f in range(hops):
        x = rc.speech_rows(wav16, 16000, ids, f)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        res = []
        for ctx in (c, d):
            pk = ctx.encode(x, bits, stream_ids=ids)
            res.append([pk, ctx.decode(pk, bits, stream_ids=ids, received=rec), ctx.encode(x, bits), ctx.decode(pk, bits),
                        *ctx.decode_track_noise(pk, bits, stream_ids=ids, received=rec), *ctx.decode_plc(pk, bits, stream_ids=ids),
                        *ctx.encode_dtx(x, bits, stream_ids=ids), *ctx.encode_dtx(x, bits)])
        for u, v in zip(*res):
            assert np.array_equal(u, v)
    assert c.launch_count == d.launch_count, (c.launch_count, d.launch_count)
    c.close()
    d.close()
