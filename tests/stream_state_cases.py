"""Cases for moving live streams (lyra_b200_export_streams / _import_streams / _copy_streams), shared by the CPU tier (emulated
kernels) and the GPU tier (real kernels).  The bar is bit-exactness: a moved stream continues exactly as it would have at its
old id, and nothing else changes."""
import numpy as np

from parity_cases import _every_stateful_call

EINVAL = -1


def _fails_einval(fn, LyraB200Error):
    try:
        fn()
    except LyraB200Error as e:
        assert e.code == EINVAL, e
        return True
    return False


def _history(ctx, ids, wav, hops, bits, f0=0):
    """hops f0 .. f0 + hops - 1 of every stateful call on `ids`; asserts that comfort noise and DTX were reached"""
    seen_cn = seen_dtx = False
    for f in range(f0, f0 + hops):
        o = _every_stateful_call(ctx, f, ids, wav, bits)
        seen_cn |= bool(o["comfort_noise"].any())
        seen_dtx |= bool((o["dtx_bytes"] == 0).any())
    assert seen_cn and seen_dtx, "the history must reach comfort noise and DTX"


def _assert_rows_equal(got, want, rows, what):
    for name, r in got.items():
        for k in rows:
            assert np.array_equal(r[k], want[name][k]), "%s: %s differs at row %d" % (what, name, k)


def run_move_between_contexts(Context, api, wav, *, max_streams, a_ids, a_fill, b_ids, b_live, hops=9, after=3, bits=64,
                              cng_seed=3, mode="exact", devices=(0, 0)):
    """Context A runs a history through every stateful call on a_ids (long enough for comfort noise and DTX) and a_fill; context
    B runs other work on b_live.  A's streams a_ids are exported and imported into B at b_ids.  For `after` more hops A runs
    a_ids + a_fill and B runs b_ids + b_live with the same inputs row by row: every output of B's moved rows equals A's, the
    control state included, and B's live rows equal those of a twin of B that imported nothing."""
    a_ids, b_ids = np.asarray(a_ids, np.int32), np.asarray(b_ids, np.int32)
    assert len(a_fill) == len(b_live) and len(a_ids) == len(b_ids)

    def make(dev):
        c = Context(max_streams, capi=api, device=dev)
        c.set_cng_seed(cng_seed)
        c.set_decoder_mode(mode)
        return c
    A, B, twin = make(devices[0]), make(devices[1]), make(devices[1])
    a_all = np.concatenate([a_ids, np.asarray(a_fill, np.int32)])
    b_all = np.concatenate([b_ids, np.asarray(b_live, np.int32)])
    _history(A, a_all, wav, hops, bits)
    for c in (B, twin):
        for f in range(hops):
            _every_stateful_call(c, f + 40, np.asarray(b_live, np.int32), wav, bits)
    recs = A.export_streams(a_ids)
    assert recs.shape == (len(a_ids), A.stream_state_bytes())
    B.import_streams(recs, b_ids)
    moved, live = range(len(a_ids)), range(len(a_ids), len(b_all))
    for f in range(hops, hops + after):
        oa = _every_stateful_call(A, f, a_all, wav, bits)
        ob = _every_stateful_call(B, f, b_all, wav, bits)
        ot = _every_stateful_call(twin, f, b_all, wav, bits)
        _assert_rows_equal(ob, oa, moved, "moved stream, hop %d" % f)
        _assert_rows_equal(ob, ot, live, "stream of B that was not moved, hop %d" % f)
    for c in (A, B, twin):
        c.close()


def _hop48(wav48, f, n):
    return np.stack([wav48[(960 * (f + 7 * k + 3)) % (len(wav48) - 960):][:960] for k in range(n)]).copy()


def run_move_at_48k(Context, api, wav48, LyraB200Error, *, max_streams=16, a_ids=(2, 9, 13), b_ids=(11, 0, 5), hops=10, after=3,
                    bits=64, cng_seed=5):
    """The move at 48 kHz through encode_dtx and decode_plc, the codec converters mid-stream.  B reached 48 kHz through another rate,
    so its converter tag differs from A's: import must rewrite it for the move to be exact.  A context at another rate refuses
    the records."""
    a_ids, b_ids = np.asarray(a_ids, np.int32), np.asarray(b_ids, np.int32)
    n = len(a_ids)

    def make(rates):
        c = Context(max_streams, capi=api)
        c.set_cng_seed(cng_seed)
        for r in rates:
            c.set_sample_rate(r)
        return c
    A, B, other = make([48000]), make([32000, 48000]), make([32000])
    lost = lambda f: (np.arange(n) + f) % 5 != 0 if f < 2 or f > 8 else np.zeros(n, bool)    # noqa: E731

    def hop(c, f, ids):
        pcm = _hop48(wav48, f, n)
        quiet = pcm.copy()
        quiet[::2] //= 64
        pk, sizes = c.encode_dtx(quiet, bits, stream_ids=ids)
        out, cn = c.decode_plc(c.encode(pcm, bits, stream_ids=ids), bits, stream_ids=ids, received=lost(f).astype(np.uint8))
        return {"dtx": pk, "dtx_bytes": sizes, "plc_pcm": out, "cn": cn, "plc_state": c.plc_state(stream_ids=ids)}
    seen_cn = False
    for f in range(hops):
        seen_cn |= bool(hop(A, f, a_ids)["cn"].any())
    assert seen_cn
    recs = A.export_streams(a_ids)
    assert _fails_einval(lambda: other.import_streams(recs, b_ids), LyraB200Error), "a context at another rate took the records"
    B.import_streams(recs, b_ids)
    for f in range(hops, hops + after):
        oa, ob = hop(A, f, a_ids), hop(B, f, b_ids)
        _assert_rows_equal(ob, oa, range(n), "moved stream at 48 kHz, hop %d" % f)
    for c in (A, B, other):
        c.close()


def run_compaction_on_the_device_path(Context, api, mem, wav, *, n0, hops, churn, split=2, bits=64, cng_seed=7):
    """An encoder and a decoder context serve the live calls on streams 0..n-1 through encode_device / decode_plc_device.  When
    calls end, the highest live streams are copied into the holes (copy_streams) and n shrinks; an arrival is copy_streams([-1],
    [n]) and n grows.  A twin pair runs the host-buffer calls with every call on its original, sparse id; every hop's packets,
    PCM, comfort-noise flags and control states must equal the twin's.  An arrival's twin id was never used: it equals a fresh
    context.  churn: {hop: (number of calls that end, number of arrivals)}.  Original calls lose their packets for 9 hops (long
    enough for comfort noise, whose key must travel with a moved stream); arrivals lose none."""
    cap = n0 + sum(a for _, a in churn.values())
    enc, dec = Context(n0, capi=api, roles="encoder"), Context(n0, capi=api, roles="decoder")
    tenc, tdec = Context(cap, capi=api, roles="encoder"), Context(cap, capi=api, roles="decoder")
    for c in (dec, tdec):
        c.set_cng_seed(cng_seed)
    for c in (enc, dec):
        c.set_split(split)
        if mem.stream is not None:
            c.set_stream(mem.stream)
    P = (bits + 7) // 8
    d_pcm, d_pk = mem.zeros((n0, 320), np.int16), mem.zeros((n0, P), np.uint8)
    d_rec, d_out, d_cn = mem.zeros(n0, np.uint8), mem.zeros((n0, 320), np.int16), mem.zeros(n0, np.uint8)
    slot_call = list(range(n0))          # slot -> call; call c has twin id c
    next_call = n0
    rng = np.random.default_rng(5)
    seen_cn = moved_cn = False
    for f in range(hops):
        if f in churn:
            ends, arrivals = churn[f]
            n = len(slot_call)
            for h in sorted(rng.choice(n - 1, size=ends, replace=False), reverse=True):
                top = len(slot_call) - 1
                if h != top:                 # the highest live stream moves into the hole
                    enc.copy_streams([top], [h])
                    dec.copy_streams([top], [h])
                    slot_call[h] = slot_call[top]
                slot_call.pop()
            for _ in range(arrivals):
                enc.copy_streams([-1], [len(slot_call)])
                dec.copy_streams([-1], [len(slot_call)])
                slot_call.append(next_call)
                next_call += 1
        n = len(slot_call)
        calls = np.asarray(slot_call, np.int32)
        pcm = np.stack([wav[(320 * (f + 13 * c + 20)) % (len(wav) - 320):][:320] for c in calls]).copy()
        rec = np.where((calls < n0) & (calls % 3 == 0) & (f >= 1) & (f <= 9), 0, 1).astype(np.uint8)
        mem.put(d_pcm[:n], pcm)
        mem.put(d_rec[:n], rec)
        enc.encode_device(n, mem.ptr(d_pcm), bits, mem.ptr(d_pk))
        dec.decode_plc_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(d_out), mem.ptr(d_cn))
        pk = tenc.encode(pcm, bits, stream_ids=calls)
        out, cn = tdec.decode_plc(pk, bits, stream_ids=calls, received=rec)
        assert np.array_equal(mem.get(d_pk)[:n], pk), "packets after compaction differ from the sparse twin, hop %d" % f
        got_out, got_cn = mem.get(d_out)[:n], mem.get(d_cn)[:n]
        bad = np.nonzero((got_out != out).any(axis=1) | (got_cn != cn.astype(np.uint8)))[0]
        assert bad.size == 0, "decode_plc after compaction differs from the sparse twin, hop %d slots %s (calls %s)" % (
            f, bad[:8], calls[bad[:8]])
        assert np.array_equal(dec.plc_state(n), tdec.plc_state(stream_ids=calls)), "control state differs, hop %d" % f
        seen_cn |= bool(cn.any())
        moved_cn |= bool(cn[calls != np.arange(n)].any())
    assert seen_cn and moved_cn, "a moved stream must play comfort noise"
    assert next_call > n0 and len(slot_call) < n0
    for c in (enc, dec, tenc, tdec):
        c.close()


def run_round_trip_and_reset(Context, api, wav, *, max_streams=16, ids=(3, 8, 12), moved_to=(10, 1, 15), hops=9, again=2, bits=64,
                             cng_seed=9):
    """Export, run more hops, import the old records into the same ids and rerun the same hops: identical outputs.  Then the
    streams are moved to other ids and reset there: from then on they equal a fresh context's streams, comfort noise included
    (the key offset goes back to 0)."""
    ids, moved_to = np.asarray(ids, np.int32), np.asarray(moved_to, np.int32)
    rows = range(len(ids))

    def make():
        c = Context(max_streams, capi=api)
        c.set_cng_seed(cng_seed)
        return c
    ctx, fresh = make(), make()
    _history(ctx, ids, wav, hops, bits)
    recs = ctx.export_streams(ids)
    first = [_every_stateful_call(ctx, f, ids, wav, bits) for f in range(hops, hops + again)]
    ctx.import_streams(recs, ids)
    assert np.array_equal(ctx.export_streams(ids), recs), "export after import differs from the imported records"
    for i, f in enumerate(range(hops, hops + again)):
        _assert_rows_equal(_every_stateful_call(ctx, f, ids, wav, bits), first[i], rows, "rerun after import, hop %d" % f)
    ctx.import_streams(ctx.export_streams(ids), moved_to)
    ctx.reset(moved_to)          # (reset keeps lyra_b200_resample's delay lines, so the records differ; the behaviour does not)
    for f in range(hops):
        _assert_rows_equal(_every_stateful_call(ctx, f, moved_to, wav, bits), _every_stateful_call(fresh, f, moved_to, wav, bits),
                           rows, "moved stream after reset vs a fresh context, hop %d" % f)
    ctx.close()
    fresh.close()


def _resized(recs, nbytes):
    """records of another context's size cut or zero-padded to nbytes, as a caller that mixed up contexts might pass them"""
    out = np.zeros((len(recs), nbytes), np.uint8)
    m = min(nbytes, recs.shape[1])
    out[:, :m] = recs[:, :m]
    return out


def run_validation(Context, api, wav, LyraB200Error, *, max_streams=16, ids=(2, 5, 11), bits=64):
    """Every refused call returns EINVAL and changes nothing: the following export is byte-identical to the one before."""
    ids = np.asarray(ids, np.int32)
    ctx = Context(max_streams, capi=api)
    for f in range(2):
        _every_stateful_call(ctx, f, ids, wav, bits)
    good = ctx.export_streams(ids)
    before = ctx.export_streams()

    def edited(word, value, row=None):
        r = good.copy()
        w = r.view(np.uint32)
        for k in range(len(r)) if row is None else (row,):
            w[k, word] = value
        return r
    hdr = good.view(np.uint32)[0]
    enc_only = Context(max_streams, capi=api, roles="encoder")
    rate = Context(max_streams, capi=api)
    rate.set_sample_rate(8000)
    bad = {
        "magic": edited(0, hdr[0] ^ 1),
        "version": edited(1, hdr[1] + 1),
        "size": edited(2, hdr[2] + 4),
        "roles": edited(3, 1),
        "sample rate": edited(4, 48000),
        "model fingerprint": edited(6, hdr[6] ^ 0x10),
        "one bad record among good ones": edited(0, 0, row=1),
        "live flag": edited(8, 7),
    }
    for what, recs in bad.items():
        assert _fails_einval(lambda: ctx.import_streams(recs, ids), LyraB200Error), "import accepted a record with a wrong %s" % what
    for what, call in {
        "a record of an encoder-only context": lambda: ctx.import_streams(_resized(enc_only.export_streams(ids[:1]), good.shape[1]), ids[:1]),
        "a record of a context at 8 kHz": lambda: ctx.import_streams(rate.export_streams(ids[:1]), ids[:1]),
        "repeated import ids": lambda: ctx.import_streams(good[:2], [4, 4]),
        "import id out of range": lambda: ctx.import_streams(good[:2], [4, max_streams]),
        "negative import id": lambda: ctx.import_streams(good[:2], [-1, 4]),
        "export id out of range": lambda: ctx.export_streams([max_streams]),
        "copy source out of range": lambda: ctx.copy_streams([max_streams], [1]),
        "copy source below -1": lambda: ctx.copy_streams([-2], [1]),
        "copy destination -1": lambda: ctx.copy_streams([1], [-1]),
        "repeated copy source": lambda: ctx.copy_streams([2, 2], [3, 4]),
        "repeated copy destination": lambda: ctx.copy_streams([2, 5], [3, 3]),
        "copy source and destination overlap": lambda: ctx.copy_streams([2, 5], [5, 3]),
        "copy onto itself": lambda: ctx.copy_streams([6], [6]),
    }.items():
        assert _fails_einval(call, LyraB200Error), "accepted %s" % what
    assert np.array_equal(ctx.export_streams(), before), "a refused call changed a stream"
    ctx.copy_streams([-1, -1], [3, 4])                   # arrivals may share the -1 source
    assert ctx.export_streams([2], n=1).shape == (1, ctx.stream_state_bytes())
    for c in (ctx, enc_only, rate):
        c.close()
