"""Cases for lyra_b200_align_streams, shared by the CPU tier (emulated kernels) and the GPU tier (real kernels).  The bar is
bit-exactness: an aligned stream computes exactly what it computed before, and only its hop counters and the slots of its
depthwise rings change."""
import numpy as np

from stream_state_cases import _fails_einval

# Words per stream of the network entries, in the order a context registers them (A, B with the encoder role, C, D with the
# decoder role), each followed by its hop counter; a record starts with 16 header words (DESIGN.md section 4).
NET_UNITS = {"encoder": (2032, 6016), "decoder": (5888, 2032)}
HEADER_WORDS = 16
ROLES = {"both": ("encoder", "decoder"), "encoder": ("encoder",), "decoder": ("decoder",)}


def net_words(roles):
    """(first word, counter word) of every network entry of a record of a context with `roles`"""
    out, w = [], HEADER_WORDS
    for r in ROLES[roles]:
        for u in NET_UNITS[r]:
            out.append((w, w + u))
            w += u + 1
    return out


def counters(recs, roles):
    """hop counters [stream, entry] of exported records"""
    w = recs.view(np.uint32)
    return np.stack([w[:, c] for _, c in net_words(roles)], axis=1).astype(np.int64)


def _pcm(wav, f, n, hop=320):
    return np.stack([wav[(hop * (f + 11 * k + 17)) % (len(wav) - hop):][:hop] for k in range(n)]).copy()


class Traffic:
    """Hop f of the encode and decode_plc paths on streams 0..n-1, dense.  Streams 0..17 are clean: every call advances them.
    Among the others, k % 3 == 1 also runs encode_dtx on near-silent input (DTX skips its noise hops) and k % 3 == 2 loses its
    packets in bursts of 9 hops (comfort noise: pure comfort-noise hops skip the decoder).  A decoder-only context decodes
    packets drawn from a seeded generator.  hop: PCM row length (the context's rate / 50)."""

    def __init__(self, wav, n, roles, bits=64, hop=320):
        self.wav, self.n, self.roles, self.bits, self.hop = wav, n, roles, bits, hop
        k = np.arange(n)
        self.dtx = np.nonzero((k >= 18) & (k % 3 == 1))[0].astype(np.int32)
        self.lossy = (k >= 18) & (k % 3 == 2)

    def run(self, ctx, f):
        out, n, bits = {}, self.n, self.bits
        enc, dec = "encoder" in ROLES[self.roles], "decoder" in ROLES[self.roles]
        pcm = _pcm(self.wav, f, n, self.hop)
        if enc:
            if self.dtx.size:
                quiet = pcm[self.dtx] // 256
                out["dtx_packets"], out["dtx_bytes"] = ctx.encode_dtx(quiet, bits, stream_ids=self.dtx)
            pk = ctx.encode(pcm, bits)
            out["packets"] = pk
        else:
            pk = np.random.default_rng(300 + f).integers(0, 256, size=(n, (bits + 7) // 8), dtype=np.uint8)
        if dec:
            lost = self.lossy & (f >= 1) & ((f + np.arange(n)) % 14 < 9)
            out["plc_pcm"], out["comfort_noise"] = ctx.decode_plc(pk, bits, received=(~lost).astype(np.uint8))
            out["plc_state"] = ctx.plc_state(n)
        return out


def _assert_same(got, want, what):
    for name, rows in want.items():
        bad = np.nonzero(np.asarray(got[name] != rows).reshape(len(rows), -1).any(axis=1))[0]
        assert bad.size == 0, "%s: %s differs at streams %s" % (what, name, bad[:8])


def staggered_history(ctxs, traffic, hops):
    """`hops` hops of traffic on every context; before hop r (1..17) the streams k with k % 18 == r are reset, so the clean
    streams end on 18 different hop counters in every network entry.  Returns whether comfort noise and DTX were reached."""
    n = traffic.n
    seen_cn = seen_dtx = False
    for f in range(hops):
        if 1 <= f < 18:
            ids = np.arange(f, n, 18, dtype=np.int32)
            for c in ctxs:
                c.reset(ids)
        for c in ctxs:
            o = traffic.run(c, f)
        seen_cn |= bool(o.get("comfort_noise", np.zeros(1, bool)).any())
        seen_dtx |= bool((o.get("dtx_bytes", np.ones(1)) == 0).any())
    return seen_cn, seen_dtx


def run_continuation(Context, api, wav, *, n=24, roles="both", mode="exact", split=None, hops=20, after=20, like=0, bits=64,
                     cng_seed=3, setup=None, hop=320):
    """Two contexts run the same staggered history (lanes on every counter residue 0..17 in every entry); one aligns every
    stream like stream `like` in one call (more than 1024 ids at full size: several launches), then both run `after` more hops:
    every packet, PCM hop, comfort-noise flag and control state is bit-identical.  setup(ctx) configures both contexts (rates,
    bits)."""
    def make():
        c = Context(n, capi=api, roles=roles)
        c.set_cng_seed(cng_seed)
        if "decoder" in ROLES[roles]:
            c.set_decoder_mode(mode)
        if split:
            c.set_split(split)
        if setup:
            setup(c)
        return c
    A, twin = make(), make()
    traffic = Traffic(wav, n, roles, bits, hop)
    seen_cn, seen_dtx = staggered_history((A, twin), traffic, hops)
    before = counters(A.export_streams(), roles)
    assert np.array_equal(before, counters(twin.export_streams(), roles))
    for e in range(before.shape[1]):
        assert set(before[:18, e]) == set(range(18)), "entry %d: the clean streams must sit at every counter residue" % e
    ids = np.asarray([k for k in range(n) if k != like], np.int32)
    A.align_streams(ids, np.full(ids.size, like, np.int32))
    got = counters(A.export_streams(), roles)
    assert (got == before[like]).all(), "after the align every stream has stream %d's counters" % like
    for f in range(hops, hops + after):
        oa, ot = traffic.run(A, f), traffic.run(twin, f)
        _assert_same(oa, ot, "aligned vs unaligned twin, hop %d" % f)
        seen_cn |= bool(ot.get("comfort_noise", np.zeros(1, bool)).any())
        seen_dtx |= bool((ot.get("dtx_bytes", np.ones(1)) == 0).any())
    if "decoder" in ROLES[roles] and n > 18:
        assert seen_cn, "the traffic must reach comfort noise"
    if "encoder" in ROLES[roles] and n > 18:
        assert seen_dtx, "the traffic must reach DTX"
    A.close()
    twin.close()


def run_records(Context, api, wav, *, n=24, hops=19, bits=64, x=3, y=7, spare=20):
    """What align writes, read from exported records: the listed stream's counters become its like stream's, every word
    outside the network entries stays, aligning to equal counters changes nothing, and aligning back (like a spare stream
    parked at the original counters) restores the record byte for byte, after a like stream and after like = -1."""
    ctx = Context(n, capi=api)
    traffic = Traffic(wav, n, "both", bits)
    staggered_history((ctx,), traffic, hops)
    words = net_words("both")
    outside = np.ones(ctx.stream_state_bytes() // 4, bool)
    outside[words[0][0]:words[-1][1] + 1] = False
    r0 = ctx.export_streams()
    c0 = counters(r0, "both")
    assert (c0[x] != c0[y]).all() and (c0[x] != 0).all()
    ctx.align_streams([spare], [x])                   # park a spare stream at x's counters
    r0 = ctx.export_streams()
    assert np.array_equal(counters(r0, "both")[spare], c0[x])
    ctx.align_streams([x], [spare])
    assert np.array_equal(ctx.export_streams(), r0), "aligning to a stream at the same counters changed a record"
    for like in (y, -1):
        ctx.align_streams([x], [like])
        r1 = ctx.export_streams()
        assert np.array_equal(counters(r1, "both")[x], c0[like] if like >= 0 else np.zeros(len(words))), "x like %d" % like
        assert np.array_equal(r1.view(np.uint32)[:, outside], r0.view(np.uint32)[:, outside]), "a word outside the networks changed"
        assert np.array_equal(np.delete(r1, x, axis=0), np.delete(r0, x, axis=0)), "a stream that was not listed changed"
        assert not np.array_equal(r1[x], r0[x])
        ctx.align_streams([x], [spare])
        assert np.array_equal(ctx.export_streams(), r0), "aligning back after like %d did not restore the record" % like
    ctx.close()


def run_realign_after_skips(Context, api, wav, *, n=16, hops=20, after=20, bits=64, dtx=(3, 12), lossy=(5, 9)):
    """Streams that sat out hops fall behind their tile: DTX streams skip their noise hops in the encoder, streams in pure comfort
    noise skip the decoder.  After the history their counters differ from their neighbours'; every lane of each tile is aligned
    like its lane 0 and the streams continue bit for bit against a twin that was not aligned."""
    def make():
        c = Context(n, capi=api)
        c.set_cng_seed(11)
        return c
    A, twin = make(), make()
    traffic = Traffic(wav, n, "both", bits)
    traffic.dtx = np.asarray(dtx, np.int32)
    traffic.lossy = np.isin(np.arange(n), lossy)
    skipped = np.zeros(len(dtx), int)
    in_cn = np.zeros(n, bool)
    for f in range(hops):
        for c in (A, twin):
            o = traffic.run(c, f)
        skipped += o["dtx_bytes"] == 0
        in_cn |= o["comfort_noise"]
    assert skipped.any() and in_cn[list(lossy)].all(), "a DTX stream must skip hops (%s), every lossy one reach comfort noise" % skipped
    c0 = counters(A.export_streams(), "both")
    for t in {s - s % 8 for s in dtx + lossy}:
        assert (c0[t:t + 8] != c0[t]).any(), "tile %d is not mixed before the align" % (t // 8)
    ids = np.asarray([k for k in range(n) if k % 8], np.int32)
    A.align_streams(ids, ids - ids % 8)
    got = counters(A.export_streams(), "both")
    assert (got == got[np.arange(n) - np.arange(n) % 8]).all(), "every tile on one counter per entry"
    for f in range(hops, hops + after):
        _assert_same(traffic.run(A, f), traffic.run(twin, f), "realigned vs twin, hop %d" % f)
    A.close()
    twin.close()


def _tile_counters_agree(ctx, roles, n):
    c = counters(ctx.export_streams(n=n), roles)
    for t in range(0, n, 8):
        rows = c[t:min(t + 8, n)]
        if not (rows == rows[0]).all():
            return t
    return None


def run_compaction_with_alignment(Context, api, mem, wav, *, n0, hops, churn, split=2, bits=64, cng_seed=7):
    """The churn loop of stream_state_cases.run_compaction_on_the_device_path with an align after every copy: an encoder and a
    decoder context serve the live calls on streams 0..n-1 through encode_device / decode_plc_device; an ended call's hole takes
    the highest live stream (copy_streams) and an arrival starts from -1, and each moved or admitted stream is then aligned like
    a live neighbour of its tile; at the end of a churn step every tile is aligned like its first lane (streams in comfort noise
    fall behind).  No host synchronisation between copies, aligns and device calls.  Every hop equals a twin pair that runs the
    host-buffer calls on the original, sparse ids, and after every churn step each tile's live lanes share one counter per
    entry."""
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
    slot_call = list(range(n0))
    next_call = n0
    rng = np.random.default_rng(5)
    seen_cn = moved_cn = False

    def align_like_neighbour(h, n):
        t0 = h - h % 8
        like = next((k for k in range(t0, min(t0 + 8, n)) if k != h), None)
        if like is not None:
            for c in (enc, dec):
                c.align_streams([h], [like])
    for f in range(hops):
        if f in churn:
            ends, arrivals = churn[f]
            for h in sorted(rng.choice(len(slot_call) - 1, size=ends, replace=False), reverse=True):
                top = len(slot_call) - 1
                if h != top:
                    enc.copy_streams([top], [h])
                    dec.copy_streams([top], [h])
                    slot_call[h] = slot_call[top]
                slot_call.pop()
                if h < len(slot_call):
                    align_like_neighbour(h, len(slot_call))
            for _ in range(arrivals):
                s = len(slot_call)
                enc.copy_streams([-1], [s])
                dec.copy_streams([-1], [s])
                slot_call.append(next_call)
                next_call += 1
                align_like_neighbour(s, len(slot_call))
            n = len(slot_call)
            ids = np.asarray([k for k in range(n) if k % 8], np.int32)
            for c in (enc, dec):
                c.align_streams(ids, ids - ids % 8)
            for c, roles in ((enc, "encoder"), (dec, "decoder")):
                bad = _tile_counters_agree(c, roles, n)
                assert bad is None, "hop %d: the live lanes of tile %d do not share one %s counter" % (f, bad // 8, roles)
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
        assert np.array_equal(mem.get(d_pk)[:n], pk), "packets after compaction and alignment differ from the sparse twin, hop %d" % f
        got_out, got_cn = mem.get(d_out)[:n], mem.get(d_cn)[:n]
        bad = np.nonzero((got_out != out).any(axis=1) | (got_cn != cn.astype(np.uint8)))[0]
        assert bad.size == 0, "decode_plc after compaction and alignment differs from the sparse twin, hop %d slots %s" % (f, bad[:8])
        assert np.array_equal(dec.plc_state(n), tdec.plc_state(stream_ids=calls)), "control state differs, hop %d" % f
        seen_cn |= bool(cn.any())
        moved_cn |= bool(cn[calls != np.arange(n)].any())
    assert seen_cn and moved_cn, "a moved stream must play comfort noise"
    assert next_call > n0 and len(slot_call) < n0
    for c in (enc, dec, tenc, tdec):
        c.close()


def run_validation(Context, api, wav, LyraB200Error, *, max_streams=16, ids=(2, 5, 11), bits=64):
    """Every refused align returns EINVAL and changes nothing: the following export is byte-identical to the one before.
    Repeated like ids are accepted, and n == 0 does nothing."""
    import ctypes as C
    ids = np.asarray(ids, np.int32)
    ctx = Context(max_streams, capi=api)
    for f in range(3):
        ctx.reset(ids[f:f + 1])
        ctx.encode(_pcm(wav, f, max_streams), bits)
    before = ctx.export_streams()
    assert len({tuple(r) for r in counters(before, "both")[ids]}) == len(ids)
    lib, h = api.lib, ctx.h
    one = np.asarray([3], np.int32)
    for what, call in {
        "an id out of range": lambda: ctx.align_streams([max_streams], [1]),
        "a negative id": lambda: ctx.align_streams([-1], [1]),
        "a like id out of range": lambda: ctx.align_streams([1], [max_streams]),
        "a like id below -1": lambda: ctx.align_streams([1], [-2]),
        "a repeated id": lambda: ctx.align_streams([2, 2], [5, 11]),
        "an id in both lists": lambda: ctx.align_streams([2, 5], [5, 11]),
        "a stream aligned like itself": lambda: ctx.align_streams([6], [6]),
        "a bad id after good ones": lambda: ctx.align_streams([2, 3, max_streams], [5, 5, 5]),
    }.items():
        assert _fails_einval(call, LyraB200Error), "accepted %s" % what
    for what, args in {"NULL stream_ids": (None, one.ctypes.data_as(C.c_void_p), 1),
                       "NULL like_ids": (one.ctypes.data_as(C.c_void_p), None, 1),
                       "a negative count": (one.ctypes.data_as(C.c_void_p), one.ctypes.data_as(C.c_void_p), -1)}.items():
        assert lib.lyra_b200_align_streams(h, *args) == -1, "accepted %s" % what
    assert lib.lyra_b200_align_streams(None, None, None, 0) == -1
    assert np.array_equal(ctx.export_streams(), before), "a refused align changed a stream"
    assert lib.lyra_b200_align_streams(h, None, None, 0) == 0, "n == 0 must succeed"
    ctx.align_streams([], [])
    assert np.array_equal(ctx.export_streams(), before), "n == 0 changed a stream"
    ctx.align_streams([2, 11, 7], [5, 5, 5])            # repeated like ids
    c = counters(ctx.export_streams(), "both")
    assert (c[[2, 11, 7]] == c[5]).all()
    ctx.close()
