"""How the tensor-core decoder mode's PCM differs from the exact mode's, shared by the CPU tier (emulated kernels) and the GPU tier.

The tensor mode (lyra_b200_set_decoder_mode "tensor": DecoderKernelC's split-TF32 mma.sync GEMMs of decoder_1 and DecoderKernelDW's
warpgroup MMAs) is the one decoder path that is not bit-exact.  Every layer after quant_decoder_1 is fp32 without requantisation,
so a correct fp32-accurate reordering of those sums can only move a sample across a truncation boundary of UnitToInt16: the
difference from the exact mode is 0 or +-1 LSB, rare, unbiased, and spread evenly over the kernel's structure.  A maximum alone
does not see an offset below it (a carried tail that keeps last_layer's bias is 2.66 LSB), nor rounding instead of truncation
(every sample moves by at most 1).  So each case profiles the difference, overall and per bucket of the kernel's structure:

  tail    sample index < 48 (last_layer's tail carried from the previous hop) vs >= 48, on hops whose tail is not the creation state
  phase   last_layer phase s % 16
  row     time row s // 16: rows 0-7, 8-15 and 16-19 belong to DW's three row warpgroups (16-19 next to the padding rows 160-191)
  lane    the stream's lane in its tile, slot % 8
  hop     the first hop after create, reset, import or copy vs later hops
  tile    streams of a partial last tile vs full tiles

and asserts max |d| <= TENSOR_PCM_MAX_LSB, and that the share of samples with d != 0 and |mean d| stay below TENSOR_RATE_MAX and
TENSOR_MEAN_MAX overall and in every bucket of at least MIN_BUCKET_SAMPLES samples.

The reference is an exact-mode context fed the same packets, received masks and active masks (the rest of the suite holds the
exact mode bit-exact with the oracle); on a few streams at tile and sub-batch edges the exact mode is also checked against
oracle.Codec / oracle.Decoder here, so these cases do not rest on the exact mode alone.

Measured.  H100 80GB HBM3 (SXM, 700 W power limit, 1980 MHz max SM clock), the decode and decode_plc cases of
test_gpu_tensor_accuracy.py at 4100 streams.  The tensor cores truncate while they accumulate, so each MMA folded into a large
running sum adds an error of that sum's size.  With the small split terms (a_lo*b_hi, a_hi*b_lo) in the same accumulator as
a_hi*b_hi, kernel C's decoder_1 GEMMs (K = 256: 96 MMAs per output) gave max 5 LSB and 3.7 % of the samples differing, with
phase 12 at -0.026.  Localised by running one kernel in each mode: kernel C tensor + kernel D exact gave max 5, 3.4 %; kernel C
exact + DW tensor max 1, 1.8 %.  GemmTf32Mma and DW now keep the small terms in an accumulator of their own:

  case                         samples   max |d|   d != 0   mean d     worst bucket: rate        worst bucket: mean
  decode / decode_device         31.5 M        4    2.40 %   +0.00011   phase 12  2.69 %          phase 12  -0.0156
  decode_plc                     26.2 M        2    2.55 %   +0.00005   lane 1    2.79 %          phase 12  -0.0116

Folding every k-step's a_hi*b_hi MMA into the sum with a round-to-nearest add would bring kernel C to max 3 and 2.0 %, but costs
kernel C 850 bytes of register spills per thread.  What is left is the truncation inside each MMA: the block simulator (its MMA
model reads TF32 operands like the hardware but adds each k8 step in double and rounds once) gives max 1, 1.4-2.4 % and
|mean| < 0.01 on the CPU tier's cases, so a 1-LSB bound does not hold on the hardware.  The phase pattern of the mean (about
+-0.015 LSB, smooth over the 16 phases) is there with DW alone too, and in the simulator at a smaller size.  The thresholds
below are set from the hardware numbers and still fail a carried last_layer tail that keeps its bias (mean +0.35, +2.63 on the
tail), rounding or flooring instead of truncation in UnitToInt16 (49-50 % of the samples) and a decoder_2/simple overlap tail
that keeps its bias (max over 1000), on both tiers."""
import numpy as np

from conftest import MODEL_DIR

# From the H100 numbers in the docstring:
TENSOR_PCM_MAX_LSB = 4              # |PCM_tensor - PCM_exact|: the suite's bound on the tensor mode against the oracle
TENSOR_RATE_MAX = 0.10              # share of samples with d != 0, overall and in every bucket: 3.7x the worst bucket measured
TENSOR_MEAN_MAX = 0.06              # |mean d| in LSB, overall and in every bucket: 4x the worst bucket measured
MIN_BUCKET_SAMPLES = 4000           # smaller buckets are checked for the maximum only

TILE = 8
TAIL = 48                           # last_layer's carried tail: 48 samples of the next hop
KINDS = ("speech1", "speech2", "noise", "loud", "silence")


# ---- the profile ----

def _stats(n, nz, sm, mx):
    return dict(samples=int(n), max=int(mx), rate=(nz / n) if n else 0.0, mean=(sm / n) if n else 0.0)


def error_profile(got, want, meta):
    """got, want: int16 PCM [hops, n, 320] of the tensor mode and the reference.  meta:
         slot    int [n], the stream ids (lane = slot % 8)
         first   bool [hops, n], the first hop after create, reset, import or copy
         fresh   bool [hops, n], hops whose carried tail is the creation state (create, reset); default: `first`
         partial bool [n], streams of a partial last tile
         valid   bool [hops, n], rows that ran (default: all)
    -> {bucket: {samples, max, rate, mean}} for "all" and every bucket of the module docstring."""
    d = got.astype(np.int32) - want.astype(np.int32)
    hops, n, hop_len = d.shape
    valid = np.ones((hops, n), bool) if meta.get("valid") is None else np.asarray(meta["valid"], bool)
    first = np.asarray(meta["first"], bool)
    fresh = first if meta.get("fresh") is None else np.asarray(meta["fresh"], bool)
    lane = np.asarray(meta["slot"]) % TILE
    partial = np.zeros(n, bool) if meta.get("partial") is None else np.asarray(meta["partial"], bool)
    a, nz = np.abs(d), d != 0
    out = {}

    # per row (hop, stream): samples, nonzeros, sum, max
    r_nz, r_sum, r_max = nz.sum(2), d.sum(2), a.max(2)

    def rows(name, sel):
        sel = sel & valid
        out[name] = _stats(sel.sum() * hop_len, r_nz[sel].sum(), r_sum[sel].sum(), r_max[sel].max() if sel.any() else 0)
    rows("all", np.ones((hops, n), bool))
    for ln in range(TILE):
        rows("lane %d" % ln, np.broadcast_to(lane == ln, (hops, n)))
    rows("hop first", first)
    rows("hop later", ~first)
    rows("tile partial", np.broadcast_to(partial, (hops, n)))
    rows("tile full", np.broadcast_to(~partial, (hops, n)))

    # per sample position, over the valid rows (phase, time row) and over those with a carried tail (tail)
    def positions(sel):
        m = sel[:, :, None]
        return ((np.broadcast_to(m, d.shape)).sum((0, 1)), (nz & m).sum((0, 1)), np.where(m, d, 0).sum((0, 1)),
                np.where(m, a, 0).max((0, 1)))
    p_cnt, p_nz, p_sum, p_max = positions(valid)
    s = np.arange(hop_len)

    def pos(name, sel, cnt=p_cnt, pnz=p_nz, psum=p_sum, pmax=p_max):
        out[name] = _stats(cnt[sel].sum(), pnz[sel].sum(), psum[sel].sum(), pmax[sel].max() if sel.any() else 0)
    for ph in range(16):
        pos("phase %d" % ph, s % 16 == ph)
    for r in range(hop_len // 16):
        pos("row %d" % r, s // 16 == r)
    t_cnt, t_nz, t_sum, t_max = positions(valid & ~fresh)
    pos("tail <48", s < TAIL, t_cnt, t_nz, t_sum, t_max)
    pos("tail >=48", s >= TAIL, t_cnt, t_nz, t_sum, t_max)
    return out


REGION = {"all": "whole output", "tail": "last_layer's carried tail (samples < 48 vs >= 48)", "phase": "last_layer phase s % 16",
          "row": "time row s // 16 (row warpgroups 0-7 / 8-15 / 16-19)", "lane": "stream lane slot % 8",
          "hop": "first hop after create / reset / import / copy", "tile": "partial last tile vs full tiles"}


def describe(name, st):
    return "%-13s [%s] %d samples: max |d| %d, d != 0 on %.3f%%, mean d %+.5f LSB" % (
        name, REGION[name.split()[0]], st["samples"], st["max"], 100 * st["rate"], st["mean"])


def summary(what, prof):
    """overall numbers and the worst bucket of each measure, as one line"""
    big = {k: v for k, v in prof.items() if v["samples"] >= MIN_BUCKET_SAMPLES}
    wr = max(big, key=lambda k: big[k]["rate"])
    wm = max(big, key=lambda k: abs(big[k]["mean"]))
    a = prof["all"]
    return "%s: %d samples, max |d| %d, d != 0 on %.3f%%, mean %+.5f; worst rate %s %.3f%%, worst |mean| %s %+.5f" % (
        what, a["samples"], a["max"], 100 * a["rate"], a["mean"], wr, 100 * big[wr]["rate"], wm, big[wm]["mean"])


def check_profile(what, prof):
    """every bucket within the thresholds; the failure names each offending bucket with its numbers"""
    bad = []
    for name, st in prof.items():
        if st["max"] > TENSOR_PCM_MAX_LSB:
            bad.append("max |d| %d > %d: %s" % (st["max"], TENSOR_PCM_MAX_LSB, describe(name, st)))
        if st["samples"] >= MIN_BUCKET_SAMPLES or name == "all":
            if st["rate"] > TENSOR_RATE_MAX:
                bad.append("d != 0 on more than %.1f%%: %s" % (100 * TENSOR_RATE_MAX, describe(name, st)))
            if abs(st["mean"]) > TENSOR_MEAN_MAX:
                bad.append("|mean d| > %.3f LSB: %s" % (TENSOR_MEAN_MAX, describe(name, st)))
    print(summary(what, prof))
    assert not bad, "%s, tensor mode vs exact mode, %d bucket(s) out of bounds:\n  %s" % (what, len(bad), "\n  ".join(bad[:12]))


# ---- inputs ----

def hop_input(wavs, n, f, rng):
    """hop f of streams 0..n-1: each stream cycles through speech of both wavs, 0.25 and full-scale noise and silence (four hops
    each, starting at its own kind), so every lane and tile sees every kind"""
    pcm = np.zeros((n, 320), np.int16)
    kind = (np.arange(n) + f // 4) % len(KINDS)
    for k in range(n):
        kd = KINDS[kind[k]]
        if kd.startswith("speech"):
            w = wavs[int(kd[-1]) - 1]
            pcm[k] = w[(320 * (f + 13 * k)) % (len(w) - 320):][:320]
    noise = kind == KINDS.index("noise")
    loud = kind == KINDS.index("loud")
    pcm[noise] = rng.integers(-8192, 8192, size=(int(noise.sum()), 320), dtype=np.int16)
    pcm[loud] = rng.integers(-32768, 32768, size=(int(loud.sum()), 320), dtype=np.int16)
    return pcm


def edge_streams(n, split):
    """streams at tile edges (first, last of the first tiles and of the partial last tile) and at the sub-batch edges that
    SplitParts (engine.cu) uses when a dense call of n streams is cut into `split` parts"""
    tiles = (n + TILE - 1) // TILE
    s = {0, TILE - 1, TILE, n - 1, (tiles - 1) * TILE, (tiles - 1) * TILE - 1}
    if split and split > 1 and tiles >= 64 * split:
        for i in range(1, split):
            b = (tiles * i // split) * TILE
            s |= {b - 1, b}
    return sorted(x for x in s if 0 <= x < n)


def _pair(Context, api, max_streams, split, stream, cng_seed=None):
    """(exact, tensor) decoder-only contexts with the same settings"""
    out = []
    for mode in ("exact", "tensor"):
        c = Context(max_streams, capi=api, roles="decoder")
        c.set_decoder_mode(mode)
        if split is not None:
            c.set_split(split)
        if cng_seed is not None:
            c.set_cng_seed(cng_seed)
        if stream is not None:
            c.set_stream(stream)
        out.append(c)
    return out


# ---- (a) decode and decode_device ----

def run_decode(Context, api, O, mem, wavs, *, n, hops=24, split=None, loss=0.15, seed=1):
    """Dense decode (even hops) and decode_device (odd hops) of n streams, the bit rate cycling 64 / 120 / 184, a random received
    mask (lost hops run the zero-feature path), inputs from hop_input.  n leaves a partial last tile; with `split` and enough
    tiles the calls are cut into sub-batches.  The exact mode must reach both clip values of UnitToInt16 (full-scale noise does).
    Oracle: edge_streams, exact mode bit for bit, tensor mode within TENSOR_PCM_MAX_LSB.  -> the profile."""
    assert n % TILE, "the case needs a partial last tile"
    enc = Context(n, capi=api, roles="encoder")
    E, T = _pair(Context, api, n, split, mem.stream)
    spot = edge_streams(n, split)
    codecs = {k: O.Codec(MODEL_DIR) for k in spot}
    rng = np.random.default_rng(seed)
    got, want = np.zeros((hops, n, 320), np.int16), np.zeros((hops, n, 320), np.int16)
    d_rec = mem.zeros((n,), np.uint8)
    d_outs = [mem.zeros((n, 320), np.int16) for _ in range(2)]
    lost = 0
    for f in range(hops):
        bits = (64, 120, 184)[f % 3]
        pk = enc.encode(hop_input(wavs, n, f, rng), bits)
        rec = (rng.random(n) >= loss).astype(np.uint8)
        lost += int((rec == 0).sum())
        if f % 2 == 0:
            want[f], got[f] = E.decode(pk, bits, received=rec), T.decode(pk, bits, received=rec)
        else:
            d_pk = mem.zeros(pk.shape, np.uint8)
            mem.put(d_pk, pk)
            mem.put(d_rec, rec)
            for c, o in zip((E, T), d_outs):
                c.decode_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(o))
            want[f], got[f] = mem.get(d_outs[0]), mem.get(d_outs[1])
        for k in spot:
            opcm = codecs[k].decode(bytes(pk[k]) if rec[k] else None, bits)[0]
            assert np.array_equal(want[f, k], opcm), "exact mode != oracle, hop %d stream %d" % (f, k)
            dk = int(np.abs(got[f, k].astype(int) - opcm.astype(int)).max())
            assert dk <= TENSOR_PCM_MAX_LSB, "tensor mode vs oracle, hop %d stream %d: max |d| %d" % (f, k, dk)
    assert lost, "no hop was lost"
    assert (want == 32767).any() and (want == -32768).any(), \
        "the exact mode never reached the clip values (32767: %d, -32768: %d samples)" % ((want == 32767).sum(), (want == -32768).sum())
    for c in (enc, E, T):
        c.close()
    slots = np.arange(n)
    first = np.zeros((hops, n), bool)
    first[0] = True
    return error_profile(got, want, dict(slot=slots, first=first, partial=slots >= n - n % TILE))


# ---- (b) decode_plc ----

def run_decode_plc(Context, api, O, wavs, *, n, hops=20, bits=64, cng_seed=5, seed=2):
    """decode_plc of n streams; stream k loses a burst of 2 + 10 * (k % 2) hops from hop 2 + k % 4 (the long bursts run into the
    fades and comfort noise, the short ones are concealed), so model audio passes through the fade mix both ways.
    Oracle: streams at the tile edges against oracle.Decoder.  -> the profile."""
    enc = Context(n, capi=api, roles="encoder")
    E, T = _pair(Context, api, n, None, None, cng_seed)
    spot = edge_streams(n, None)
    decs = {k: O.Decoder(MODEL_DIR, cng_seed=cng_seed + k) for k in spot}
    rng = np.random.default_rng(seed)
    got, want = np.zeros((hops, n, 320), np.int16), np.zeros((hops, n, 320), np.int16)
    k = np.arange(n)
    start, length = 2 + k % 4, 2 + 10 * (k % 2)
    seen_cn = seen_fade = False
    for f in range(hops):
        pk = enc.encode(hop_input(wavs, n, f, rng), bits)
        rec = ((f < start) | (f >= start + length)).astype(np.uint8)
        want[f], cn = E.decode_plc(pk, bits, received=rec)
        got[f], tcn = T.decode_plc(pk, bits, received=rec)
        assert np.array_equal(cn, tcn), "comfort-noise flags differ between the modes, hop %d" % f
        st = E.plc_state(n)
        seen_cn |= bool(cn.any())
        seen_fade |= bool(((st[:, 1] > 0) & (st[:, 1] < 640)).any())
        for s in spot:
            if rec[s]:
                assert decs[s].set_encoded_packet(bytes(pk[s]))
            opcm = decs[s].decode_samples(320)
            assert np.array_equal(want[f, s], opcm), "exact decode_plc != oracle, hop %d stream %d" % (f, s)
            ds = int(np.abs(got[f, s].astype(int) - opcm.astype(int)).max())
            assert ds <= TENSOR_PCM_MAX_LSB, "tensor decode_plc vs oracle, hop %d stream %d: max |d| %d" % (f, s, ds)
    assert seen_cn and seen_fade, "the bursts must reach a fade and comfort noise (fade %s, comfort noise %s)" % (seen_fade, seen_cn)
    for c in (enc, E, T):
        c.close()
    first = np.zeros((hops, n), bool)
    first[0] = True
    return error_profile(got, want, dict(slot=k, first=first, partial=k >= n - n % TILE))


# ---- (c) sparse calls and streams that sit out; (d) the hop after a stream's state was replaced ----

def sparse_ids(max_streams):
    """one stream of every tile, two of every other one (the partial last tile included), a multiple of four of them: the
    first ones are dropped"""
    ids = []
    for t in range((max_streams + TILE - 1) // TILE):
        for s in ([t % TILE] if t % 2 == 0 else [t % TILE, (t + 3) % TILE]):
            if t * TILE + s < max_streams:
                ids.append(t * TILE + s)
    return np.asarray(ids[len(ids) % 4:], np.int32)


def run_sparse_and_replaced(Context, api, wavs, *, max_streams, hops=10, bits=120, seed=3):
    """Sparse host calls over sparse_ids(max_streams) (tiles holding one or two of them), with streams' states replaced half way:
    in every group of four ids the first is reset, the second takes the third's state (copy_streams) and the fourth gets its own
    record back (exported the hop before, so it loses a hop of history).  The next hop of each of them carries a tail that is
    not the one its own history left (or the creation state): the hop a carried-tail mistake shows on.  -> the profile."""
    ids = sparse_ids(max_streams)
    n = len(ids)
    assert set(np.bincount(ids // TILE)[np.unique(ids // TILE)]) == {1, 2}, "tiles must hold one or two of the ids"
    enc = Context(max_streams, capi=api, roles="encoder")
    E, T = _pair(Context, api, max_streams, None, None)
    rng = np.random.default_rng(seed)
    got, want = np.zeros((hops, n, 320), np.int16), np.zeros((hops, n, 320), np.int16)
    first, fresh = np.zeros((hops, n), bool), np.zeros((hops, n), bool)
    first[0] = fresh[0] = True
    at = hops // 2
    recs = None
    for f in range(hops):
        if f == at - 1:
            recs = [c.export_streams(ids[3::4]) for c in (E, T)]
        if f == at:
            for c, r in zip((E, T), recs):
                c.reset(ids[0::4])
                c.copy_streams(ids[2::4], ids[1::4])
                c.import_streams(r, ids[3::4])
            first[f, 0::4] = first[f, 1::4] = first[f, 3::4] = True
            fresh[f, 0::4] = True
        pk = enc.encode(hop_input(wavs, n, f, rng), bits, stream_ids=ids)
        rec = (rng.random(n) >= 0.1).astype(np.uint8)
        want[f] = E.decode(pk, bits, stream_ids=ids, received=rec)
        got[f] = T.decode(pk, bits, stream_ids=ids, received=rec)
    for c in (enc, E, T):
        c.close()
    last = (max_streams - 1) // TILE * TILE
    return error_profile(got, want, dict(slot=ids, first=first, fresh=fresh, partial=(ids >= last) & (max_streams % TILE != 0)))


def run_sat_out_lanes(Context, api, mem, wavs, *, n, hops=8, bits=64, seed=4):
    """decode_device under an active mask that sits out every other lane, alternating between hops: the lanes that run keep the
    distribution; the rows of the streams that sit out are zero in both modes and left out of the profile.  -> the profile."""
    enc = Context(n, capi=api, roles="encoder")
    E, T = _pair(Context, api, n, None, mem.stream)
    d_mask, d_rec = mem.zeros((n,), np.uint8), mem.zeros((n,), np.uint8)
    d_pk = mem.zeros((n, (bits + 7) // 8), np.uint8)
    d_outs = [mem.zeros((n, 320), np.int16) for _ in range(2)]
    for c in (E, T):
        c.set_active_mask(mem.ptr(d_mask))
    rng = np.random.default_rng(seed)
    got, want = np.zeros((hops, n, 320), np.int16), np.zeros((hops, n, 320), np.int16)
    valid, first = np.zeros((hops, n), bool), np.zeros((hops, n), bool)
    k = np.arange(n)
    for f in range(hops):
        m = ((k + f) % 2 == 0).astype(np.uint8)
        valid[f] = m != 0
        first[f] = valid[f] & ~valid[:f].any(0)
        mem.put(d_mask, m)
        mem.put(d_pk, enc.encode(hop_input(wavs, n, f, rng), bits))
        mem.put(d_rec, (rng.random(n) >= 0.1).astype(np.uint8))
        for c, o in zip((E, T), d_outs):
            c.decode_device(n, mem.ptr(d_pk), mem.ptr(d_rec), bits, mem.ptr(o))
        want[f], got[f] = mem.get(d_outs[0]), mem.get(d_outs[1])
        assert not want[f][m == 0].any() and not got[f][m == 0].any(), "hop %d: a stream that sat out has output" % f
    for c in (E, T):
        c.set_active_mask(None)
    for c in (enc, E, T):
        c.close()
    return error_profile(got, want, dict(slot=k, first=first, valid=valid, partial=k >= n - n % TILE))
