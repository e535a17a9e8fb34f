"""Cases for the fused codec calls at an external sample rate (lyra_b200_set_sample_rate), shared by the CPU tier (emulated kernels)
and the GPU tier.  The oracle for rate R is a composition of existing oracle objects, as LyraEncoder / LyraDecoder compose them
(lyra/lyra_encoder.cc:58-66,80-89,118-141, lyra/lyra_decoder.cc:108-114):
  encode: Resampler(R, 16000) -> (DTX: NoiseEstimator(R, 320, 640, 160) fed the 16 kHz hop) -> the 16 kHz encoder;
  decode: the 16 kHz decoder -> BufferedResampler(16000, R).filter_and_buffer(..., R // 50), whose leftover stays 0.
Bar: bit-exact packets, flags, control state and PCM; decoded PCM within TENSOR_PCM_TOL_LSB in the tensor decoder mode."""
import numpy as np

from conftest import MODEL_DIR
from parity_cases import TENSOR_PCM_TOL_LSB, Guarded


RATES = (8000, 32000, 48000)


def hop_of(rate):
    return rate // 50


class OracleEncoder:
    """LyraEncoder::Create(rate, ..., enable_dtx) from oracle pieces.  est_rate: the rate the DTX estimator is built for (the
    reference uses the external rate; another value builds the composition a test must be able to tell apart)."""

    def __init__(self, O, rate, dtx=False, est_rate=None):
        self.rs = O.Resampler(rate, 16000) if rate != 16000 else None
        self.est = O.NoiseEstimator(est_rate or rate, 320, 640, 160) if dtx else None
        self.enc = O.Encoder(MODEL_DIR)

    def encode(self, pcm, bits):
        x = self.rs.resample(pcm) if self.rs is not None else np.asarray(pcm, np.int16)
        assert len(x) == 320, "the resampler must deliver whole 16 kHz hops"
        if self.est is not None:
            self.est.receive_samples(x)
            if self.est.is_noise:
                return b""
        return self.enc.encode(x, bits)


class OracleUp:
    """The decoder's 16 kHz -> rate conversion (BufferedResampler), one whole hop at a time."""

    def __init__(self, O, rate):
        self.rate = rate
        self.br = O.BufferedResampler(16000, rate) if rate != 16000 else None

    def __call__(self, pcm16):
        if self.br is None:
            return pcm16
        out = self.br.filter_and_buffer(lambda k: pcm16 if k == 320 else None, hop_of(self.rate))
        assert out is not None and self.br.leftover == 0
        return out


class OracleCodec:
    """Encoder + plain decoder (lyra_b200_encode / lyra_b200_decode: zero features for a lost packet) of one stream at `rate`;
    with track=True also the decoder-side 16 kHz noise estimator fed the decoded hops of received packets."""

    def __init__(self, O, rate, track=False):
        self.rs = O.Resampler(rate, 16000) if rate != 16000 else None
        self.codec = O.Codec(MODEL_DIR)
        self.up = OracleUp(O, rate)
        self.est = O.NoiseEstimator() if track else None

    def encode(self, pcm, bits):
        x = self.rs.resample(pcm) if self.rs is not None else np.asarray(pcm, np.int16)
        assert len(x) == 320
        return self.codec.encode(x, bits)[0]

    def decode(self, packet, bits):
        pcm16 = self.codec.decode(packet, bits)[0]
        if self.est is not None and packet is not None:
            self.est.receive_samples(pcm16)
        return self.up(pcm16)

    def set_rate(self, O, rate):
        """lyra_b200_set_sample_rate: fresh converters, the codec state carries on."""
        self.rs = O.Resampler(rate, 16000) if rate != 16000 else None
        self.up = OracleUp(O, rate)


class OraclePlcDecoder:
    def __init__(self, O, rate, cng_seed):
        self.dec = O.Decoder(MODEL_DIR, cng_seed=cng_seed)
        self.up = OracleUp(O, rate)

    def tick(self, packet):
        if packet is not None:
            assert self.dec.set_encoded_packet(packet)
        return self.up(self.dec.decode_samples(320))


def speech_rows(wav, rate, ids, f, stride=7, base=20):
    hop = hop_of(rate)
    return np.stack([wav[(hop * (f + stride * int(k) + base)) % (len(wav) - hop):][:hop] for k in ids]).copy()


def _pcm_diff(a, b):
    return int(np.abs(np.asarray(a, int) - np.asarray(b, int)).max())


def run_rate_parity(Context, api, O, wav, *, rate, max_streams, stream_ids=None, n=None, frames=12, check=None, decoder_mode="exact",
                    calls=("track", "plc", "dtx"), split=None, cng_seed=7, seed=1):
    """Every fused call at `rate` hop by hop against the oracle composition.  stream_ids None = dense streams 0..n-1.  Inputs: speech,
    with every third stream silent in the second half (so DTX and the estimators' noise branch run).  decode / decode_track_noise get
    random loss masks; decode_plc gets bursts of 7 lost hops (concealment -> comfort noise -> fade back) on even streams and of 2 on
    odd ones; the bit rate changes every fourth hop.  Between hops the codec context also runs lyra_b200_resample on the same
    streams with ragged chunks: that plugin's converters are not the codec's, so the codec hops must not notice."""
    ids = np.arange(n, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    sparse = stream_ids is not None
    call_ids = ids if sparse else None
    check = list(range(n)) if check is None else list(check)
    tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    exact = decoder_mode == "exact"
    ctx = {k: Context(max_streams, capi=api) for k in ("codec",) + tuple(calls)}
    for c in ctx.values():
        c.set_sample_rate(rate)
        c.set_decoder_mode(decoder_mode)
        c.set_cng_seed(cng_seed)
        if split is not None:
            c.set_split(split)
    codec = {k: OracleCodec(O, rate) for k in check}
    track = {k: OracleCodec(O, rate, track=True) for k in check}
    plc = {k: OraclePlcDecoder(O, rate, cng_seed + int(ids[k])) for k in check}
    dtx = {k: OracleEncoder(O, rate, dtx=True) for k in check}
    rng = np.random.default_rng(seed)
    burst = [(1 + k % 3, 7 if k % 2 == 0 else 2) for k in range(n)]
    seen = dict(cn=False, dtx=set(), loss=False)
    hop = hop_of(rate)
    for f in range(frames):
        bits = (64, 120, 184)[(f // 4) % 3]
        pcm = speech_rows(wav, rate, ids, f)
        if f >= frames // 2:
            pcm[::3] = 0
        c = ctx["codec"]                    # its packets feed the other decoders
        pk = c.encode(pcm, bits, stream_ids=call_ids)
        rec = (rng.random(n) >= 0.3).astype(np.uint8)
        out = c.decode(pk, bits, stream_ids=call_ids, received=rec)
        assert out.shape == (n, hop)
        chunk = (7, hop - 3, 1)[f % 3]
        c.resample(rng.integers(-9000, 9000, size=(n, chunk)).astype(np.int16), rate, True, stream_ids=ids)
        c.resample(rng.integers(-9000, 9000, size=(n, 13 + f)).astype(np.int16), rate, False, stream_ids=ids)
        for k in check:
            opkt = codec[k].encode(pcm[k], bits)
            assert bytes(pk[k]) == opkt, "encode at %d Hz != oracle, hop %d stream %d" % (rate, f, ids[k])
            want = codec[k].decode(opkt if rec[k] else None, bits)
            d = _pcm_diff(out[k], want)
            assert d <= tol, "decode at %d Hz != oracle, hop %d stream %d: max |d| %d" % (rate, f, ids[k], d)
            seen["loss"] |= not rec[k]
        if "track" in ctx:
            rec = (rng.random(n) >= 0.25).astype(np.uint8)
            out, flags = ctx["track"].decode_track_noise(pk, bits, stream_ids=call_ids, received=rec)
            for k in check:
                want = track[k].decode(bytes(pk[k]) if rec[k] else None, bits)
                d = _pcm_diff(out[k], want)
                assert d <= tol, "decode_track_noise at %d Hz != oracle, hop %d stream %d: max |d| %d" % (rate, f, ids[k], d)
                if exact:
                    assert bool(flags[k]) == track[k].est.is_noise, "track is_noise != oracle, hop %d stream %d" % (f, ids[k])
        if "plc" in ctx:
            rec = np.array([0 if b0 <= f < b0 + bl else 1 for b0, bl in burst], dtype=np.uint8)
            out, cn = ctx["plc"].decode_plc(pk, bits, stream_ids=call_ids, received=rec)
            st = ctx["plc"].plc_state(stream_ids=ids)
            for k in check:
                want = plc[k].tick(bytes(pk[k]) if rec[k] else None)
                d = _pcm_diff(out[k], want)
                assert d <= tol, "decode_plc at %d Hz != oracle, hop %d stream %d: max |d| %d" % (rate, f, ids[k], d)
                assert tuple(int(x) for x in st[k]) == plc[k].dec.state and bool(cn[k]) == plc[k].dec.is_comfort_noise(), (f, k)
                seen["cn"] |= bool(cn[k])
        if "dtx" in ctx:
            xpk, sizes = ctx["dtx"].encode_dtx(pcm, bits, stream_ids=call_ids)
            for k in check:
                want = dtx[k].encode(pcm[k], bits)
                assert sizes[k] == len(want) and bytes(xpk[k][:sizes[k]]) == want, "encode_dtx at %d Hz != oracle, hop %d stream %d" % (
                    rate, f, ids[k])
                if sizes[k] == 0:
                    assert not xpk[k].any()
                seen["dtx"].add(int(sizes[k] == 0))
    assert seen["loss"]
    if "plc" in ctx:
        assert seen["cn"], "the case never reached comfort noise"
    if "dtx" in ctx:
        assert seen["dtx"] == {0, 1}, "the case must produce both DTX and encoded hops"
    for c in ctx.values():
        c.close()


def run_equivalence_with_plugin_chain(Context, api, *, rate, max_streams=16, stream_ids=(2, 9, 10), frames=3, bits=64, seed=3):
    """encode at `rate` == resample(rate -> 16k) + encode at 16 kHz on a twin context, decode at `rate` == decode + resample(16k -> rate),
    bit for bit; and set_sample_rate(16000) on a fresh context == never calling the setter, launch counts included."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    a, b = Context(max_streams, capi=api), Context(max_streams, capi=api)
    a.set_sample_rate(rate)
    assert a.sample_rate == rate and b.sample_rate == 16000
    rng = np.random.default_rng(seed)
    for f in range(frames):
        x = rng.integers(-12000, 12000, size=(n, hop_of(rate))).astype(np.int16)
        pk = a.encode(x, bits, stream_ids=ids)
        x16 = np.stack(b.resample(x, rate, True, stream_ids=ids))
        assert x16.shape == (n, 320)
        assert np.array_equal(pk, b.encode(x16, bits, stream_ids=ids)), "encode at %d Hz != resample + encode, hop %d" % (rate, f)
        out = a.decode(pk, bits, stream_ids=ids)
        want = np.stack(b.resample(b.decode(pk, bits, stream_ids=ids), rate, False, stream_ids=ids))
        assert np.array_equal(out, want), "decode at %d Hz != decode + resample, hop %d" % (rate, f)
    a.close()
    b.close()
    # 16 kHz: no conversion and no extra launch, whether or not the setter was called
    c, d = Context(max_streams, capi=api), Context(max_streams, capi=api)
    c.set_sample_rate(16000)
    for f in range(2):
        x = rng.integers(-12000, 12000, size=(n, 320)).astype(np.int16)
        pc_, pd_ = c.encode(x, bits, stream_ids=ids), d.encode(x, bits, stream_ids=ids)
        assert np.array_equal(pc_, pd_)
        assert np.array_equal(c.decode(pc_, bits), d.decode(pd_, bits))
        assert np.array_equal(c.encode_dtx(x, bits)[1], d.encode_dtx(x, bits)[1])
        assert np.array_equal(c.decode_plc(pc_, bits, stream_ids=ids)[0], d.decode_plc(pd_, bits, stream_ids=ids)[0])
    assert c.launch_count == d.launch_count, (c.launch_count, d.launch_count)
    c.close()
    d.close()


def run_device_twins(Context, api, mem, wav, *, rate, n, frames, decoder_mode="exact", split=None, cng_seed=5, seed=4):
    """Every *_device codec call at `rate` against its host-buffer twin, all n streams, with caller buffers of external-rate rows
    guarded on both sides (Guarded): a call that touches a row outside [0, n) or leaves an output row unwritten fails.  The device
    contexts run on mem.stream when there is one."""
    hop = hop_of(rate)
    roles = dict(enc="encoder", dec="decoder", trk="decoder", plc="decoder", dtx="encoder")
    dev = {k: Context(n, capi=api, roles=r) for k, r in roles.items()}
    host = {k: Context(n, capi=api, roles=r) for k, r in roles.items()}
    for c in list(dev.values()) + list(host.values()):
        c.set_sample_rate(rate)
        c.set_decoder_mode(decoder_mode)
        c.set_cng_seed(cng_seed)
    for c in dev.values():
        if split is not None:
            c.set_split(split)
        if mem.stream is not None:
            c.set_stream(mem.stream)
    G = lambda row, dtype, s: Guarded(mem, n, row, dtype, s)     # noqa: E731
    d_pcm = G((hop,), np.int16, 0x3C)
    d_rec, d_plc_rec = G((), np.uint8, 0xC3), G((), np.uint8, 0xC3)
    d_out, d_trk, d_plc = G((hop,), np.int16, 0x5A), G((hop,), np.int16, 0x5A), G((hop,), np.int16, 0x5A)
    d_trk_flags, d_cn, d_dtx_flags = (G((), np.uint8, 0xAA) for _ in range(3))
    rng = np.random.default_rng(seed)
    ks = np.arange(n)
    for f in range(frames):
        bits = (64, 184, 120)[f % 3]
        P = (bits + 7) // 8
        pcm = speech_rows(wav, rate, ks, f, stride=13)
        pcm[(ks % 3 == 1) & (f < frames // 2)] = 0
        d_pcm.put(pcm)
        d_pk, d_dtx_pk = G((P,), np.uint8, 0xA5), G((P,), np.uint8, 0xFF)
        for buf in (d_out, d_trk, d_plc, d_trk_flags, d_cn, d_dtx_flags):
            buf.fill()
        rec = (rng.random(n) >= 0.25).astype(np.uint8) if f % 2 else None
        if rec is not None:
            d_rec.put(rec)
        plc_rec = np.array([0 if 1 <= f < 1 + (6 if k % 2 else 2) else 1 for k in range(n)], dtype=np.uint8)
        d_plc_rec.put(plc_rec)
        dev["enc"].encode_device(n, d_pcm.ptr, bits, d_pk.ptr)
        dev["dec"].decode_device(n, d_pk.ptr, d_rec.ptr if rec is not None else 0, bits, d_out.ptr)
        dev["trk"].decode_track_noise_device(n, d_pk.ptr, d_rec.ptr if rec is not None else 0, bits, d_trk.ptr, d_trk_flags.ptr)
        dev["plc"].decode_plc_device(n, d_pk.ptr, d_plc_rec.ptr, bits, d_plc.ptr, d_cn.ptr)
        dev["dtx"].encode_dtx_device(n, d_pcm.ptr, bits, d_dtx_pk.ptr, d_dtx_flags.ptr)
        pk = host["enc"].encode(pcm, bits)
        assert np.array_equal(d_pk.get("packets"), pk), "encode_device != encode at %d Hz, hop %d" % (rate, f)
        assert np.array_equal(d_out.get("PCM"), host["dec"].decode(pk, bits, received=rec)), "decode_device != decode, hop %d" % f
        t_out, t_flags = host["trk"].decode_track_noise(pk, bits, received=rec)
        assert np.array_equal(d_trk.get("PCM"), t_out) and np.array_equal(d_trk_flags.get("flags"), t_flags.astype(np.uint8)), f
        p_out, p_cn = host["plc"].decode_plc(pk, bits, received=plc_rec)
        assert np.array_equal(d_plc.get("PCM"), p_out), "decode_plc_device != decode_plc at %d Hz, hop %d" % (rate, f)
        assert np.array_equal(d_cn.get("flags"), p_cn.astype(np.uint8)), f
        x_pk, x_sizes = host["dtx"].encode_dtx(pcm, bits)
        assert np.array_equal(d_dtx_flags.get("flags"), (x_sizes == 0).astype(np.uint8)), "encode_dtx_device flags, hop %d" % f
        assert np.array_equal(d_dtx_pk.get("packets"), x_pk), "encode_dtx_device packets, hop %d" % f
        d_pcm.get("input PCM")
    for c in list(dev.values()) + list(host.values()):
        c.close()


def run_dtx_at_rate(Context, api, O, wav, *, rate, speech_hops=10, noise_hops=20, bits=64, stream_ids=(1, 6), level=12, seed=5):
    """encode_dtx at `rate` over speech followed by low-level noise: the per-hop packet sizes equal the oracle composition whose DTX
    estimator is built for `rate`, as the reference builds it.  The same composition with a 16 kHz estimator gives a different
    sequence, so the case tells the two apart."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n, hop = len(ids), hop_of(rate)
    ctx = Context(int(ids.max()) + 1, capi=api)
    ctx.set_sample_rate(rate)
    want = {k: OracleEncoder(O, rate, dtx=True) for k in range(n)}
    other = {k: OracleEncoder(O, rate, dtx=True, est_rate=16000) for k in range(n)}
    rng = np.random.default_rng(seed)
    got_sizes, other_sizes = [], []
    for f in range(speech_hops + noise_hops):
        if f < speech_hops:
            pcm = speech_rows(wav, rate, range(n), f, stride=11, base=30)
        else:
            pcm = rng.integers(-level, level + 1, size=(n, hop)).astype(np.int16)
        pk, sizes = ctx.encode_dtx(pcm, bits, stream_ids=ids)
        for k in range(n):
            w = want[k].encode(pcm[k], bits)
            assert sizes[k] == len(w) and bytes(pk[k][:sizes[k]]) == w, "encode_dtx at %d Hz, hop %d stream %d: %d bytes, oracle %d" % (
                rate, f, ids[k], sizes[k], len(w))
            other_sizes.append(len(other[k].encode(pcm[k], bits)))
        got_sizes += [int(s) for s in sizes]
    assert 0 in got_sizes and max(got_sizes) > 0, "the case must produce both DTX and encoded hops"
    assert got_sizes != other_sizes, "a 16 kHz DTX estimator would pass this case too"
    ctx.close()
    return got_sizes


def run_rate_change_and_reset(Context, api, O, wav, LyraB200Error, *, rates=(48000, 8000), max_streams=16, stream_ids=(1, 3, 9), hops=3,
                              bits=64):
    """set_sample_rate(R2) between hops: the next hop equals the oracle with fresh converters and the codec state carried on.  Then
    lyra_b200_reset of one stream: it equals a fresh context at R2, its tile neighbours equal a twin that was not reset.  Unsupported
    rates return EINVAL and leave the setting unchanged."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    r1, r2 = rates
    ctx, twin = Context(max_streams, capi=api), Context(max_streams, capi=api)
    for c in (ctx, twin):
        c.set_sample_rate(r1)
    ref = {k: OracleCodec(O, r1) for k in range(n)}

    def hop(c, r, f):
        x = speech_rows(wav[r], r, range(n), f, stride=5)
        pk = c.encode(x, bits, stream_ids=ids)
        return x, pk, c.decode(pk, bits, stream_ids=ids)

    for f in range(hops):
        for c in (ctx, twin):
            x, pk, out = hop(c, r1, f)
        for k in range(n):
            assert bytes(pk[k]) == ref[k].encode(x[k], bits) and np.array_equal(out[k], ref[k].decode(bytes(pk[k]), bits)), (f, k)
    for c in (ctx, twin):
        c.set_sample_rate(r2)
    for k in range(n):
        ref[k].set_rate(O, r2)
    for f in range(hops, hops + 2):
        for c in (ctx, twin):
            x, pk, out = hop(c, r2, f)
        for k in range(n):
            assert bytes(pk[k]) == ref[k].encode(x[k], bits), "encode after a rate change, hop %d stream %d" % (f, ids[k])
            assert np.array_equal(out[k], ref[k].decode(bytes(pk[k]), bits)), "decode after a rate change, hop %d stream %d" % (f, ids[k])
    # reset of stream ids[0]: a fresh context's first hop; ids[1] (same tile) and ids[2] carry on like the twin
    ctx.reset(stream_ids=ids[:1])
    fresh = Context(max_streams, capi=api)
    fresh.set_sample_rate(r2)
    f = hops + 2
    x, pk, out = hop(ctx, r2, f)
    _, fpk, fout = hop(fresh, r2, f)
    _, tpk, tout = hop(twin, r2, f)
    assert bytes(pk[0]) == bytes(fpk[0]) and np.array_equal(out[0], fout[0]), "a reset stream must equal a fresh context"
    assert np.array_equal(pk[1:], tpk[1:]) and np.array_equal(out[1:], tout[1:]), "reset changed a stream that was not listed"
    assert not np.array_equal(out[0], tout[0]), "the reset must make a difference here"
    for bad in (44100, 0, -1, 16001):
        try:
            ctx.set_sample_rate(bad)
            raise AssertionError("rate %d accepted" % bad)
        except LyraB200Error as e:
            assert e.code == -1
        assert ctx.sample_rate == r2
    for c in (ctx, twin, fresh):
        c.close()


def run_integration_at_rate(Context, api, O, *, rate, wav, bits=64, hops=60, skip=3):
    """lyra_integration_test.cc:60-149 at an external rate through the rate-aware calls: one encode and one decode call per hop, the
    64-bin log-mel spectra (at the external rate) of input and output within LSD 2.0 on every hop after the priming hops."""
    hop = hop_of(rate)
    ctx = Context(4, capi=api)
    ctx.set_sample_rate(rate)
    ie, oe = O.LogMel(rate, hop, 2 * hop, 64), O.LogMel(rate, hop, 2 * hop, 64)
    worst = 0.0
    for f in range(hops):
        x = wav[f * hop:(f + 1) * hop]
        y = ctx.decode(ctx.encode(x, bits, stream_ids=[2]), bits, stream_ids=[2])[0]
        assert len(y) == hop
        fi, fo = ie.extract(x), oe.extract(y)
        if f >= skip:
            worst = max(worst, O.log_spectral_distance(fi, fo))
    ctx.close()
    return worst
