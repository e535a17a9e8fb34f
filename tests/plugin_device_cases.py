"""Cases for the device twins of the plugin-level calls (extract_features_device, quantize_device, dequantize_device,
generate_device, logmel_device, noise_estimate_device, cng_generate_device, resample_device), shared by the CPU tier (emulated
kernels) and the GPU tier.  Each twin runs on caller buffers of exactly n rows inside a larger allocation with sentinel rows
around them (parity_cases.Guarded), against its host-buffer twin on a second context created alike, hop by hop with the state
carried between hops: outputs bit for bit, and the exported stream records of both contexts equal after every hop.  The chains
are checked against the fused encode_device + decode_device and against the oracle."""
import numpy as np

import rate_cases as rc
from conftest import MODEL_DIR
from parity_cases import Guarded

EINVAL = -1
CNG_SEED = 21
RESAMPLE_RATES = (8000, 32000, 48000)
LOGMEL_BANKS_BINS = ((0, 160), (1, 64), (0, 64), (1, 160))


def _pair(Context, api, mem, max_streams, *, roles="both", mode="exact", split=None, mask_n=None, seed=0):
    """(device context, host context) created alike.  The device context runs on mem.stream, with `split` sub-batches and,
    with mask_n, an active mask of mask_n rows with zeros in it installed (the plugin-level twins ignore it), kept alive on the
    context."""
    A, B = Context(max_streams, capi=api, roles=roles), Context(max_streams, capi=api, roles=roles)
    for c in (A, B):
        c.set_cng_seed(CNG_SEED)
        if roles != "encoder":
            c.set_decoder_mode(mode)
    if split is not None:
        A.set_split(split)
    if mem.stream is not None:
        A.set_stream(mem.stream)
    if mask_n is not None:
        A._mask = Guarded(mem, mask_n, (), np.uint8, 0x5A)
        A._mask.put((np.random.default_rng(seed).random(mask_n) < 0.5).astype(np.uint8))
        A.set_active_mask(A._mask.ptr)
    return A, B


def _records_equal(A, B, what, f):
    assert np.array_equal(A.export_streams(), B.export_streams()), "hop %d: stream records differ from the host twin's (%s)" % (f, what)


def _close(*cs):
    for c in cs:
        c.set_active_mask(None)
        c.close()


def run_nets_twin(Context, api, mem, wav, *, n, hops, mode="exact", split=None, tail=5, mask=False):
    """extract_features_device -> generate_device (of those features) against extract_features -> generate, hop by hop"""
    A, B = _pair(Context, api, mem, n + tail, mode=mode, split=split, mask_n=n if mask else None)
    d_pcm = Guarded(mem, n, (320,), np.int16, 0x3C)
    d_feat = Guarded(mem, n, (64,), np.float32, 0x7F)
    d_out = Guarded(mem, n, (320,), np.int16, 0x5A)
    for f in range(hops):
        pcm = rc.speech_rows(wav, 16000, range(n), f)
        d_pcm.put(pcm)
        d_feat.fill()
        d_out.fill()
        A.extract_features_device(n, d_pcm.ptr, d_feat.ptr)
        feats = d_feat.get("features")
        want = B.extract_features(pcm)
        assert np.array_equal(feats.view(np.uint32), want.view(np.uint32)), "hop %d: extract_features_device != extract_features" % f
        A.generate_device(n, d_feat.ptr, d_out.ptr)
        assert np.array_equal(d_out.get("PCM"), B.generate(want)), "hop %d: generate_device != generate (%s)" % (f, mode)
        d_pcm.get("input PCM")
        d_feat.get("features")
        _records_equal(A, B, "nets", f)
    _close(A, B)


def run_rvq_twin(Context, api, mem, *, n, hops, bits, indices, roles="both", mask=False, seed=5):
    """quantize_device (with and without indices) and dequantize_device against quantize / dequantize; dequantize_device also
    on random packets"""
    A, B = _pair(Context, api, mem, n + 3, roles=roles, mask_n=n if mask else None)
    P = (bits + 7) // 8
    d_feat = Guarded(mem, n, (64,), np.float32, 0x7F)
    d_pk = Guarded(mem, n, (P,), np.uint8, 0xA5)
    d_idx = Guarded(mem, n, (46,), np.int32, 0xEE)
    d_lossy = Guarded(mem, n, (64,), np.float32, 0x3D)
    rng = np.random.default_rng(seed)
    for f in range(hops):
        feats = rng.normal(0.0, 1.5, size=(n, 64)).astype(np.float32)
        d_feat.put(feats)
        d_pk.fill()
        d_idx.fill()
        A.quantize_device(n, d_feat.ptr, bits, d_pk.ptr, d_idx.ptr if indices else 0)
        pk, idx = B.quantize(feats, bits, want_indices=True)
        assert np.array_equal(d_pk.get("packets"), pk), "hop %d: quantize_device != quantize at %d bits" % (f, bits)
        got_idx = d_idx.get("indices")
        if indices:
            assert np.array_equal(got_idx, idx), "hop %d: quantize_device indices != quantize at %d bits" % (f, bits)
        else:
            assert (got_idx == d_idx.sentinel).all(), "quantize_device wrote indices without an index buffer"
        d_feat.get("features")
        for src in (pk, rng.integers(0, 256, size=(n, P)).astype(np.uint8)):
            d_pk.put(src)
            d_lossy.fill()
            A.dequantize_device(n, d_pk.ptr, bits, d_lossy.ptr)
            want = B.dequantize(src, bits)
            assert np.array_equal(d_lossy.get("features").view(np.uint32), want.view(np.uint32)), \
                "hop %d: dequantize_device != dequantize at %d bits" % (f, bits)
            d_pk.get("packets")
    _records_equal(A, B, "rvq", hops)
    _close(A, B)


def run_logmel_twin(Context, api, mem, wav, *, n, hops, banks_bins=LOGMEL_BANKS_BINS, mask=False):
    """logmel_device against logmel on every (bank, bins) of banks_bins, each hop, so both banks carry their samples"""
    A, B = _pair(Context, api, mem, n + 4, roles="encoder", mask_n=n if mask else None)
    d_pcm = Guarded(mem, n, (320,), np.int16, 0x3C)
    d_out = {bins: Guarded(mem, n, (bins,), np.float32, 0x7F) for bins in (64, 160)}
    for f in range(hops):
        pcm = rc.speech_rows(wav, 16000, range(n), f, stride=5)
        d_pcm.put(pcm)
        for bank, bins in banks_bins:
            d_out[bins].fill()
            A.logmel_device(n, d_pcm.ptr, d_out[bins].ptr, bins, bank)
            want = B.logmel(pcm, bins, bank)
            assert np.array_equal(d_out[bins].get("spectra").view(np.uint32), want.view(np.uint32)), \
                "hop %d: logmel_device != logmel (bank %d, %d bins)" % (f, bank, bins)
        d_pcm.get("input PCM")
        _records_equal(A, B, "logmel", f)
    _close(A, B)


def _cng_features(rng, n):
    """log-mel conditioning vectors in the range of the noise estimates (log(500) / 10 and up)"""
    return rng.uniform(0.62, 1.3, size=(n, 160)).astype(np.float32)


def run_cng_twin(Context, api, mem, *, n, hops, mask=False, seed=7):
    """cng_generate_device against cng_generate (the seed and each stream's key apply; the overlap-add buffers carry)"""
    A, B = _pair(Context, api, mem, n + 2, roles="decoder", mask_n=n if mask else None)
    d_feat = Guarded(mem, n, (160,), np.float32, 0x7F)
    d_out = Guarded(mem, n, (320,), np.int16, 0x5A)
    rng = np.random.default_rng(seed)
    for f in range(hops):
        feats = _cng_features(rng, n)
        d_feat.put(feats)
        d_out.fill()
        A.cng_generate_device(n, d_feat.ptr, d_out.ptr)
        out = d_out.get("PCM")
        assert np.array_equal(out, B.cng_generate(feats)), "hop %d: cng_generate_device != cng_generate" % f
        assert out.any(), "comfort noise is all zero"
        d_feat.get("features")
        _records_equal(A, B, "cng", f)
    _close(A, B)


def run_noise_twin(Context, api, mem, wav, *, n, hops, mask=False, seed=8):
    """noise_estimate_device after noise_update_device against noise_estimate after noise_update; each hop reads both outputs,
    the estimate only or the flags only"""
    A, B = _pair(Context, api, mem, n + 3, roles="decoder", mask_n=n if mask else None)
    d_pcm = Guarded(mem, n, (320,), np.int16, 0x3C)
    d_upd = Guarded(mem, n, (), np.uint8, 0xC3)
    d_est = Guarded(mem, n, (160,), np.float32, 0x7F)
    d_flags = Guarded(mem, n, (), np.uint8, 0xAA)
    rng = np.random.default_rng(seed)
    for f in range(hops):
        pcm = rc.speech_rows(wav, 16000, range(n), f, stride=3)
        pcm[np.arange(n) % 3 == 1] = 0                # silence on every third stream: the estimators' noise branch runs
        upd = (rng.random(n) < 0.8).astype(np.uint8)
        d_pcm.put(pcm)
        d_upd.put(upd)
        A.noise_update_device(n, d_pcm.ptr, d_upd.ptr, 0, 0)
        B.noise_update(pcm, update_mask=upd)
        want_est, want_flags = B.noise_estimate(n=n)
        want_flags = want_flags.astype(np.uint8)
        est_out, flag_out = (True, True) if f % 3 == 0 else (True, False) if f % 3 == 1 else (False, True)
        d_est.fill()
        d_flags.fill()
        A.noise_estimate_device(n, d_est.ptr if est_out else 0, d_flags.ptr if flag_out else 0)
        est, flags = d_est.get("estimate"), d_flags.get("is_noise")
        if est_out:
            assert np.array_equal(est.view(np.uint32), want_est.view(np.uint32)), "hop %d: noise_estimate_device estimate" % f
        else:
            assert (est == d_est.sentinel).all(), "noise_estimate_device wrote an estimate without an estimate buffer"
        if flag_out:
            assert np.array_equal(flags, want_flags), "hop %d: noise_estimate_device is_noise" % f
        else:
            assert (flags == d_flags.sentinel).all(), "noise_estimate_device wrote flags without a flag buffer"
        d_pcm.get("input PCM")
        _records_equal(A, B, "noise", f)
    _close(A, B)


def resample_sizes(rate, to_internal):
    """input sizes per hop: one 20 ms hop, then sizes that leave the filters at other phases"""
    return (rate // 50 if to_internal else 320, 157, 77, 240)


def run_resample_twin(Context, api, mem, *, n, hops, rate, to_internal, mask=False, seed=9):
    """resample_device against resample; the samples after a row's count stay as they were; the counts are written on the
    device"""
    A, B = _pair(Context, api, mem, n + 2, mask_n=n if mask else None)
    rng = np.random.default_rng(seed + rate)
    sizes = resample_sizes(rate, to_internal)
    ratio = (16000 / rate) if to_internal else (rate / 16000)
    for f in range(hops):
        n_in = sizes[f % len(sizes)]
        stride = int(np.ceil(n_in * ratio)) + 1         # the host binding's stride
        t = np.arange(n_in) + f * 1000
        x = (8000 * np.sin(2 * np.pi * (t[None, :] * (1 + np.arange(n)[:, None] % 7)) / 97.0)).astype(np.int16)
        x += rng.integers(-500, 500, size=x.shape, dtype=np.int16)
        d_in = Guarded(mem, n, (n_in,), np.int16, 0x3C)
        d_out = Guarded(mem, n, (stride,), np.int16, 0x5A)
        d_cnt = Guarded(mem, n, (), np.int32, 0xEE)
        d_in.put(x)
        A.resample_device(n, rate, to_internal, d_in.ptr, n_in, d_out.ptr, stride, d_cnt.ptr if f % 2 == 0 else 0)
        want = B.resample(x, rate, to_internal)
        got, cnt = d_out.get("output"), d_cnt.get("counts")
        lens = np.array([len(w) for w in want])
        if f % 2 == 0:
            assert np.array_equal(cnt, lens), "hop %d: resample_device counts != resample (%d Hz, to_internal %d)" % (f, rate, to_internal)
        else:
            assert (cnt == d_cnt.sentinel).all(), "resample_device wrote counts without a count buffer"
        for k in range(n):
            assert np.array_equal(got[k, :lens[k]], want[k]), "hop %d row %d: resample_device != resample (%d Hz)" % (f, k, rate)
            assert (got[k, lens[k]:] == d_out.sentinel).all(), "hop %d row %d: samples after the count were written" % (f, k)
        d_in.get("input")
        _records_equal(A, B, "resample", f)
    _close(A, B)


def run_chain(Context, api, mem, wav, O=None, *, n, hops, mode="exact", split=None, oracle_rows=(), bit_seq=(64, 120, 184),
              mask=False):
    """extract_features_device -> quantize_device -> dequantize_device -> generate_device on one context against
    encode_device + decode_device on a twin: the same packets and PCM, hop by hop, and the same records.  The bit rate changes
    every hop (bit_seq).  oracle_rows: those streams' features, packets, lossy features (and in the exact mode PCM) against
    oracle codecs."""
    A, B = _pair(Context, api, mem, n + 3, mode=mode, split=split, mask_n=n if mask else None)
    if split is not None:
        B.set_split(split)
    if mem.stream is not None:
        B.set_stream(mem.stream)
    d_pcm = Guarded(mem, n, (320,), np.int16, 0x3C)
    d_feat = Guarded(mem, n, (64,), np.float32, 0x7F)
    d_lossy = Guarded(mem, n, (64,), np.float32, 0x7F)
    d_out, d_out_b = Guarded(mem, n, (320,), np.int16, 0x5A), Guarded(mem, n, (320,), np.int16, 0x5A)
    codecs = {k: O.Codec(MODEL_DIR) for k in oracle_rows}
    for f in range(hops):
        bits = bit_seq[f % len(bit_seq)]
        P = (bits + 7) // 8
        d_pk, d_pk_b = Guarded(mem, n, (P,), np.uint8, 0xA5), Guarded(mem, n, (P,), np.uint8, 0xA5)
        pcm = rc.speech_rows(wav, 16000, range(n), f)
        d_pcm.put(pcm)
        for g in (d_feat, d_lossy, d_out, d_out_b):
            g.fill()
        A.extract_features_device(n, d_pcm.ptr, d_feat.ptr)
        A.quantize_device(n, d_feat.ptr, bits, d_pk.ptr)
        A.dequantize_device(n, d_pk.ptr, bits, d_lossy.ptr)
        A.generate_device(n, d_lossy.ptr, d_out.ptr)
        B.encode_device(n, d_pcm.ptr, bits, d_pk_b.ptr)
        B.decode_device(n, d_pk_b.ptr, 0, bits, d_out_b.ptr)
        pk, out = d_pk.get("packets"), d_out.get("PCM")
        assert np.array_equal(pk, d_pk_b.get("packets")), "hop %d: chain packets != encode_device (%d bits)" % (f, bits)
        assert np.array_equal(out, d_out_b.get("PCM")), "hop %d: chain PCM != decode_device (%s)" % (f, mode)
        feats, lossy = d_feat.get("features"), d_lossy.get("lossy features")
        for k in oracle_rows:
            opkt, ofeat, _ = codecs[k].encode(pcm[k], bits)
            assert np.array_equal(feats[k], ofeat), "hop %d row %d: features != oracle" % (f, k)
            assert bytes(pk[k]) == opkt, "hop %d row %d: packet != oracle" % (f, k)
            opcm, olossy, _ = codecs[k].decode(opkt, bits)
            assert np.array_equal(lossy[k], olossy), "hop %d row %d: lossy features != oracle" % (f, k)
            if mode == "exact":
                assert np.array_equal(out[k], opcm), "hop %d row %d: generate_device PCM != oracle" % (f, k)
        d_pcm.get("input PCM")
        _records_equal(A, B, "chain", f)
    _close(A, B)


def run_cng_chain(Context, api, mem, wav, *, n, hops, mask=False, seed=10):
    """noise_update_device -> noise_estimate_device -> cng_generate_device (comfort noise from the decoder-side estimate) against
    the same chain of host-buffer calls"""
    A, B = _pair(Context, api, mem, n + 2, roles="decoder", mask_n=n if mask else None)
    d_pcm = Guarded(mem, n, (320,), np.int16, 0x3C)
    d_est = Guarded(mem, n, (160,), np.float32, 0x7F)
    d_out = Guarded(mem, n, (320,), np.int16, 0x5A)
    rng = np.random.default_rng(seed)
    for f in range(hops):
        pcm = rc.speech_rows(wav, 16000, range(n), f, stride=11)
        pcm[np.arange(n) % 2 == 0] //= 64                # quiet streams
        d_pcm.put(pcm)
        d_est.fill()
        d_out.fill()
        A.noise_update_device(n, d_pcm.ptr, 0, 0, 0)
        A.noise_estimate_device(n, d_est.ptr, 0)
        A.cng_generate_device(n, d_est.ptr, d_out.ptr)
        B.noise_update(pcm)
        est, _ = B.noise_estimate(n=n)
        want = B.cng_generate(est)
        assert np.array_equal(d_est.get("estimate").view(np.uint32), est.view(np.uint32)), "hop %d: estimate != host chain" % f
        assert np.array_equal(d_out.get("PCM"), want), "hop %d: comfort noise != host chain" % f
        _records_equal(A, B, "cng chain", f)
    _close(A, B)


def run_refusals(Context, api, mem):
    """Every way to call a twin wrongly returns LYRA_B200_EINVAL and launches nothing"""
    n_max = 16
    ctx = Context(n_max, capi=api)
    enc, dec = Context(n_max, capi=api, roles="encoder"), Context(n_max, capi=api, roles="decoder")
    pcm = mem.zeros((n_max, 960), np.int16)
    feat = mem.zeros((n_max, 160), np.float32)
    pk = mem.zeros((n_max, 24), np.uint8)
    idx = mem.zeros((n_max, 46), np.int32)
    out = mem.zeros((n_max, 968), np.int16)
    cnt = mem.zeros((n_max,), np.int32)
    fl = mem.zeros((n_max,), np.uint8)
    P, F, K, I, O, N, L = (mem.ptr(b) for b in (pcm, feat, pk, idx, out, cnt, fl))
    lib = api.lib

    def calls(c, n):
        h = c.h
        return {
            "extract": lambda p=P, q=F: lib.lyra_b200_extract_features_device(h, n, p, q),
            "quantize": lambda p=F, q=K, b=64: lib.lyra_b200_quantize_device(h, n, p, b, q, I),
            "dequantize": lambda p=K, q=F, b=64: lib.lyra_b200_dequantize_device(h, n, p, b, q),
            "generate": lambda p=F, q=P: lib.lyra_b200_generate_device(h, n, p, q),
            "logmel": lambda p=P, q=F, bank=0, bins=160: lib.lyra_b200_logmel_device(h, bank, n, p, bins, q),
            "noise_estimate": lambda p=F, q=L: lib.lyra_b200_noise_estimate_device(h, n, p, q),
            "cng": lambda p=F, q=P: lib.lyra_b200_cng_generate_device(h, n, p, q),
            "resample": lambda p=P, q=O, rate=48000, to=1, n_in=960, stride=321: lib.lyra_b200_resample_device(h, to, n, rate, p, n_in, q,
                                                                                                               stride, N),
        }

    bad = []
    ok = calls(ctx, 4)
    for name, fn in ok.items():
        bad.append((ctx, name + " n=0", calls(ctx, 0)[name]))
        bad.append((ctx, name + " n=-1", calls(ctx, -1)[name]))
        bad.append((ctx, name + " n>max", calls(ctx, n_max + 1)[name]))
    bad += [
        (ctx, "extract NULL pcm", lambda: ok["extract"](p=None)), (ctx, "extract NULL features", lambda: ok["extract"](q=None)),
        (ctx, "quantize NULL features", lambda: ok["quantize"](p=None)), (ctx, "quantize NULL packets", lambda: ok["quantize"](q=None)),
        (ctx, "dequantize NULL packets", lambda: ok["dequantize"](p=None)),
        (ctx, "dequantize NULL features", lambda: ok["dequantize"](q=None)),
        (ctx, "generate NULL features", lambda: ok["generate"](p=None)), (ctx, "generate NULL pcm", lambda: ok["generate"](q=None)),
        (ctx, "logmel NULL pcm", lambda: ok["logmel"](p=None)), (ctx, "logmel NULL out", lambda: ok["logmel"](q=None)),
        (ctx, "noise_estimate both NULL", lambda: ok["noise_estimate"](p=None, q=None)),
        (ctx, "cng NULL features", lambda: ok["cng"](p=None)), (ctx, "cng NULL pcm", lambda: ok["cng"](q=None)),
        (ctx, "resample NULL in", lambda: ok["resample"](p=None)), (ctx, "resample NULL out", lambda: ok["resample"](q=None)),
    ]
    for b in (0, -4, 6, 188, 1000):
        bad.append((ctx, "quantize bits %d" % b, lambda b=b: ok["quantize"](b=b)))
        bad.append((ctx, "dequantize bits %d" % b, lambda b=b: ok["dequantize"](b=b)))
    for bank in (-1, 2):
        bad.append((ctx, "logmel bank %d" % bank, lambda bank=bank: ok["logmel"](bank=bank)))
    for bins in (0, 63, 80, 161):
        bad.append((ctx, "logmel bins %d" % bins, lambda bins=bins: ok["logmel"](bins=bins)))
    for rate in (0, 16000, 44100, 96000):
        bad.append((ctx, "resample rate %d" % rate, lambda rate=rate: ok["resample"](rate=rate)))
    bad += [
        (ctx, "resample n_in 0", lambda: ok["resample"](n_in=0, stride=1)),
        (ctx, "resample n_in 961", lambda: ok["resample"](n_in=961)),
        (ctx, "resample stride below the outputs", lambda: ok["resample"](stride=319)),
        (ctx, "resample stride 969", lambda: ok["resample"](stride=969)),
        (ctx, "resample more than 960 outputs", lambda: ok["resample"](to=0, n_in=321, stride=964)),
        (dec, "extract in a decoder-only context", calls(dec, 4)["extract"]),
        (enc, "generate in an encoder-only context", calls(enc, 4)["generate"]),
    ]
    for c, what, fn in bad:
        l0 = c.launch_count
        assert fn() == EINVAL, "%s: not refused" % what
        assert c.launch_count == l0, "%s: refused but launched" % what
    # the same arguments, corrected, are accepted (so each refusal above is the one thing it names)
    for name, fn in ok.items():
        c = {"extract": enc, "generate": dec}.get(name, ctx)
        assert calls(c, 4)[name]() == 0, "%s: a good call refused" % name
    assert ok["resample"](to=0, n_in=320, stride=960) == 0 and ok["resample"](rate=8000, to=1, n_in=160, stride=321) == 0
    ctx.synchronize()
    for c in (ctx, enc, dec):
        c.close()
