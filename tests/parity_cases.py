"""Parity cases shared by the CPU tier (emulated kernels) and the GPU tier (real kernels): every case drives
the C ABI and compares with the oracle on the same seeded inputs.  Bar: bit-exact packets, RVQ indices,
features, int16 PCM, log-mel spectra and noise-estimator state (the one libm call on each of those paths, log / exp,
is taken in double and rounded once on both sides).

The decoder's opt-in tensor-core mode (lyra_b200_set_decoder_mode, split-precision TF32) is the one floating-point
path that is compared with a tolerance: decoded int16 PCM within TENSOR_PCM_TOL_LSB of the oracle (the drop-in
target in BASELINE.json allows 1e-3 of full scale = 32.8 LSB); packets stay bit-exact in that mode too."""
import numpy as np

from conftest import MODEL_DIR


TENSOR_PCM_TOL_LSB = 4      # |PCM_tensor - PCM_oracle| <= 4 int16 LSB = 1.2e-4 of full scale


def synth_pcm(rng, n, kind="noise"):
    if kind == "noise":      # 0.25 full-scale uniform noise, the reference benchmark's input (lyra_benchmark_lib.cc:233-239)
        return rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16)
    if kind == "loud":       # full-scale, exercises clipping in UnitToInt16 and int8 saturation
        return rng.integers(-32768, 32768, size=(n, 320), dtype=np.int16)
    if kind == "silence":
        return np.zeros((n, 320), dtype=np.int16)
    raise ValueError(kind)


def run_codec_parity(Context, api, O, *, max_streams, stream_ids, frames, bits, kind="noise", seed=0, loss_every=0,
                     wav=None, check=None, decoder_mode="exact"):
    """Encode+decode `frames` hops of the listed streams; compare `check` (default: all) against per-stream oracles.
    Returns the largest |PCM difference| seen (0 unless decoder_mode == "tensor")."""
    ctx = Context(max_streams, capi=api)
    ctx.set_decoder_mode(decoder_mode)
    pcm_tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    worst = 0
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    check = list(range(n)) if check is None else check
    codecs = {k: O.Codec(MODEL_DIR) for k in check}
    rng = np.random.default_rng(seed)
    for f in range(frames):
        if wav is not None:
            pcm = np.stack([wav[(320 * (f + 7 * k)) % (len(wav) - 320):][:320] for k in range(n)])
        else:
            pcm = synth_pcm(rng, n, kind)
        packets = ctx.encode(pcm, bits, stream_ids=ids)
        received = None
        if loss_every:
            received = np.array([0 if (f + k) % loss_every == 0 else 1 for k in range(n)], dtype=np.uint8)
        out = ctx.decode(packets, bits, stream_ids=ids, received=received)
        for k in check:
            opkt, _, _ = codecs[k].encode(pcm[k], bits)
            lost = received is not None and received[k] == 0
            opcm, _, _ = codecs[k].decode(None if lost else opkt, bits)
            assert bytes(packets[k]) == opkt, "packet mismatch frame %d stream %d" % (f, ids[k])
            diff = int(np.abs(out[k].astype(int) - opcm.astype(int)).max())
            worst = max(worst, diff)
            assert diff <= pcm_tol, "PCM mismatch frame %d stream %d (max |d| %d, allowed %d)" % (f, ids[k], diff, pcm_tol)
    ctx.close()
    return worst


def run_priority_switch(Context, api, O, *, n=3, frames=4, bits=64, split=2):
    """lyra_b200_set_priority between hops (streams re-created, sub-batches in use): the streaming state is untouched, results stay
    the oracle's."""
    ctx = Context(max(16, n), capi=api)
    ctx.set_split(split)
    codecs = [O.Codec(MODEL_DIR) for _ in range(n)]
    rng = np.random.default_rng(21)
    for f in range(frames):
        ctx.set_priority([-1, 0, -2, 0][f % 4])
        pcm = synth_pcm(rng, n)
        packets = ctx.encode(pcm, bits)
        out = ctx.decode(packets, bits)
        for k in range(n):
            opkt, _, _ = codecs[k].encode(pcm[k], bits)
            opcm, _, _ = codecs[k].decode(opkt, bits)
            assert bytes(packets[k]) == opkt and np.array_equal(out[k], opcm), "mismatch after a priority switch (hop %d stream %d)" % (f, k)
    ctx.close()


def run_plugin_surface_parity(Context, api, O, *, n=5, frames=3, seed=1):
    """extract_features / quantize / dequantize / generate one by one against the oracle's pieces."""
    import os
    ctx = Context(n, capi=api)
    rng = np.random.default_rng(seed)
    codecs = [O.Codec(MODEL_DIR) for _ in range(n)]
    rvq = O.Rvq(os.path.join(MODEL_DIR, "quantizer.tflite"))
    for f in range(frames):
        pcm = synth_pcm(rng, n, "noise")
        feats = ctx.extract_features(pcm)
        for bits in (64, 120, 184):
            packets, idx = ctx.quantize(feats, bits, want_indices=True)
            lossy = ctx.dequantize(packets, bits)
            for k in range(n):
                want_idx = rvq.encode(feats[k], bits // 4)
                assert np.array_equal(idx[k], want_idx)
                want_bits = rvq.quantize(feats[k], bits)
                assert bytes(packets[k]) == O.packet_pack(want_bits, 0, bits)
                assert np.array_equal(lossy[k], rvq.decode_to_lossy_features(want_bits))
        lossy = ctx.dequantize(ctx.quantize(feats, 120), 120)
        out = ctx.generate(lossy)
        for k in range(n):
            opkt, ofeat, _ = codecs[k].encode(pcm[k], 120)
            assert np.array_equal(feats[k], ofeat)
            opcm, olossy, _ = codecs[k].decode(opkt, 120)
            assert np.array_equal(lossy[k], olossy)
            assert np.array_equal(out[k], opcm)
    ctx.close()


def run_reset_and_isolation(Context, api, O, *, seed=2):
    """Streams are independent; reset(ids) restores exactly the initial state of those streams only."""
    ctx = Context(40, capi=api)
    rng = np.random.default_rng(seed)
    a = synth_pcm(rng, 3, "noise")
    ids = np.array([3, 19, 33], dtype=np.int32)
    first = [ctx.encode(a, 64, stream_ids=ids) for _ in range(2)]
    # other streams running in between must not disturb 3/19/33
    ctx.encode(synth_pcm(rng, 4, "noise"), 64, stream_ids=np.array([2, 4, 18, 32], dtype=np.int32))
    third = ctx.encode(a, 64, stream_ids=ids)
    ref = O.Codec(MODEL_DIR)
    want = [ref.encode(a[0], 64)[0] for _ in range(3)]
    assert [bytes(first[0][0]), bytes(first[1][0]), bytes(third[0])] == want
    ctx.reset(np.array([19], dtype=np.int32))
    again = ctx.encode(a, 64, stream_ids=ids)
    ref19 = O.Codec(MODEL_DIR)
    assert bytes(again[1]) == ref19.encode(a[1], 64)[0]          # stream 19 restarted from zero state
    assert bytes(again[0]) == ref.encode(a[0], 64)[0]            # stream 3 carried on
    ctx.close()


def run_error_paths(Context, api, LyraB200Error):
    ctx = Context(8, capi=api)
    pcm = np.zeros((2, 320), dtype=np.int16)
    feats = np.zeros((1, 64), dtype=np.float32)

    def fails(fn):
        try:
            fn()
        except LyraB200Error as e:
            assert e.code == -1
            return True
        return False
    assert fails(lambda: ctx.quantize(feats, 185))                                  # too many bits
    assert fails(lambda: ctx.quantize(feats, 62))                                   # not divisible by 4
    assert fails(lambda: ctx.encode(pcm, 64, stream_ids=np.array([1, 1], dtype=np.int32)))   # duplicate id
    assert fails(lambda: ctx.encode(pcm, 64, stream_ids=np.array([1, 8], dtype=np.int32)))   # id out of range
    assert fails(lambda: ctx.encode(np.zeros((9, 320), np.int16), 64))              # more rows than streams
    assert fails(lambda: ctx.logmel(pcm, num_mel_bins=80))
    # every call that takes stream ids refuses ids out of range and, except reset and the control-state calls, repeated ids
    pk = np.zeros((2, 8), dtype=np.uint8)
    takes_ids = {
        "encode": lambda ids: ctx.encode(pcm, 64, stream_ids=ids),
        "decode": lambda ids: ctx.decode(pk, 64, stream_ids=ids),
        "extract_features": lambda ids: ctx.extract_features(pcm, stream_ids=ids),
        "generate": lambda ids: ctx.generate(np.zeros((2, 64), np.float32), stream_ids=ids),
        "logmel": lambda ids: ctx.logmel(pcm, stream_ids=ids),
        "noise_update": lambda ids: ctx.noise_update(pcm, stream_ids=ids),
        "noise_estimate": lambda ids: ctx.noise_estimate(stream_ids=ids),
        "decode_track_noise": lambda ids: ctx.decode_track_noise(pk, 64, stream_ids=ids),
        "decode_plc": lambda ids: ctx.decode_plc(pk, 64, stream_ids=ids),
        "cng_generate": lambda ids: ctx.cng_generate(np.zeros((2, 160), np.float32), stream_ids=ids),
        "encode_dtx": lambda ids: ctx.encode_dtx(pcm, 64, stream_ids=ids),
        "resample": lambda ids: ctx.resample(np.zeros((2, 160), np.int16), 8000, True, stream_ids=ids),
    }
    repeats_ok = {
        "reset": lambda ids: ctx.reset(stream_ids=ids),
        "plc_state": lambda ids: ctx.plc_state(stream_ids=ids),
        "set_plc_state": lambda ids: ctx.set_plc_state([(0, 0, -1)] * len(ids), stream_ids=ids),
    }
    for name, call in list(takes_ids.items()) + list(repeats_ok.items()):
        for bad in ([1, 8], [-1, 2]):
            assert fails(lambda: call(np.array(bad, dtype=np.int32))), "%s accepted stream ids %s" % (name, bad)
        if name in takes_ids:
            assert fails(lambda: call(np.array([3, 3], dtype=np.int32))), "%s accepted a repeated stream id" % name
        else:
            call(np.array([3, 3], dtype=np.int32))
    ctx.close()


def _every_stateful_call(ctx, f, ids, wav, bits):
    """Hop f of every call that advances per-stream state, on streams `ids`; the inputs depend on f only.  Decode_plc receives hop 0,
    loses hops 1..7 (long enough to reach comfort noise) and then every other stream's packets.  Returns {name: per-stream rows}."""
    n = len(ids)
    rng = np.random.default_rng(100 + f)
    pcm = np.stack([wav[(320 * (f + 9 * k + 30)) % (len(wav) - 320):][:320] for k in range(n)]).copy()
    quiet = pcm.copy()
    quiet[::2] = 0                                       # DTX and the estimators' noise branch on every other stream
    out = {}
    pk = ctx.encode(pcm, bits, stream_ids=ids)
    out["packets"] = pk
    out["pcm"] = ctx.decode(pk, bits, stream_ids=ids, received=(np.arange(n) + f) % 4 != 0)
    plc_rec = np.ones(n, np.uint8) if f == 0 else (np.arange(n) % 2).astype(np.uint8) if f >= 8 else np.zeros(n, np.uint8)
    out["plc_pcm"], out["comfort_noise"] = ctx.decode_plc(pk, bits, stream_ids=ids, received=plc_rec)
    out["plc_state"] = ctx.plc_state(stream_ids=ids)
    out["dtx_packets"], out["dtx_bytes"] = ctx.encode_dtx(quiet, bits, stream_ids=ids)
    out["logmel_bank0"] = ctx.logmel(pcm, 160, bank=0, stream_ids=ids)
    out["logmel_bank1"] = ctx.logmel(quiet, 64, bank=1, stream_ids=ids)
    out["is_noise"], out["noise_estimate"] = ctx.noise_update(quiet, stream_ids=ids)
    out["cng"] = ctx.cng_generate(rng.uniform(0.62, 1.2, size=(n, 160)).astype(np.float32), stream_ids=ids)
    chunk = (960, 7, 955, 480, 13, 960)[f % 6]           # ragged chunks leave the resamplers mid-phase
    out["resample_in"] = ctx.resample(rng.integers(-20000, 20000, size=(n, chunk)).astype(np.int16), 48000, True, stream_ids=ids)
    out["resample_out"] = ctx.resample(pcm[:, :320 - 17 * (f % 5)], 8000, False, stream_ids=ids)
    return out


def run_reset_restores_every_stream_state(Context, api, wav, *, max_streams=16, ids=(1, 6, 9, 14), reset_ids=(9, 1, 9), dense_n=8,
                                          hops=9, bits=64, cng_seed=3, dense_launches=None):
    """lyra_b200_reset restores all per-stream state: three contexts run the same history through every stateful call, then one
    resets `reset_ids` (an id listed twice) and one resets streams 0..dense_n-1.  On the next hop a reset stream must equal a fresh
    context's first hop and every other stream the twin that was not reset, in every output and in the control state, bit for bit.
    dense_launches: the kernel launches the dense reset must take (one per 1024 streams)."""
    ids = np.asarray(ids, dtype=np.int32)

    def make():
        c = Context(max_streams, capi=api)
        c.set_cng_seed(cng_seed)
        return c
    sparse, dense, twin = make(), make(), make()
    seen_cn = seen_dtx = False
    for f in range(hops):
        for c in (sparse, dense, twin):
            o = _every_stateful_call(c, f, ids, wav, bits)
        seen_cn |= bool(o["comfort_noise"].any())
        seen_dtx |= bool((o["dtx_bytes"] == 0).any())
    assert seen_cn and seen_dtx, "the history must reach comfort noise and DTX"
    sparse.reset(np.asarray(reset_ids, dtype=np.int32))
    launches = dense.launch_count
    dense.reset(n=dense_n)
    if dense_launches is not None:
        assert dense.launch_count - launches == dense_launches, "reset(n=%d) took %d launches" % (dense_n, dense.launch_count - launches)
    fresh = make()
    twin_state = twin.plc_state(stream_ids=ids)
    want = {True: _every_stateful_call(fresh, hops, ids, wav, bits), False: _every_stateful_call(twin, hops, ids, wav, bits)}
    for c, was_reset, how in ((sparse, np.isin(ids, reset_ids), "reset(%s)" % list(reset_ids)), (dense, ids < dense_n, "reset(n=%d)" % dense_n)):
        assert was_reset.any() and not was_reset.all()
        st = c.plc_state(stream_ids=ids)
        got = _every_stateful_call(c, hops, ids, wav, bits)
        for k, s in enumerate(ids):
            assert tuple(st[k]) == ((0, 0, -1) if was_reset[k] else tuple(twin_state[k])), "control state of stream %d after %s" % (s, how)
            for name, rows in got.items():
                assert np.array_equal(rows[k], want[bool(was_reset[k])][name][k]), "%s of stream %d after %s" % (name, s, how)
    for c in (sparse, dense, twin, fresh):
        c.close()


def run_logmel_parity(Context, api, O, wav, *, n=4, frames=4, tol=0.0):
    ctx = Context(n, capi=api)
    for nmel, bank in ((160, 0), (64, 1)):
        refs = [O.LogMel(16000, 320, 640, nmel) for _ in range(n)]
        for f in range(frames):
            pcm = np.stack([wav[320 * (f + 11 * k):][:320] for k in range(n)])
            out = ctx.logmel(pcm, num_mel_bins=nmel, bank=bank)
            for k in range(n):
                want = refs[k].extract(pcm[k])
                assert np.abs(out[k] - want).max() <= tol, (nmel, f, k, np.abs(out[k] - want).max())
    ctx.close()


def run_noise_estimator_parity(Context, api, O, wav, *, n=3, frames=30, seed=4):
    """lyra_b200_noise_update against one oracle NoiseEstimator per stream: speech with silent stretches (so both the
    update and the decay branch run), some hops withheld (update_mask 0, as after a lost packet), sparse stream ids.
    Bar: is_noise identical; noise_estimate bit-identical (the kernel evaluates the C++ expressions operation by operation)."""
    ctx = Context(4 * n, capi=api)
    ids = np.arange(n, dtype=np.int32) * 3 + 1
    est = [O.NoiseEstimator() for _ in range(n)]
    rng = np.random.default_rng(seed)
    seen_noise, seen_speech = False, False
    for f in range(frames):
        hop = np.stack([wav[(320 * (f + 11 * k)) % (len(wav) - 320):][:320] for k in range(n)]).copy()
        quiet = rng.random(n) < 0.4                   # silence / faint noise: exercises the is-noise branch
        for k in range(n):
            if quiet[k]:
                hop[k] = rng.integers(-2, 3, size=320, dtype=np.int16) if f % 2 else 0
        mask = (rng.random(n) < 0.85).astype(np.uint8)
        flags, got = ctx.noise_update(hop, stream_ids=ids, update_mask=mask)
        for k in range(n):
            if mask[k]:
                est[k].receive_samples(hop[k])
            assert bool(flags[k]) == est[k].is_noise, "is_noise mismatch frame %d stream %d" % (f, k)
            want = est[k].noise_estimate()
            assert np.array_equal(got[k], want), "noise estimate mismatch frame %d stream %d (max |d| %g)" % (
                f, k, np.abs(got[k] - want).max())
            seen_noise |= bool(flags[k]) and f > 0
            seen_speech |= not bool(flags[k])
    assert seen_noise and seen_speech, "the case must exercise both branches"
    # reset restores the freshly constructed estimator for the listed streams only
    ctx.reset(stream_ids=ids[:1])
    flags, got = ctx.noise_update(np.zeros((n, 320), dtype=np.int16), stream_ids=ids, update_mask=np.zeros(n, dtype=np.uint8))
    assert flags[0] and not got[0].any()
    assert np.array_equal(got[1], est[1].noise_estimate())
    ctx.close()


def run_decode_track_noise_parity(Context, api, O, wav, *, n=3, frames=12, max_streams=None, stream_ids=None, loss_every=4,
                                  check=None):
    """lyra_b200_decode_track_noise = decode + NoiseEstimator::ReceiveSamples for the received streams
    (LyraDecoder::DecodeSamplesInternal, lyra/lyra_decoder.cc:306-311): PCM, is_noise and the estimate bit-exact."""
    ids = np.arange(n, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    ctx = Context(max_streams or int(ids.max()) + 1, capi=api)
    dense = stream_ids is None and (max_streams is None or max_streams == n)
    check = list(range(n)) if check is None else check
    codecs = {k: O.Codec(MODEL_DIR) for k in check}
    est = {k: O.NoiseEstimator() for k in check}
    for f in range(frames):
        pcm = np.stack([wav[(320 * (f + 5 * k)) % (len(wav) - 320):][:320] for k in range(n)]).copy()
        if f % 3 == 2:
            pcm[:] = 0                                  # silent hops: the decoder output becomes noise-like
        packets = ctx.encode(pcm, 64, stream_ids=None if dense else ids)
        received = np.array([0 if (f + k) % loss_every == 0 else 1 for k in range(n)], dtype=np.uint8)
        out, flags = ctx.decode_track_noise(packets, 64, stream_ids=None if dense else ids, received=received)
        for k in check:
            opkt, _, _ = codecs[k].encode(pcm[k], 64)
            opcm, _, _ = codecs[k].decode(opkt if received[k] else None, 64)
            assert np.array_equal(out[k], opcm), "PCM mismatch frame %d stream %d" % (f, k)
            if received[k]:
                est[k].receive_samples(opcm)
            assert bool(flags[k]) == est[k].is_noise, "is_noise mismatch frame %d stream %d" % (f, k)
    _, got = ctx.noise_update(np.zeros((n, 320), dtype=np.int16), stream_ids=None if dense else ids, update_mask=np.zeros(n, dtype=np.uint8))
    for k in check:
        assert np.array_equal(got[k], est[k].noise_estimate()), "noise estimate mismatch stream %d" % k
    ctx.close()


def run_role_contexts(Context, api, O, LyraB200Error, mem, *, frames=4, seed=9):
    """lyra_b200_create_ex: an encoder-only and a decoder-only context together reproduce the oracle; calls of the missing
    role are refused with EINVAL (the mirror of LyraEncoder / LyraDecoder being separate objects), the device-resident
    variants included.  `mem` provides device buffers (HostMem / a torch-backed equivalent)."""
    n = 3
    enc = Context(8, capi=api, roles="encoder")
    dec = Context(8, capi=api, roles="decoder")
    codecs = [O.Codec(MODEL_DIR) for _ in range(n)]
    rng = np.random.default_rng(seed)
    for f in range(frames):
        pcm = synth_pcm(rng, n)
        pk = enc.encode(pcm, 120)
        out = dec.decode(pk, 120)
        for k in range(n):
            opkt, _, _ = codecs[k].encode(pcm[k], 120)
            opcm, _, _ = codecs[k].decode(opkt, 120)
            assert bytes(pk[k]) == opkt and np.array_equal(out[k], opcm), (f, k)
    d_pcm, d_pk = mem.zeros((n, 320), np.int16), mem.zeros((n, 15), np.uint8)
    d_flags, d_est = mem.zeros(n, np.uint8), mem.zeros((n, 160), np.float32)
    mem.put(d_pcm, pcm)
    p = mem.ptr
    for bad in (lambda: enc.decode(pk, 120), lambda: dec.encode(pcm, 120), lambda: enc.decode_plc(pk, 120),
                lambda: dec.encode_dtx(pcm, 120), lambda: dec.extract_features(pcm),
                lambda: dec.encode_device(n, p(d_pcm), 120, p(d_pk)), lambda: enc.decode_device(n, p(d_pk), 0, 120, p(d_pcm)),
                lambda: enc.decode_track_noise_device(n, p(d_pk), 0, 120, p(d_pcm)),
                lambda: enc.decode_plc_device(n, p(d_pk), 0, 120, p(d_pcm)),
                lambda: dec.encode_dtx_device(n, p(d_pcm), 120, p(d_pk), p(d_flags))):
        try:
            bad()
            raise AssertionError("a call of the missing role must fail")
        except LyraB200Error as e:
            assert e.code == -1
    assert enc.quantize(np.zeros((1, 64), dtype=np.float32), 64).shape == (1, 8)      # stateless calls work in any context
    assert enc.noise_update(pcm)[1].shape == (n, 160)                                  # ... and so do the self-contained estimators
    # ... through the device-resident variant as well: the encoder-only context's second hop, against a fresh oracle estimator
    # fed the same two hops
    mem.put(d_pcm, pcm)
    enc.set_stream(mem.stream)
    enc.noise_update_device(n, p(d_pcm), 0, p(d_flags), p(d_est))
    enc.set_stream(None)
    for k in range(n):
        est = O.NoiseEstimator()
        est.receive_samples(pcm[k])
        est.receive_samples(pcm[k])
        assert mem.get(d_flags)[k] == int(est.is_noise) and np.array_equal(mem.get(d_est)[k], est.noise_estimate()), k
    enc.reset()
    dec.reset()
    enc.close()
    dec.close()


# ---- packet-loss concealment / comfort noise / DTX (SURVEY.md section 8 rows f2, f4) ----

def run_cng_parity(Context, api, O, *, stream_ids=(0, 5), hops=4, seed=9, cng_seed=77):
    """lyra_b200_cng_generate vs the oracle's ComfortNoiseGenerator on the same features and the same seeded phases:
    bit-identical int16 hops (overlap-add state included), several hops in a row."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    ctx = Context(int(ids.max()) + 1, capi=api)
    ctx.set_cng_seed(cng_seed)
    gens = [O.ComfortNoiseGenerator(seed=cng_seed + int(i)) for i in ids]
    rng = np.random.default_rng(seed)
    for h in range(hops):
        feats = rng.uniform(0.62, 1.2, size=(len(ids), 160)).astype(np.float32)       # log-mel values between the floor and loud noise
        out = ctx.cng_generate(feats, stream_ids=ids)
        for k, g in enumerate(gens):
            want = g.condition(feats[k])
            assert np.array_equal(out[k], want), "comfort noise mismatch hop %d stream %d (max |d| %d)" % (
                h, ids[k], int(np.abs(out[k].astype(int) - want.astype(int)).max()))
    ctx.close()


def run_plc_parity(Context, api, O, *, max_streams=16, stream_ids=(1, 6, 9), frames=26, bits=64, wav=None, seed=4, cng_seed=5,
                   outages=((3, 12), (5, 3), (0, 0)), decoder_mode="exact"):
    """lyra_b200_decode_plc tick by tick vs one oracle LyraDecoder per stream: stream k loses `outages[k] = (first, count)` hops.
    PCM (model audio, comfort noise and their cross-fades), the control state and is_comfort_noise must all agree bit for bit
    (PCM within the stated tolerance in the tensor decoder mode)."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    ctx = Context(max_streams, capi=api)
    ctx.set_decoder_mode(decoder_mode)
    ctx.set_cng_seed(cng_seed)
    tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    encs = [O.Encoder(MODEL_DIR) for _ in range(n)]
    decs = [O.Decoder(MODEL_DIR, cng_seed=cng_seed + int(i)) for i in ids]
    rng = np.random.default_rng(seed)
    seen_cn = False
    for f in range(frames):
        if wav is not None:
            pcm = np.stack([wav[(320 * (f + 11 * k)) % (len(wav) - 320):][:320] for k in range(n)])
        else:
            pcm = synth_pcm(rng, n, "noise")
        pk = np.stack([np.frombuffer(encs[k].encode(pcm[k], bits), dtype=np.uint8) for k in range(n)])
        rec = np.array([0 if outages[k][0] <= f < outages[k][0] + outages[k][1] else 1 for k in range(n)], dtype=np.uint8)
        out, cn = ctx.decode_plc(pk, bits, stream_ids=ids, received=rec)
        st = ctx.plc_state(stream_ids=ids)
        for k in range(n):
            if rec[k]:
                assert decs[k].set_encoded_packet(bytes(pk[k]))
            want = decs[k].decode_samples(320)
            d = int(np.abs(out[k].astype(int) - want.astype(int)).max())
            assert d <= tol, "PLC PCM mismatch frame %d stream %d: max |d| %d (state %s)" % (f, ids[k], d, decs[k].state)
            assert tuple(int(x) for x in st[k]) == decs[k].state, (f, k, st[k], decs[k].state)
            assert bool(cn[k]) == decs[k].is_comfort_noise()
            seen_cn |= bool(cn[k])
    assert seen_cn, "the case never reached comfort noise"
    ctx.close()


def run_plc_state_peer(Context, api, O):
    """The reference's test peer (lyra_decoder_test.cc:56-90): forced states produce the same next hop as the oracle, and
    misaligned states are refused."""
    ctx = Context(4, capi=api)
    ctx.set_cng_seed(3)
    pk = np.zeros((1, 8), dtype=np.uint8)
    for state, rec in [((1280, 0, 1), 0), ((1280, 640, 1), 0), ((0, 640, -1), 1), ((1280, 320, 1), 1), ((640, 0, -1), 0)]:
        ctx.reset()
        ctx.set_plc_state([state], stream_ids=[2])
        dec = O.Decoder(MODEL_DIR, cng_seed=3 + 2)
        dec.state = state
        if rec:
            assert dec.set_encoded_packet(bytes(pk[0]))
        want = dec.decode_samples(320)
        out, cn = ctx.decode_plc(pk, 64, stream_ids=[2], received=[rec])
        assert np.array_equal(out[0], want), state
        assert tuple(int(x) for x in ctx.plc_state(stream_ids=[2])[0]) == dec.state
    try:
        ctx.set_plc_state([(100, 0, 1)], stream_ids=[0])
    except Exception:
        pass
    else:
        raise AssertionError("a misaligned control state must be refused")
    ctx.close()


def run_dtx_parity(Context, api, O, *, wav, frames=24, bits=64, stream_ids=(0, 3, 4)):
    """lyra_b200_encode_dtx vs the oracle's LyraEncoder(enable_dtx): stream 0 speech, stream 1 digital silence, stream 2
    silence then speech.  Packet sizes (0 = DTX) and bytes agree; encoder state only advances on encoded hops."""
    ids = np.asarray(stream_ids, dtype=np.int32)
    n = len(ids)
    ctx = Context(int(ids.max()) + 1, capi=api)
    encs = [O.Encoder(MODEL_DIR, enable_dtx=True) for _ in range(n)]
    sizes_seen = set()
    for f in range(frames):
        speech = wav[320 * (f + 20):320 * (f + 21)]
        pcm = np.stack([speech, np.zeros(320, np.int16), speech if f >= frames // 2 else np.zeros(320, np.int16)])
        pk, sizes = ctx.encode_dtx(pcm, bits, stream_ids=ids)
        for k in range(n):
            want = encs[k].encode(pcm[k], bits)
            assert sizes[k] == len(want), (f, k, sizes[k], len(want))
            assert bytes(pk[k][:sizes[k]]) == want
            if sizes[k] == 0:
                assert not pk[k].any()
            sizes_seen.add(int(sizes[k]))
    assert sizes_seen == {0, (bits + 7) // 8}
    ctx.close()


def run_resampler_parity(Context, api, O, *, seed=12):
    """lyra_b200_resample vs the oracle's Resampler: every supported pair, both directions, ragged chunk sizes (phase and delay line
    carry over between calls), several streams with different histories, a rate switch; int16 output bit for bit."""
    ctx = Context(8, capi=api)
    rng = np.random.default_rng(seed)
    ids = np.array([0, 3, 5], dtype=np.int32)
    for rate in (8000, 32000, 48000):
        for to_internal in (True, False):
            a, b = (rate, 16000) if to_internal else (16000, rate)
            refs = [O.Resampler(a, b) for _ in ids]
            ctx.reset()
            for chunk in (a // 50, 1, 7, a // 50 - 3, 2, a // 50):
                x = rng.integers(-30000, 30000, size=(len(ids), chunk)).astype(np.int16)
                got = ctx.resample(x, rate, to_internal, stream_ids=ids)
                for k in range(len(ids)):
                    want = refs[k].resample(x[k])
                    assert np.array_equal(got[k], want), (rate, to_internal, chunk, k, len(got[k]), len(want))
    # a stream that switches rate restarts from the fully primed state
    x = rng.integers(-30000, 30000, size=(1, 160)).astype(np.int16)
    ctx.resample(x, 8000, True, stream_ids=[2])
    y = rng.integers(-30000, 30000, size=(1, 960)).astype(np.int16)
    got = ctx.resample(y, 48000, True, stream_ids=[2])
    assert np.array_equal(got[0], O.Resampler(48000, 16000).resample(y[0]))
    ctx.close()


def run_integration_other_rates(Context, api, O, *, rate, wav, bits=64, hops=60):
    """lyra_integration_test.cc:60-149 at an external rate of 8 / 32 / 48 kHz through the batched C ABI: resample to 16 kHz, encode,
    decode, resample back; the log-mel spectra (64 bins at the external rate, the oracle's extractor) of input and output stay
    within LSD 2.0 on every hop once the filters are primed."""
    hop = rate // 50
    ctx = Context(2, capi=api)
    ie, oe = O.LogMel(rate, hop, 2 * hop, 64), O.LogMel(rate, hop, 2 * hop, 64)
    worst = 0.0
    outs = []
    for f in range(hops):
        x = wav[f * hop:(f + 1) * hop]
        internal = ctx.resample(x, rate, True, stream_ids=[1])[0]
        assert len(internal) == 320
        pk = ctx.encode(internal, bits, stream_ids=[1])
        dec = ctx.decode(pk, bits, stream_ids=[1])[0]
        y = ctx.resample(dec, rate, False, stream_ids=[1])[0]
        assert len(y) == hop
        outs.append(y)
    # the codec (one hop) and the two resamplers (17 + 17 * 16000 / rate ... samples) delay the output: compare hop f of the input
    # with hop f of the output like the reference does (its criterion tolerates the misalignment), skipping the priming hops
    for f in range(hops):
        fi = ie.extract(wav[f * hop:(f + 1) * hop])
        fo = oe.extract(outs[f])
        if f >= 3:
            worst = max(worst, O.log_spectral_distance(fi, fo))
    ctx.close()
    return worst


# ---- the device-resident entry points (lyra_b200_*_device, lyra_b200_set_stream) ----

class HostMem:
    """Device buffers of the emulated library: cudaMalloc returns host memory there, so numpy arrays stand in for device
    memory and pointers are their addresses.  The GPU tier passes an equivalent built on torch CUDA tensors."""
    stream = None           # the emulator has no streams to install

    def zeros(self, shape, dtype):
        return np.zeros(shape, dtype)

    def ptr(self, buf):
        return buf.ctypes.data

    def put(self, buf, a):
        buf[...] = a

    def get(self, buf):
        return np.array(buf)


GUARD_ROWS = 3


class Guarded:
    """A caller buffer of n rows with GUARD_ROWS rows of a sentinel byte on each side: `ptr` is the address of row 0.  put()
    rewrites the sentinels, get() checks that no call wrote outside rows [0, n).  fill() sets the n rows to the sentinel too,
    so an output row that a call fails to write does not silently keep an earlier, correct value."""

    def __init__(self, mem, n, row, dtype, sentinel):
        self.mem, self.n = mem, n
        self.shape = (n + 2 * GUARD_ROWS,) + tuple(row)
        self.row_bytes = int(np.prod(row, dtype=np.int64)) * np.dtype(dtype).itemsize
        self.sentinel = np.frombuffer(np.array([sentinel] * np.dtype(dtype).itemsize, np.uint8).tobytes(), dtype)[0]
        self.dtype = dtype
        self.buf = mem.zeros(self.shape, dtype)
        self.fill()

    @property
    def ptr(self):
        return self.mem.ptr(self.buf) + GUARD_ROWS * self.row_bytes

    def put(self, a=None):
        full = np.full(self.shape, self.sentinel, self.dtype)
        if a is not None:
            full[GUARD_ROWS:GUARD_ROWS + self.n] = a
        self.mem.put(self.buf, full)

    def fill(self):
        self.put(None)

    def get(self, what="buffer"):
        a = self.mem.get(self.buf)
        g = GUARD_ROWS
        assert (a[:g] == self.sentinel).all() and (a[g + self.n:] == self.sentinel).all(), \
            "a call wrote outside rows [0, %d) of the caller's %s" % (self.n, what)
        return a[g:g + self.n]


def _device_case_pcm(wav, n, f, frames):
    """Hop f of the device-entry-point case: speech for streams k % 3 == 0, digital silence for the first half then speech for
    k % 3 == 1, speech then silence for k % 3 == 2 (so DTX, the noise branch of the estimators and a restart from DTX all run)."""
    pcm = np.stack([wav[(320 * (f + 13 * k + 20)) % (len(wav) - 320):][:320] for k in range(n)]).copy()
    for k in range(n):
        if (k % 3 == 1 and f < frames // 2) or (k % 3 == 2 and f >= frames // 2):
            pcm[k] = 0
    return pcm


def run_device_parity(Context, api, O, mem, wav, *, n, frames, check, decoder_mode="exact", split=None, cng_seed=11, seed=3):
    """Every *_device entry point against its host-buffer twin on a second context (all n streams), and a sample of streams
    (`check`) against the oracle, hop by hop.  The device contexts run on mem.stream when there is one (lyra_b200_set_stream),
    their inputs and outputs are caller buffers with guard rows (Guarded), outputs are pre-filled with a sentinel.
    Covered: encode / decode with and without a received mask and with a bit-rate change between hops; decode_track_noise
    (PCM, is_noise, the estimate read back at the end); noise_update with and without a mask, in an encoder-only context;
    decode_plc with bursts long enough to reach comfort noise (PCM, flags, control state); encode_dtx over speech and silence
    (empty-packet flags, zeroed bytes, the encoder state held on DTX hops).  n need not be a multiple of the tile size.
    Bar: twins bit-exact in both decoder modes; oracle bit-exact, decoded PCM within TENSOR_PCM_TOL_LSB in the tensor mode."""
    tol = TENSOR_PCM_TOL_LSB if decoder_mode == "tensor" else 0
    exact = decoder_mode == "exact"
    roles = dict(enc="encoder", dec="decoder", trk="decoder", plc="decoder", dtx="encoder", nz="encoder")
    dev = {k: Context(n, capi=api, roles=r) for k, r in roles.items()}
    host = {k: Context(n, capi=api, roles=r) for k, r in roles.items()}
    for k in ("dec", "trk", "plc"):
        dev[k].set_decoder_mode(decoder_mode)
        host[k].set_decoder_mode(decoder_mode)
    dev["plc"].set_cng_seed(cng_seed)
    host["plc"].set_cng_seed(cng_seed)
    for c in dev.values():
        if split is not None:
            c.set_split(split)
        if mem.stream is not None:
            c.set_stream(mem.stream)
    G = lambda row, dtype, s: Guarded(mem, n, row, dtype, s)     # noqa: E731
    d_pcm, d_zero = G((320,), np.int16, 0x3C), G((320,), np.int16, 0x3C)
    d_rec, d_plc_rec, d_nz_mask = G((), np.uint8, 0xC3), G((), np.uint8, 0xC3), G((), np.uint8, 0xC3)
    d_out, d_trk_out, d_plc_out = G((320,), np.int16, 0x5A), G((320,), np.int16, 0x5A), G((320,), np.int16, 0x5A)
    d_trk_flags, d_cn, d_nz_flags, d_dtx_flags = (G((), np.uint8, 0xAA) for _ in range(4))
    d_est = G((160,), np.float32, 0x7F)
    d_zero.put(np.zeros((n, 320), np.int16))
    codecs = {k: O.Codec(MODEL_DIR) for k in check}
    trk_est = {k: O.NoiseEstimator() for k in check}
    nz_est = {k: O.NoiseEstimator() for k in check}
    plc_dec = {k: O.Decoder(MODEL_DIR, cng_seed=cng_seed + k) for k in check}
    dtx_enc = {k: O.Encoder(MODEL_DIR, enable_dtx=True) for k in check}
    rng = np.random.default_rng(seed)
    burst = [(1 + k % 3, 8 if k % 2 == 0 else 2) for k in range(n)]      # (first lost hop, length) of each stream's outage
    seen_dtx, seen_cn = set(), False
    for f in range(frames):
        bits = (64, 120, 184)[(f // 3) % 3]                               # the bit rate changes every third hop
        P = (bits + 7) // 8
        pcm = _device_case_pcm(wav, n, f, frames)
        d_pcm.put(pcm)
        # encode_device / decode_device (received mask on odd hops only: NULL = all received); the decoders read the packets
        # where the encoder wrote them
        d_pk, d_dtx_pk = G((P,), np.uint8, 0xA5), G((P,), np.uint8, 0xFF)
        d_out.fill()
        dev["enc"].encode_device(n, d_pcm.ptr, bits, d_pk.ptr)
        rec = None
        if f % 2:          # random, not periodic: a sub-batch that read another part's mask rows must see a different mask
            rec = (rng.random(n) >= 0.25).astype(np.uint8)
            d_rec.put(rec)
        dev["dec"].decode_device(n, d_pk.ptr, d_rec.ptr if rec is not None else 0, bits, d_out.ptr)
        pk = host["enc"].encode(pcm, bits)
        out = host["dec"].decode(pk, bits, received=rec)
        pk_rows = d_pk.get("packets")
        assert np.array_equal(pk_rows, pk), "encode_device != encode, hop %d" % f
        assert np.array_equal(d_out.get("PCM"), out), "decode_device != decode, hop %d" % f
        # decode_track_noise_device (same packets and mask)
        d_trk_out.fill()
        d_trk_flags.fill()
        dev["trk"].decode_track_noise_device(n, d_pk.ptr, d_rec.ptr if rec is not None else 0, bits, d_trk_out.ptr, d_trk_flags.ptr)
        t_out, t_flags = host["trk"].decode_track_noise(pk, bits, received=rec)
        assert np.array_equal(d_trk_out.get("PCM"), t_out), "decode_track_noise_device PCM != twin, hop %d" % f
        assert np.array_equal(d_trk_flags.get("is_noise"), t_flags.astype(np.uint8)), "is_noise != twin, hop %d" % f
        # noise_update_device in an encoder-only context (mask on even hops)
        mask = (rng.random(n) < 0.8).astype(np.uint8) if f % 2 == 0 else None
        if mask is not None:
            d_nz_mask.put(mask)
        d_nz_flags.fill()
        d_est.fill()
        dev["nz"].noise_update_device(n, d_pcm.ptr, d_nz_mask.ptr if mask is not None else 0, d_nz_flags.ptr, d_est.ptr)
        nz_flags, nz_est_h = host["nz"].noise_update(pcm, update_mask=mask)
        assert np.array_equal(d_nz_flags.get("is_noise"), nz_flags.astype(np.uint8)), "noise_update_device flags != twin, hop %d" % f
        assert np.array_equal(d_est.get("estimate"), nz_est_h), "noise_update_device estimate != twin, hop %d" % f
        # decode_plc_device: bursts of 8 lost hops (concealment -> fade -> comfort noise -> fade back) and of 2
        plc_rec = np.array([0 if b0 <= f < b0 + bl else 1 for b0, bl in burst], dtype=np.uint8)
        d_plc_rec.put(plc_rec)
        d_plc_out.fill()
        d_cn.fill()
        dev["plc"].decode_plc_device(n, d_pk.ptr, d_plc_rec.ptr, bits, d_plc_out.ptr, d_cn.ptr)
        p_out, p_cn = host["plc"].decode_plc(pk, bits, received=plc_rec)
        assert np.array_equal(d_plc_out.get("PCM"), p_out), "decode_plc_device PCM != twin, hop %d" % f
        assert np.array_equal(d_cn.get("flags"), p_cn.astype(np.uint8)), "decode_plc_device flags != twin, hop %d" % f
        st = dev["plc"].plc_state(n)
        assert np.array_equal(st, host["plc"].plc_state(n)), "control state != twin, hop %d" % f
        seen_cn |= bool(p_cn.any())
        # encode_dtx_device (its packet buffer starts as 0xFF bytes: the empty packets' zeros are written by the call)
        d_dtx_flags.fill()
        dev["dtx"].encode_dtx_device(n, d_pcm.ptr, bits, d_dtx_pk.ptr, d_dtx_flags.ptr)
        x_pk, x_sizes = host["dtx"].encode_dtx(pcm, bits)
        got_flags = d_dtx_flags.get("empty-packet flags")
        got_pk = d_dtx_pk.get("packets")
        assert np.array_equal(got_flags, (x_sizes == 0).astype(np.uint8)), "encode_dtx_device flags != twin, hop %d" % f
        assert np.array_equal(got_pk, x_pk), "encode_dtx_device packets != twin, hop %d" % f
        assert not got_pk[got_flags == 1].any(), "an empty packet's bytes must be zero"
        seen_dtx |= set(int(x) for x in got_flags)
        for k in check:
            opkt, _, _ = codecs[k].encode(pcm[k], bits)
            assert bytes(pk_rows[k]) == opkt, "packet != oracle, hop %d stream %d" % (f, k)
            lost = rec is not None and rec[k] == 0
            opcm, _, _ = codecs[k].decode(None if lost else opkt, bits)
            for name, got in (("decode_device", out[k]), ("decode_track_noise_device", t_out[k])):
                d = int(np.abs(got.astype(int) - opcm.astype(int)).max())
                assert d <= tol, "%s PCM != oracle, hop %d stream %d: max |d| %d" % (name, f, k, d)
            if exact:            # in the tensor mode the estimator is fed PCM that may differ by a few LSB: twins only
                if not lost:
                    trk_est[k].receive_samples(opcm)
                assert bool(t_flags[k]) == trk_est[k].is_noise, "track is_noise != oracle, hop %d stream %d" % (f, k)
            if mask is None or mask[k]:
                nz_est[k].receive_samples(pcm[k])
            assert bool(nz_flags[k]) == nz_est[k].is_noise and np.array_equal(nz_est_h[k], nz_est[k].noise_estimate()), \
                "noise_update != oracle, hop %d stream %d" % (f, k)
            if plc_rec[k]:
                assert plc_dec[k].set_encoded_packet(opkt)
            want = plc_dec[k].decode_samples(320)
            d = int(np.abs(p_out[k].astype(int) - want.astype(int)).max())
            assert d <= tol, "decode_plc PCM != oracle, hop %d stream %d: max |d| %d" % (f, k, d)
            assert tuple(int(x) for x in st[k]) == plc_dec[k].state and bool(p_cn[k]) == plc_dec[k].is_comfort_noise(), (f, k)
            want = dtx_enc[k].encode(pcm[k], bits)
            assert x_sizes[k] == len(want) and bytes(x_pk[k][:x_sizes[k]]) == want, "encode_dtx != oracle, hop %d stream %d" % (f, k)
        d_pcm.get("input PCM")                   # inputs are read only
    assert seen_dtx == {0, 1}, "the case must produce both DTX and encoded hops"
    assert seen_cn, "the case never reached comfort noise"
    # the tracked estimates, read back through noise_update_device without feeding (mask all zero)
    d_nz_mask.put(np.zeros(n, np.uint8))
    d_est.fill()
    d_trk_flags.fill()
    dev["trk"].noise_update_device(n, d_zero.ptr, d_nz_mask.ptr, d_trk_flags.ptr, d_est.ptr)
    h_flags, h_est = host["trk"].noise_update(np.zeros((n, 320), np.int16), update_mask=np.zeros(n, np.uint8))
    est = d_est.get("estimate")
    assert np.array_equal(est, h_est) and np.array_equal(d_trk_flags.get("is_noise"), h_flags.astype(np.uint8))
    if exact:
        for k in check:
            assert np.array_equal(est[k], trk_est[k].noise_estimate()), "tracked estimate != oracle, stream %d" % k
    for c in list(dev.values()) + list(host.values()):
        c.close()
