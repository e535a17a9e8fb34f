"""GPU tier (H100): parity tests proper, through the C ABI of the nvcc-built library, against the oracle on the
same seeded inputs; plus size-independent properties at BASELINE.json's full sizes."""
import json
import os
import sys

import numpy as np
import pytest

import parity_cases as pc
from conftest import GOLDEN_DIR, ROOT
from lyra_b200 import _capi

sys.path.insert(0, os.path.join(ROOT, "tools"))        # duplex_schedule

pytestmark = pytest.mark.gpu


class TorchMem:
    """Device buffers for the device-resident entry points: torch CUDA tensors, allocated, filled and read on one torch stream
    of their own, which is also the stream the cases install in their contexts (lyra_b200_set_stream) - so every copy and every
    library call is ordered on that stream and reading a result back needs no other synchronisation.  (Not the default stream:
    its handle is 0, which lyra_b200_set_stream takes as "the context's own stream".)"""

    def __init__(self):
        import torch
        self.torch = torch
        self.s = torch.cuda.Stream()
        self.stream = self.s.cuda_stream

    def zeros(self, shape, dtype):
        with self.torch.cuda.stream(self.s):
            return self.torch.zeros(shape, dtype=getattr(self.torch, np.dtype(dtype).name), device="cuda")

    def ptr(self, t):
        return t.data_ptr()

    def put(self, t, a):
        with self.torch.cuda.stream(self.s):
            t.copy_(self.torch.from_numpy(np.ascontiguousarray(a)))

    def get(self, t):
        with self.torch.cuda.stream(self.s):
            return t.cpu().numpy()


def test_codec_parity_speech_with_loss(gpu_api, oracle, sample1):
    pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=100, stream_ids=[0, 5, 17, 31, 32, 64, 99],
                        frames=60, bits=64, wav=sample1, loss_every=6)


@pytest.mark.parametrize("bits", [64, 120, 184])
def test_codec_parity_noise_all_bitrates(gpu_api, oracle, bits):
    pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=48, stream_ids=list(range(48)), frames=25, bits=bits,
                        seed=bits, check=[0, 1, 15, 16, 33, 47])


@pytest.mark.parametrize("kind", ["loud", "silence"])
def test_codec_parity_extreme_inputs(gpu_api, oracle, kind):
    pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=16, stream_ids=[3, 4, 9], frames=12, bits=120, kind=kind)


@pytest.mark.parametrize("kind", ["speech", "noise", "loud"])
def test_tensor_decoder_mode_within_tolerance(gpu_api, oracle, sample1, kind):
    # opt-in split-precision TF32 decoder: packets stay bit-exact, PCM within TENSOR_PCM_TOL_LSB of the oracle
    worst = pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=40, stream_ids=[0, 7, 8, 21, 39], frames=60,
                                bits=64 if kind != "loud" else 184, wav=sample1 if kind == "speech" else None,
                                kind="noise" if kind == "speech" else kind, loss_every=9, decoder_mode="tensor", seed=5)
    print("tensor-mode decoder, %s: worst |PCM - oracle| = %d LSB" % (kind, worst))
    assert worst <= pc.TENSOR_PCM_TOL_LSB


def test_tensor_decoder_mode_full_size_matches_exact_mode(gpu_api):
    # 4096 streams x 20 frames: the tensor-mode PCM stays within the tolerance of the exact-mode PCM on every stream
    n = 4096
    rng = np.random.default_rng(11)
    a = _capi.Context(n, capi=gpu_api)
    b = _capi.Context(n, capi=gpu_api)
    b.set_decoder_mode("tensor")
    worst = 0
    for f in range(20):
        pcm = pc.synth_pcm(rng, n, "noise")
        pk = a.encode(pcm, 64)
        assert np.array_equal(pk, b.encode(pcm, 64))
        worst = max(worst, int(np.abs(a.decode(pk, 64).astype(int) - b.decode(pk, 64).astype(int)).max()))
    a.close()
    b.close()
    print("tensor vs exact decoder, 4096 streams: worst |dPCM| = %d LSB" % worst)
    assert worst <= pc.TENSOR_PCM_TOL_LSB


def test_priority_switch(gpu_api, oracle):
    # lyra_b200_set_priority re-creates the context's streams between hops; state and results are unaffected
    pc.run_priority_switch(_capi.Context, gpu_api, oracle, n=20, frames=8)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_sparse_tiles_with_loss(gpu_api, oracle, sample1, mode):
    # stream ids 0 / 15 / 16 / 33 / 39 fall in tiles 0, 1, 2 and 4: sparse calls whose tiles hold one or two active streams
    pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=40, stream_ids=[0, 15, 16, 33, 39], frames=24, bits=120,
                        wav=sample1, loss_every=5, decoder_mode=mode)


def test_bitrate_switch_mid_stream(gpu_api, oracle):
    # LyraEncoder::set_bitrate (lyra/lyra_encoder.cc:158-167): the number of quantized bits may change from hop to hop
    n, ids = 3, np.array([1, 8, 9], dtype=np.int32)
    ctx = _capi.Context(16, capi=gpu_api)
    from conftest import MODEL_DIR
    codecs = [oracle.Codec(MODEL_DIR) for _ in range(n)]
    rng = np.random.default_rng(3)
    for f, bits in enumerate([64, 184, 120, 64, 120, 184, 64, 64]):
        pcm = pc.synth_pcm(rng, n)
        pk = ctx.encode(pcm, bits, stream_ids=ids)
        out = ctx.decode(pk, bits, stream_ids=ids)
        for k in range(n):
            opkt, _, _ = codecs[k].encode(pcm[k], bits)
            opcm, _, _ = codecs[k].decode(opkt, bits)
            assert bytes(pk[k]) == opkt and np.array_equal(out[k], opcm), (f, bits, k)
    ctx.close()


def test_non_standard_bit_counts(gpu_api, oracle):
    # any multiple of 4 up to 184 is accepted by Quantize (residual_vector_quantizer.cc:79-89)
    for bits in (4, 60, 100, 180):
        pc.run_codec_parity(_capi.Context, gpu_api, oracle, max_streams=4, stream_ids=[2], frames=2, bits=bits, seed=bits)


def test_plugin_surface(gpu_api, oracle):
    pc.run_plugin_surface_parity(_capi.Context, gpu_api, oracle, n=9, frames=4)


def test_reset_and_isolation(gpu_api, oracle):
    pc.run_reset_and_isolation(_capi.Context, gpu_api, oracle)


def test_reset_restores_every_stream_state(gpu_api, sample1):
    pc.run_reset_restores_every_stream_state(_capi.Context, gpu_api, sample1, max_streams=64, ids=(1, 6, 9, 14, 33, 40, 63),
                                             reset_ids=(40, 9, 1, 9), dense_n=16)


def test_reset_across_launch_chunks(gpu_api, sample1):
    # reset launches one copy kernel per 1024 streams: ids on both sides of the chunk edges at 1024 and 2048
    pc.run_reset_restores_every_stream_state(_capi.Context, gpu_api, sample1, max_streams=2112, ids=(5, 1030, 2050, 2100),
                                             reset_ids=(2050, 5, 2050), dense_n=2060, dense_launches=3)


def test_error_paths(gpu_api):
    pc.run_error_paths(_capi.Context, gpu_api, _capi.LyraB200Error)


def test_logmel(gpu_api, oracle, sample1):
    pc.run_logmel_parity(_capi.Context, gpu_api, oracle, sample1, n=6, frames=8)


def test_noise_estimator(gpu_api, oracle, sample1):
    pc.run_noise_estimator_parity(_capi.Context, gpu_api, oracle, sample1, n=9, frames=120)


def test_decode_track_noise_sparse_and_dense(gpu_api, oracle, sample1):
    pc.run_decode_track_noise_parity(_capi.Context, gpu_api, oracle, sample1, stream_ids=[0, 3, 8, 30], max_streams=32, frames=40)
    # dense call over 1024 streams: cut into two concurrent sub-batches, each followed by its own estimator update
    pc.run_decode_track_noise_parity(_capi.Context, gpu_api, oracle, sample1, n=1024, frames=8, check=[0, 7, 511, 512, 777, 1023])


def test_role_contexts(gpu_api, oracle):
    pc.run_role_contexts(_capi.Context, gpu_api, oracle, _capi.LyraB200Error, TorchMem(), frames=20)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_schedule_independence_full_size(gpu_api, mode):
    # 4096 streams x 24 frames: the result may not depend on how the call is cut into concurrent sub-batches, on the number
    # of resident blocks the scheduler mixes, or on encoder and decoder living in separate contexts
    n = 4096
    rng = np.random.default_rng(21)
    ref = _capi.Context(n, capi=gpu_api)
    ref.set_split(1)
    ref.set_decoder_mode(mode)
    alt = _capi.Context(n, capi=gpu_api)
    alt.set_split(3)
    alt.set_decoder_mode(mode)
    enc = _capi.Context(n, capi=gpu_api, roles="encoder")
    dec = _capi.Context(n, capi=gpu_api, roles="decoder")
    dec.set_decoder_mode(mode)
    enc.set_split(2)
    dec.set_split(4)
    for f in range(24):
        pcm = pc.synth_pcm(rng, n, "noise" if f % 5 else "loud")
        bits = (64, 120, 184)[f % 3]
        received = (rng.random(n) < 0.9).astype(np.uint8)
        pk = ref.encode(pcm, bits)
        out = ref.decode(pk, bits, received=received)
        assert np.array_equal(pk, alt.encode(pcm, bits)) and np.array_equal(pk, enc.encode(pcm, bits)), f
        assert np.array_equal(out, alt.decode(pk, bits, received=received)), f
        assert np.array_equal(out, dec.decode(pk, bits, received=received)), f
    for c in (ref, alt, enc, dec):
        c.close()


@pytest.mark.parametrize("n", [64, 1024])
def test_cuda_graphs_replay_matches_direct_calls(gpu_api, n):
    # lyra_b200_set_graphs: dense host-buffer calls on page-locked buffers replay a captured graph; the streaming state must
    # advance exactly as with directly issued calls (30 hops, two rotating buffer pairs, loss masks, a change of bit rate)
    import ctypes as C

    import torch
    rng = np.random.default_rng(5)
    ref = _capi.Context(n, capi=gpu_api)
    gr = _capi.Context(n, capi=gpu_api)
    gr.set_graphs(True)
    lib = gpu_api.lib
    pin_pcm = [torch.zeros((n, 320), dtype=torch.int16).pin_memory() for _ in range(2)]
    pin_pk = [torch.zeros((n, 23), dtype=torch.uint8).pin_memory() for _ in range(2)]
    pin_rec = [torch.zeros(n, dtype=torch.uint8).pin_memory() for _ in range(2)]
    pin_out = torch.zeros((n, 320), dtype=torch.int16).pin_memory()

    def p(t):
        return C.c_void_p(t.data_ptr())
    for f in range(30):
        b = f % 2
        bits = 64 if f < 20 else 120
        pb = _capi.packet_bytes(bits)
        pcm = pc.synth_pcm(rng, n, "noise" if f % 4 else "loud")
        received = (rng.random(n) < 0.85).astype(np.uint8)
        pk = ref.encode(pcm, bits)
        out = ref.decode(pk, bits, received=received)
        pin_pcm[b].numpy()[:] = pcm
        pin_rec[b].numpy()[:] = received
        assert lib.lyra_b200_encode(gr.h, None, n, p(pin_pcm[b]), bits, p(pin_pk[b])) == 0
        got_pk = pin_pk[b].numpy().reshape(-1)[: n * pb].reshape(n, pb)
        assert np.array_equal(pk, got_pk), f
        assert lib.lyra_b200_decode(gr.h, None, n, p(pin_pk[b]), p(pin_rec[b]), bits, p(pin_out)) == 0
        assert np.array_equal(out, pin_out.numpy()), f
    # 30 encode + 30 decode calls over 2 buffer pairs and 2 bit rates: 4 + 4 captures, every other call is a replay
    assert gr.graph_replays() >= 40, gr.graph_replays()
    assert ref.graph_replays() == 0
    # pageable host buffers (the ctypes wrappers allocate with numpy) cannot be captured: the call must run directly, same results
    replays = gr.graph_replays()
    pcm = pc.synth_pcm(rng, n, "noise")
    pk = ref.encode(pcm, 64)
    assert np.array_equal(pk, gr.encode(pcm, 64)) and np.array_equal(ref.decode(pk, 64), gr.decode(pk, 64))
    assert gr.graph_replays() == replays
    gr.set_graphs(False)
    pcm = pc.synth_pcm(rng, n, "noise")
    assert np.array_equal(ref.encode(pcm, 64), gr.encode(pcm, 64))
    ref.close()
    gr.close()


def test_golden_fixture_packets(gpu_api, sample1):
    """Committed fixtures (tests/golden/oracle_sample1.json): the GPU path reproduces them without the oracle present."""
    with open(os.path.join(GOLDEN_DIR, "oracle_sample1.json")) as f:
        g = json.load(f)
    ctx = _capi.Context(3, capi=gpu_api)
    for h in range(g["hops"]):
        x = np.tile(sample1[320 * h:320 * h + 320], (3, 1))
        for k, bits in enumerate((64, 120, 184)):
            pkt = ctx.encode(x[k:k + 1], bits, stream_ids=np.array([k], dtype=np.int32))
            assert bytes(pkt[0]).hex() == g["packets_%d" % bits][h], (bits, h)
            pcm = ctx.decode(pkt, bits, stream_ids=np.array([k], dtype=np.int32))
            assert int((pcm[0].astype(np.int64) * np.arange(1, 321)).sum()) == g["pcm_checksum_%d" % bits][h]
    ctx.close()


def test_integration_criterion_on_gpu(gpu_api, oracle, sample1):
    """lyra/lyra_integration_test.cc:132-142 on the GPU path: every hop's log-spectral distance < 2.0."""
    ctx = _capi.Context(3, capi=gpu_api)
    hops = 150
    worst = [0.0, 0.0, 0.0]
    for h in range(hops):
        x = sample1[320 * h:320 * h + 320]
        for k, bits in enumerate((64, 120, 184)):
            ids = np.array([k], dtype=np.int32)
            y = ctx.decode(ctx.encode(x[None], bits, stream_ids=ids), bits, stream_ids=ids)[0]
            a = ctx.logmel(x[None], num_mel_bins=64, bank=0, stream_ids=ids)[0]
            b = ctx.logmel(y[None], num_mel_bins=64, bank=1, stream_ids=ids)[0]
            worst[k] = max(worst[k], oracle.log_spectral_distance(a, b))
    assert max(worst) < 2.0, worst
    ctx.close()


@pytest.mark.parametrize("n,bits", [(1024, 64), (4096, 64), (4096, 120), (4096, 184)])
def test_full_size_properties(gpu_api, oracle, n, bits):
    """BASELINE configs 2/3 sizes.  Properties that need no per-stream oracle:
    (1) batch independence: streams fed the same audio produce identical packets/PCM wherever they sit in the batch;
    (2) a sample of streams with distinct audio matches the oracle bit for bit;
    (3) packet -> dequantize -> quantize is idempotent on the decoded features' indices."""
    ctx = _capi.Context(n, capi=gpu_api)
    rng = np.random.default_rng(n + bits)
    base = rng.integers(-8192, 8192, size=(6, 320), dtype=np.int16)
    distinct = sorted(set([7, 100, n // 2 + 1, n - 2]))
    refs = {k: oracle.Codec(_capi.MODEL_DIR) for k in distinct}
    same_ref = oracle.Codec(_capi.MODEL_DIR)
    for f in range(6):
        pcm = np.tile(base[f], (n, 1))
        other = rng.integers(-8192, 8192, size=(len(distinct), 320), dtype=np.int16)
        for j, k in enumerate(distinct):
            pcm[k] = other[j]
        pk = ctx.encode(pcm, bits)
        out = ctx.decode(pk, bits)
        same = np.array([k for k in range(n) if k not in distinct])
        assert (pk[same] == pk[same[0]]).all()
        assert (out[same] == out[same[0]]).all()
        opkt, _, _ = same_ref.encode(base[f], bits)
        opcm, _, _ = same_ref.decode(opkt, bits)
        assert bytes(pk[same[0]]) == opkt and np.array_equal(out[same[-1]], opcm)
        for j, k in enumerate(distinct):
            opkt, _, _ = refs[k].encode(pcm[k], bits)
            opcm, _, _ = refs[k].decode(opkt, bits)
            assert bytes(pk[k]) == opkt and np.array_equal(out[k], opcm)
        feats = ctx.dequantize(pk[:64], bits)
        assert (ctx.quantize(feats, 4)[:, 0] >> 4 == pk[:64, 0] >> 4).all()     # first-stage index is a fixed point
    ctx.close()


def test_decoder_only_concealment_4096(gpu_api, oracle):
    """BASELINE config 4 (decoder-only PLC path): no packets at all, then Bernoulli(0.9) reception."""
    n, bits = 4096, 64
    ctx = _capi.Context(n, capi=gpu_api)
    rng = np.random.default_rng(1234)
    check = [0, 77, 2048, 4095]
    refs = {k: oracle.Codec(_capi.MODEL_DIR) for k in check}
    mels = {k: oracle.LogMel(16000, 320, 640, 160) for k in check}
    pk = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    for f in range(5):
        rec = np.zeros(n, np.uint8) if f < 2 else (rng.random(n) < 0.9).astype(np.uint8)
        out = ctx.decode(pk, bits, received=rec)
        mel = ctx.logmel(out, num_mel_bins=160)                 # NoiseEstimator's extractor runs on every decoded hop
        assert np.isfinite(mel).all() and mel.shape == (n, 160)
        for k in check:
            assert np.array_equal(mel[k], mels[k].extract(out[k])), "log-mel mismatch frame %d stream %d" % (f, k)
        for k in check:
            opcm, _, _ = refs[k].decode(bytes(pk[k]) if rec[k] else None, bits)
            assert np.array_equal(out[k], opcm)
    ctx.close()


def test_cpp_components_against_oracle(gpu_api, oracle, tmp_path):
    """include/lyra_b200/lyra_b200_components.h: the reference's plugin classes re-hosted on the C ABI (C++)."""
    import subprocess
    from conftest import ROOT
    exe = str(tmp_path / "test_components")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "oracle"),
                           os.path.join(ROOT, "tests", "cpp", "test_components.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "lyra_b200"), "-llyra_b200", "-L" + os.path.join(ROOT, "oracle", "_build"), "-llyra_oracle",
                           "-Wl,-rpath," + os.path.join(ROOT, "lyra_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle", "_build"), "-lpthread"])
    env = dict(os.environ, LYRA_B200_MAX_STREAMS="64")
    out = subprocess.run([exe, _capi.MODEL_DIR], capture_output=True, text=True, env=env)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr


def test_cpp_duplex_server_example(gpu_api, oracle, tmp_path):
    """examples/duplex_server.cc on the GPU: checksum of the decoded audio against the oracle (small), then a full-size run."""
    import subprocess
    from conftest import MODEL_DIR, ROOT
    exe = str(tmp_path / "duplex_server")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "duplex_server.cc"),
                           "-o", exe, "-L" + os.path.join(ROOT, "lyra_b200"), "-llyra_b200", "-Wl,-rpath," + os.path.join(ROOT, "lyra_b200"), "-lpthread"])
    streams, steps = 16, 5

    def hop(stream, step):          # FillHop of the example
        x = (2463534242 ^ (stream * 7919 + step * 104729)) & 0xFFFFFFFF
        out = np.empty(320, dtype=np.int16)
        for i in range(320):
            x = (x * 1664525 + 1013904223) & 0xFFFFFFFF
            out[i] = ((x >> 16) & 16383) - 8192
        return out

    want = 0
    for s in range(streams):
        c = oracle.Codec(MODEL_DIR)
        for i in range(steps):
            pkt, _, _ = c.encode(hop(s, i), 120)
            pcm, _, _ = c.decode(pkt, 120)
        want += int(pcm.astype(np.int64).sum())
    out = subprocess.run([exe, MODEL_DIR, str(streams), str(steps), "2", "120"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert int(out.stdout.strip().rsplit("checksum", 1)[1]) == want, out.stdout
    big = subprocess.run([exe, MODEL_DIR, "4096", "60", "2", "64"], capture_output=True, text=True, timeout=300)
    assert big.returncode == 0, big.stdout + big.stderr
    print(big.stdout.strip())


def test_wgmma_probe_on_hardware(tmp_path):
    """tests/cpp/wgmma_probe.cu built with nvcc: the wgmma instruction sequences of device_compat.h that the product's tensor-core
    decoder kernel (DecoderKernelDW) is made of - shared-memory descriptors, register A operands, fragment layouts, split-precision
    TF32 MMAs, the accumulator-to-operand shuffle.  The product depends on them: a mismatch is a failure."""
    import subprocess
    import __graft_entry__ as g
    from conftest import ROOT
    exe = str(tmp_path / "wgmma_probe")
    subprocess.check_call([g.NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I" + os.path.join(ROOT, "lyra_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "wgmma_probe.cu")])
    out = subprocess.run(["timeout", "60", exe], capture_output=True, text=True, timeout=120)
    print(out.stdout.strip())
    assert out.returncode == 0 and out.stdout.count("MATCH") == 2 and "MISMATCH" not in out.stdout, out.stdout + out.stderr


# ---- packet-loss concealment, comfort noise, DTX (SURVEY.md section 8 rows f2, f4) ----

def test_comfort_noise_generator_parity(gpu_api, oracle):
    pc.run_cng_parity(_capi.Context, gpu_api, oracle, stream_ids=(0, 5, 63, 64), hops=12)


def test_comfort_noise_reference_criterion_on_gpu(gpu_api, oracle):
    """comfort_noise_generator_test.cc:100-138 on the GPU path: log-mel of the generated noise within LSD 0.7 of its conditioning."""
    ctx = _capi.Context(8, capi=gpu_api)
    ctx.set_cng_seed(1)
    rng = np.random.default_rng(1)
    x = rng.integers(-10000, 10001, size=(8, 320)).astype(np.int16)
    for _ in range(10):
        fi = ctx.logmel(x, 160, bank=0)
        fo = ctx.logmel(ctx.cng_generate(fi), 160, bank=1)
    lsd = [oracle.log_spectral_distance(fi[k], fo[k]) for k in range(8)]
    print("CNG log-spectral distance per stream:", ["%.3f" % v for v in lsd])
    assert max(lsd) < 0.7
    ctx.close()


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_plc_state_machine_parity(gpu_api, oracle, sample1, mode):
    pc.run_plc_parity(_capi.Context, gpu_api, oracle, max_streams=64, stream_ids=(1, 6, 9, 40, 63), frames=40, wav=sample1,
                      outages=((3, 12), (5, 3), (0, 0), (10, 25), (20, 7)), decoder_mode=mode)
    if mode == "exact":
        pc.run_plc_state_peer(_capi.Context, gpu_api, oracle)


def test_plc_full_size_bernoulli_loss(gpu_api, oracle):
    """BASELINE configs[3] with the reference's real state machine: 4096 streams, burst losses; a few streams are checked against
    the oracle, all of them against the invariants of the state machine."""
    n, bits = 4096, 64
    ctx = _capi.Context(n, capi=gpu_api)
    ctx.set_cng_seed(21)
    rng = np.random.default_rng(1234)
    check = [0, 77, 2048, 4095]
    decs = {k: oracle.Decoder(_capi.MODEL_DIR, cng_seed=21 + k) for k in check}
    pk = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    burst = np.zeros(n, dtype=np.int32)
    cn_hops = 0
    for f in range(24):
        start = (rng.random(n) < 0.08) & (burst == 0)
        burst[start] = rng.integers(1, 12, size=int(start.sum()))
        rec = (burst == 0).astype(np.uint8)
        burst = np.maximum(burst - 1, 0)
        out, cn = ctx.decode_plc(pk, bits, received=rec)
        st = ctx.plc_state(n)
        assert ((st[:, 0] % 320 == 0) & (st[:, 0] >= 0) & (st[:, 0] <= 1280)).all()
        assert np.isin(st[:, 1], [0, 320, 640]).all() and np.isin(st[:, 2], [-1, 1]).all()
        assert (st[rec == 1, 0] == 0).all()                      # a received packet always ends concealment
        assert (cn == (st[:, 1] == 640)).all()
        cn_hops += int(cn.sum())
        for k in check:
            if rec[k]:
                assert decs[k].set_encoded_packet(bytes(pk[k]))
            assert np.array_equal(out[k], decs[k].decode_samples(320)), (f, k)
    assert cn_hops > 0
    ctx.close()


def test_dtx_encoder_parity(gpu_api, oracle, sample1):
    pc.run_dtx_parity(_capi.Context, gpu_api, oracle, wav=sample1, frames=40)


def test_resampler_parity(gpu_api, oracle):
    pc.run_resampler_parity(_capi.Context, gpu_api, oracle)


@pytest.mark.parametrize("rate", [8000, 32000, 48000])
def test_integration_criterion_other_sample_rates(gpu_api, oracle, rate):
    from conftest import read_wav_any
    wav = read_wav_any("sample1_%dkHz.wav" % (rate // 1000), rate)
    worst = pc.run_integration_other_rates(_capi.Context, gpu_api, oracle, rate=rate, wav=wav)
    print("integration LSD at %d Hz: worst hop %.3f" % (rate, worst))
    assert worst < 2.0


# ---- the device-resident entry points: the path bench.py times ----

@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_device_entry_points(gpu_api, oracle, sample1, mode):
    # every *_device call against its host-buffer twin (all 1100 streams) and the oracle; 1100 streams = 138 tiles, the last one
    # partial, and split 2 engages (>= 128 tiles): the check streams sit at the edges of both sub-batches
    pc.run_device_parity(_capi.Context, gpu_api, oracle, TorchMem(), sample1, n=1100, frames=12, check=[0, 551, 552, 1097, 1099],
                         decoder_mode=mode, split=2)


def _torch():
    import torch
    return torch


@pytest.mark.parametrize("workload,mode,split", [("codec", "exact", 2), ("codec", "tensor", 3),
                                                 ("decode_plc", "exact", 3), ("decode_plc", "tensor", 2)])
def test_bench_device_schedule(gpu_api, oracle, workload, mode, split):
    """bench.py's device-resident pass (measure -> run_device, as tools/duplex_schedule.py runs it) at a size where its
    sub-batches engage: G = 2 context pairs over slices of shared buffers, caller streams at priorities -1 / 0, encoder ->
    decoder events, 12 hops over 8 rotating slots queued with no host synchronisation.  2 x 1540 streams: 193 tiles per context,
    the last one partial, so a slice's last tile ends in the middle of the shared buffer.  Every hop's output goes to its own
    buffer; all streams are compared with host-buffer calls on a reference context per group, the streams at the slice edges
    with the oracle."""
    import duplex_schedule as ds
    plc = workload == "decode_plc"
    G, m, NBUF, hops, bits = 2, 1540, ds.NBUF, 12, 64
    n = G * m
    tol = pc.TENSOR_PCM_TOL_LSB if mode == "tensor" else 0
    rng = np.random.default_rng(17)
    host_pcm = [pc.synth_pcm(rng, n, "noise" if b % 4 else "loud") for b in range(NBUF)]
    edges = [0, m - 1, m, n - 1]
    if plc:
        # the workload's packets come from an encoder over the 8 input slots; bursts of 7 lost hops (slots 1..7) reach comfort
        # noise on every 5th stream and on the edge streams, the others lose packets at random
        tmp = _capi.Context(n, roles="encoder")
        h_pks = [tmp.encode(x, bits) for x in host_pcm]
        tmp.close()
        burst = np.zeros(n, bool)
        burst[::5] = True
        burst[edges] = True
        h_masks = [((rng.random(n) >= 0.15) & ~(burst & (b > 0))).astype(np.uint8) for b in range(NBUF)]
        sched = ds.Schedule(h_pks, G, split, mode, bits, masks=h_masks, keep_hops=hops)
    else:
        sched = ds.Schedule(host_pcm, G, split, mode, bits, keep_hops=hops)
    ds.run([sched], hops)
    _torch().cuda.synchronize()
    outs = [x.cpu().numpy() for x in sched.out]
    flags = [x.cpu().numpy() for x in sched.flags] if plc else None
    pks = None if plc else [x.cpu().numpy() for x in sched.kept_pks]
    # reference: one context per group (the comfort-noise seed of a stream is the context's seed plus its id in that context)
    refs = [(None if plc else _capi.Context(m, roles="encoder"), _capi.Context(m, roles="decoder")) for _ in range(G)]
    for _, rd in refs:
        rd.set_decoder_mode(mode)
    oracles = {s: (oracle.Decoder(_capi.MODEL_DIR, cng_seed=s % m) if plc else oracle.Codec(_capi.MODEL_DIR)) for s in edges}
    seen_cn = False
    for i in range(hops):
        b = i % NBUF
        for g, (re, rd) in enumerate(refs):
            sl = slice(g * m, (g + 1) * m)
            if plc:
                want, cn = rd.decode_plc(h_pks[b][sl], bits, received=h_masks[b][sl])
                assert np.array_equal(flags[i][sl], cn.astype(np.uint8)), (i, g)
                seen_cn |= bool(cn.any())
            else:
                pk = re.encode(host_pcm[b][sl], bits)
                assert np.array_equal(pks[i][sl], pk), "packets of hop %d group %d" % (i, g)
                want = rd.decode(pk, bits)
            bad = np.nonzero((outs[i][sl] != want).any(axis=1))[0]
            assert bad.size == 0, "PCM of hop %d group %d differs from host-buffer calls at streams %s" % (i, g, (bad + g * m)[:8])
        for s in edges:
            if plc:
                if h_masks[b][s]:
                    assert oracles[s].set_encoded_packet(bytes(h_pks[b][s]))
                opcm = oracles[s].decode_samples(320)
                assert bool(flags[i][s]) == oracles[s].is_comfort_noise(), (i, s)
            else:
                opkt, _, _ = oracles[s].encode(host_pcm[b][s], bits)
                assert bytes(pks[i][s]) == opkt, (i, s)
                opcm, _, _ = oracles[s].decode(opkt, bits)
            d = int(np.abs(outs[i][s].astype(int) - opcm.astype(int)).max())
            assert d <= tol, "hop %d stream %d: max |PCM - oracle| %d" % (i, s, d)
    assert not plc or seen_cn
    sched.close()
    for c in [c for r in refs for c in r]:
        if c is not None:
            c.close()


def _device_pairs(n, split):
    """One context per *_device entry point and its host-buffer twin, dense calls over n streams."""
    roles = dict(enc="encoder", dec="decoder", trk="decoder", nz="encoder", plc="decoder", dtx="encoder")
    dev = {k: _capi.Context(n, roles=r) for k, r in roles.items()}
    host = {k: _capi.Context(n, roles=r) for k, r in roles.items()}
    for c in dev.values():
        c.set_split(split)
    return dev, host


def test_device_calls_follow_the_caller_stream(gpu_api):
    """lyra_b200_set_stream: the calls read their inputs in stream order on the installed stream.  The caller stream fills the
    input buffer, makes the call, then at once overwrites the buffer with the next hop's input - no host synchronisation
    anywhere; a spin queued first keeps the caller stream far behind the host, so a call that read its input on any other stream
    would read it before it was written.  Results must be those of the un-overwritten inputs."""
    torch = _torch()
    n, bits, hops = 1024, 120, 4
    P = _capi.packet_bytes(bits)
    rng = np.random.default_rng(8)
    pcm = [pc.synth_pcm(rng, n) for _ in range(hops)]
    d_src = [torch.from_numpy(x).cuda() for x in pcm]
    trash = torch.from_numpy(pc.synth_pcm(rng, n, "loud")).cuda()
    enc = _capi.Context(n, roles="encoder")
    dec = _capi.Context(n, roles="decoder")
    ref = _capi.Context(n)
    s = torch.cuda.Stream()
    for c in (enc, dec):
        c.set_split(2)
        c.set_stream(s.cuda_stream)
    buf = torch.zeros((n, 320), dtype=torch.int16, device="cuda")
    pk_buf = torch.zeros((n, P), dtype=torch.uint8, device="cuda")
    pks = [torch.zeros((n, P), dtype=torch.uint8, device="cuda") for _ in range(hops)]
    outs = [torch.zeros((n, 320), dtype=torch.int16, device="cuda") for _ in range(hops)]
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        for f in range(hops):
            buf.copy_(d_src[f])
            enc.encode_device(n, buf.data_ptr(), bits, pks[f].data_ptr())
            buf.copy_(d_src[f + 1] if f + 1 < hops else trash)
            pk_buf.copy_(pks[f])
            dec.decode_device(n, pk_buf.data_ptr(), 0, bits, outs[f].data_ptr())
            pk_buf.zero_()
    s.synchronize()
    for f in range(hops):
        want_pk = ref.encode(pcm[f], bits)
        assert np.array_equal(pks[f].cpu().numpy(), want_pk), "encode_device read an overwritten input (hop %d)" % f
        assert np.array_equal(outs[f].cpu().numpy(), ref.decode(want_pk, bits)), "decode_device read overwritten packets (hop %d)" % f
    for c in (enc, dec, ref):
        c.close()


def test_device_calls_do_not_wait_for_the_gpu(gpu_api, sample1):
    """The *_device calls are asynchronous on the installed stream (include/lyra_b200.h, DESIGN.md section 4): with a spin of a
    few tens of ms queued ahead on the caller stream, every dense call returns while the stream is still busy.  Ordering only:
    the results, read after synchronising, equal the host-buffer twins'."""
    torch = _torch()
    n, bits = 1024, 64
    P = _capi.packet_bytes(bits)
    dev, host = _device_pairs(n, 2)
    s = torch.cuda.Stream()
    for c in dev.values():
        c.set_stream(s.cuda_stream)
    pcm = np.stack([sample1[(320 * (7 * k)) % (len(sample1) - 320):][:320] for k in range(n)]).copy()
    pcm[::3] = 0
    rec = (np.arange(n) % 5 != 0).astype(np.uint8)
    d_pcm, d_rec = torch.from_numpy(pcm).cuda(), torch.from_numpy(rec).cuda()
    d_pk = torch.zeros((n, P), dtype=torch.uint8, device="cuda")
    d_out = torch.zeros((n, 320), dtype=torch.int16, device="cuda")
    d_flags = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_est = torch.zeros((n, 160), dtype=torch.float32, device="cuda")
    calls = [("encode_device", lambda: dev["enc"].encode_device(n, d_pcm.data_ptr(), bits, d_pk.data_ptr()),
              lambda: host["enc"].encode(pcm, bits), lambda: d_pk),
             ("decode_device", lambda: dev["dec"].decode_device(n, d_pk.data_ptr(), d_rec.data_ptr(), bits, d_out.data_ptr()),
              lambda: host["dec"].decode(want["encode_device"], bits, received=rec), lambda: d_out),
             ("decode_track_noise_device", lambda: dev["trk"].decode_track_noise_device(n, d_pk.data_ptr(), d_rec.data_ptr(), bits,
                                                                                          d_out.data_ptr(), d_flags.data_ptr()),
              lambda: host["trk"].decode_track_noise(want["encode_device"], bits, received=rec)[0], lambda: d_out),
             ("noise_update_device", lambda: dev["nz"].noise_update_device(n, d_pcm.data_ptr(), d_rec.data_ptr(), d_flags.data_ptr(),
                                                                           d_est.data_ptr()),
              lambda: host["nz"].noise_update(pcm, update_mask=rec)[1], lambda: d_est),
             ("decode_plc_device", lambda: dev["plc"].decode_plc_device(n, d_pk.data_ptr(), d_rec.data_ptr(), bits, d_out.data_ptr(),
                                                                        d_flags.data_ptr()),
              lambda: host["plc"].decode_plc(want["encode_device"], bits, received=rec)[0], lambda: d_out),
             ("encode_dtx_device", lambda: dev["dtx"].encode_dtx_device(n, d_pcm.data_ptr(), bits, d_pk.data_ptr(), d_flags.data_ptr()),
              lambda: host["dtx"].encode_dtx(pcm, bits)[0], lambda: d_pk)]
    torch.cuda.synchronize()
    want = {}
    for hop in range(2):                   # hop 0 warms every call up (first launches, stream maps); hop 1 is checked
        for name, call, twin, result in calls:
            with torch.cuda.stream(s):
                if hop:
                    torch.cuda._sleep(50_000_000)
                call()
            if hop:
                assert not s.query(), "%s waited for the GPU" % name
            s.synchronize()
            want[name] = twin()
            assert np.array_equal(result().cpu().numpy(), want[name]), "%s (hop %d) != its host-buffer twin" % (name, hop)
    for c in list(dev.values()) + list(host.values()):
        c.close()


def test_reset_follows_the_caller_stream(gpu_api):
    """lyra_b200_reset on an installed caller stream runs behind the work already queued there: decode_plc_device hops with every
    packet lost wait behind a spin on the caller stream, then a dense reset() is called.  Afterwards every stream's control state
    is the initial (0, 0, -1), and the next hop equals a fresh context's first hop."""
    torch = _torch()
    n, bits, hops = 1024, 64, 6
    P = _capi.packet_bytes(bits)
    rng = np.random.default_rng(31)
    pk = rng.integers(0, 256, size=(n, P), dtype=np.uint8)
    rec = (np.arange(n) % 3 != 0).astype(np.uint8)
    ctx = _capi.Context(n, roles="decoder")
    fresh = _capi.Context(n, roles="decoder")
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    d_pk, d_rec = torch.from_numpy(pk).cuda(), torch.from_numpy(rec).cuda()
    d_lost = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros((n, 320), dtype=torch.int16, device="cuda")
    d_cn = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        for _ in range(hops):
            ctx.decode_plc_device(n, d_pk.data_ptr(), d_lost.data_ptr(), bits, d_out.data_ptr(), d_cn.data_ptr())
        ctx.reset()
    st = ctx.plc_state(n)
    bad = np.nonzero((st != np.array([0, 0, -1])).any(axis=1))[0]
    assert bad.size == 0, "control state after reset: %s at streams %s" % (st[bad[0]], bad[:8])
    with torch.cuda.stream(s):
        ctx.decode_plc_device(n, d_pk.data_ptr(), d_rec.data_ptr(), bits, d_out.data_ptr(), d_cn.data_ptr())
    s.synchronize()
    want, want_cn = fresh.decode_plc(pk, bits, received=rec)
    assert np.array_equal(d_out.cpu().numpy(), want) and np.array_equal(d_cn.cpu().numpy(), want_cn.astype(np.uint8))
    assert np.array_equal(ctx.plc_state(n), fresh.plc_state(n))
    ctx.close()
    fresh.close()


@pytest.mark.parametrize("workload,mode", [("codec", "exact"), ("codec", "tensor"), ("decode_plc", "exact"), ("decode_plc", "tensor")])
def test_bench_dumps_match_the_oracle(gpu_api, oracle, tmp_path, workload, mode):
    """bench.py --dump-outputs at a small size against the oracle replaying the same seeded schedule: the warm-up hops, then the
    timed hops restarting at hop 0, hop i feeding input slot i % 8 (bench.synth_pcm_np); decode_plc: packets of a fresh encoder
    over slots 0..7, the received mask of slot b = the b-th Bernoulli(1 - loss) draw of default_rng(1234 + rank) (bench.py, measure),
    comfort-noise seed = the context's (0) + the stream's id in its group."""
    import subprocess
    import sys
    import bench
    from conftest import ROOT
    n, groups, steps, hps, warmup, bits, loss = 64, 2, 2, 2, 3, 64, 0.1
    out = tmp_path / "dump"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        os.path.join(ROOT, "bench.py"), "--gpus", "1", "--streams", str(n), "--groups", str(groups), "--split", "2",
        "--steps", str(steps), "--hops-per-step", str(hps), "--warmup", str(warmup), "--no-cpu-baseline", "--no-other-configs",
        "--workload", workload, "--loss", str(loss), "--decoder-mode", mode, "--dump-outputs", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    json.loads(r.stdout.strip().splitlines()[-1])
    dump = {name: np.load(str(out / (name + ".npy"))) for name in (("pcm", "flags") if workload == "decode_plc" else ("pcm", "packets"))}
    hop_order = list(range(max(3, max(3, warmup) * hps))) + list(range(steps * hps))
    host = bench.synth_pcm_np(n, 8, bench.SEED, "noise")
    m = n // groups
    tol = pc.TENSOR_PCM_TOL_LSB if mode == "tensor" else 0
    mrng = np.random.default_rng(1234 + 0)                # rank 0
    masks = [(mrng.random(n) >= loss).astype(np.uint8) for _ in range(8)]
    for s in (0, m - 1, m, n - 1):
        if workload == "decode_plc":
            enc = oracle.Encoder(_capi.MODEL_DIR)
            pks = [enc.encode(host[b][s], bits) for b in range(8)]
            dec = oracle.Decoder(_capi.MODEL_DIR, cng_seed=s % m)
            for i in hop_order:
                if masks[i % 8][s]:
                    assert dec.set_encoded_packet(pks[i % 8])
                pcm = dec.decode_samples(320)
            assert dump["flags"][s] == float(dec.is_comfort_noise()), s
        else:
            codec = oracle.Codec(_capi.MODEL_DIR)
            for i in hop_order:
                pkt, _, _ = codec.encode(host[i % 8][s], bits)
                pcm, _, _ = codec.decode(pkt, bits)
            assert bytes(dump["packets"][s].astype(np.uint8)) == pkt, s
        d = int(np.abs(dump["pcm"][s].astype(int) - pcm.astype(int)).max())
        assert d <= tol, "stream %d: max |dumped PCM - oracle| %d" % (s, d)
