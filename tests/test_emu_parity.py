"""CPU tier: the product kernels' source, compiled for the test-only CUDA block simulator (tests/cuda_emu),
checked against the oracle.  Small sizes (the simulator runs every CUDA thread as a fiber)."""
import numpy as np
import pytest

import parity_cases as pc
from lyra_b200 import _capi


def test_emu_codec_parity_sparse_ids_and_loss(emu_api, oracle, sample1):
    # 3 streams spread over 2 tiles, speech input, a lost packet every 5th frame, 20 frames (ring wrap at 18)
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=20, stream_ids=[0, 5, 17], frames=20, bits=64,
                        wav=sample1, loss_every=5)


def test_emu_codec_parity_all_bitrates(emu_api, oracle):
    for bits in (120, 184):
        pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=[1, 2], frames=3, bits=bits, seed=bits)


def test_emu_loud_and_silent_input(emu_api, oracle):
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=[4], frames=3, bits=64, kind="loud")
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=[4], frames=2, bits=64, kind="silence")


def test_emu_tensor_decoder_mode(emu_api, oracle, sample1):
    # split-precision TF32 decoder: packets bit-exact, PCM within the stated tolerance, over a ring wrap, with loss
    worst = pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=[0, 9], frames=20, bits=64,
                                wav=sample1, loss_every=7, decoder_mode="tensor")
    assert worst <= pc.TENSOR_PCM_TOL_LSB
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=8, stream_ids=[3], frames=3, bits=184, kind="loud",
                        decoder_mode="tensor")


def test_emu_plugin_surface(emu_api, oracle):
    pc.run_plugin_surface_parity(_capi.Context, emu_api, oracle, n=3, frames=2)


def test_emu_reset_and_isolation(emu_api, oracle):
    pc.run_reset_and_isolation(_capi.Context, emu_api, oracle)


def test_emu_error_paths(emu_api):
    pc.run_error_paths(_capi.Context, emu_api, _capi.LyraB200Error)


def test_emu_logmel(emu_api, oracle, sample1):
    pc.run_logmel_parity(_capi.Context, emu_api, oracle, sample1, n=2, frames=3)


def test_emu_noise_estimator(emu_api, oracle, sample1):
    pc.run_noise_estimator_parity(_capi.Context, emu_api, oracle, sample1, n=2, frames=14)


def test_emu_decode_track_noise(emu_api, oracle, sample1):
    pc.run_decode_track_noise_parity(_capi.Context, emu_api, oracle, sample1, stream_ids=[1, 10], max_streams=16, frames=5, loss_every=3)


def test_emu_cpp_components(emu_api, oracle, tmp_path):
    """The C++ adapters (include/lyra_b200/lyra_b200_components.h: SoundStreamEncoder / ResidualVectorQuantizer /
    LyraGanModel / NoiseEstimator / LyraEncoder / LyraDecoder counterparts) over the emulated library, vs the oracle."""
    import os
    import shutil
    import subprocess
    from conftest import ROOT
    shutil.copy(emu_api.path, str(tmp_path / "liblyra_b200.so"))
    exe = str(tmp_path / "test_components")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "oracle"),
                           os.path.join(ROOT, "tests", "cpp", "test_components.cc"), "-o", exe,
                           "-L" + str(tmp_path), "-llyra_b200", "-L" + os.path.join(ROOT, "oracle", "_build"), "-llyra_oracle",
                           "-Wl,-rpath," + str(tmp_path), "-Wl,-rpath," + os.path.join(ROOT, "oracle", "_build"), "-lpthread"])
    out = subprocess.run([exe, _capi.MODEL_DIR], capture_output=True, text=True, env=dict(os.environ, LYRA_B200_MAX_STREAMS="16"))
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr


def test_emu_priority_switch(emu_api, oracle):
    pc.run_priority_switch(_capi.Context, emu_api, oracle, n=2, frames=3)


def test_emu_sixteen_stream_tiles(emu_api, oracle, monkeypatch):
    monkeypatch.setenv("LYRA_B200_TILE_STREAMS", "16")
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=32, stream_ids=[3, 17], frames=3, bits=64)
    pc.run_codec_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=[5], frames=2, bits=64, decoder_mode="tensor")


def test_emu_role_contexts(emu_api, oracle):
    pc.run_role_contexts(_capi.Context, emu_api, oracle, _capi.LyraB200Error, frames=2)


def test_emu_full_duplex_threads(emu_api, oracle):
    """An encoder-only and a decoder-only context driven concurrently by two host threads (the benchmark's host-buffer pass,
    INTEGRATION.md section 3): packets and PCM still equal the oracle's."""
    import queue
    import threading
    from conftest import MODEL_DIR
    n, frames = 2, 4
    enc = _capi.Context(8, capi=emu_api, roles="encoder")
    dec = _capi.Context(8, capi=emu_api, roles="decoder")
    rng = np.random.default_rng(12)
    pcm = [pc.synth_pcm(rng, n) for _ in range(frames)]
    q, packets, outs, errors = queue.Queue(), [None] * frames, [None] * frames, []

    def uplink():
        try:
            for f in range(frames):
                packets[f] = enc.encode(pcm[f], 64)
                q.put(f)
        except Exception as e:      # pragma: no cover
            errors.append(e)
            q.put(None)

    def downlink():
        try:
            for _ in range(frames):
                f = q.get()
                if f is None:
                    return
                outs[f] = dec.decode(packets[f], 64)
        except Exception as e:      # pragma: no cover
            errors.append(e)

    th = [threading.Thread(target=uplink), threading.Thread(target=downlink)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    codecs = [oracle.Codec(MODEL_DIR) for _ in range(n)]
    for f in range(frames):
        for k in range(n):
            opkt, _, _ = codecs[k].encode(pcm[f][k], 64)
            opcm, _, _ = codecs[k].decode(opkt, 64)
            assert bytes(packets[f][k]) == opkt and np.array_equal(outs[f][k], opcm), (f, k)
    enc.close()
    dec.close()


def test_emu_cpp_duplex_server_example(emu_api, oracle, tmp_path):
    """examples/duplex_server.cc (C++ worker threads over encoder-only / decoder-only contexts) against the oracle."""
    import os
    import shutil
    import subprocess
    from conftest import MODEL_DIR, ROOT
    shutil.copy(emu_api.path, str(tmp_path / "liblyra_b200.so"))
    exe = str(tmp_path / "duplex_server")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "duplex_server.cc"),
                           "-o", exe, "-L" + str(tmp_path), "-llyra_b200", "-Wl,-rpath," + str(tmp_path), "-lpthread"])
    streams, steps = 4, 3

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
            pkt, _, _ = c.encode(hop(s, i), 64)
            pcm, _, _ = c.decode(pkt, 64)
        want += int(pcm.astype(np.int64).sum())
    for groups in (1, 2):
        out = subprocess.run([exe, MODEL_DIR, str(streams), str(steps), str(groups), "64"], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert int(out.stdout.strip().rsplit("checksum", 1)[1]) == want, out.stdout


def test_emu_wgmma_probe(tmp_path):
    """tests/cpp/wgmma_probe.cu on the emulator's wgmma model (device_compat.h): matrix descriptors, register and shared-memory A
    operands, fragment layouts, split-precision MMAs, the accumulator-to-operand shuffle.  The same source runs on the GPU tier,
    which is what ties the emulator's model to the hardware."""
    import os
    import subprocess
    from conftest import EMU_DIR, ROOT
    exe = str(tmp_path / "wgmma_probe")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DLYRA_EMU", "-x", "c++", "-I" + EMU_DIR, "-I" + os.path.join(ROOT, "lyra_b200", "csrc"),
                           "-Wno-unknown-pragmas", os.path.join(ROOT, "tests", "cpp", "wgmma_probe.cu"), os.path.join(EMU_DIR, "cuda_emu.cc"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.count("MATCH") == 2 and "MISMATCH" not in out.stdout, out.stdout + out.stderr


def test_emu_comfort_noise_generator(emu_api, oracle):
    pc.run_cng_parity(_capi.Context, emu_api, oracle, stream_ids=(0, 5), hops=3)


def test_emu_plc_state_machine(emu_api, oracle, sample1):
    # batched LyraDecoder tick (plan -> RVQ -> LyraGAN -> comfort noise -> cross-fade -> noise estimator) vs the oracle decoder
    pc.run_plc_parity(_capi.Context, emu_api, oracle, max_streams=16, stream_ids=(1, 9), frames=14, wav=sample1, outages=((2, 9), (4, 2)))
    pc.run_plc_state_peer(_capi.Context, emu_api, oracle)


def test_emu_dtx_encoder(emu_api, oracle, sample1):
    pc.run_dtx_parity(_capi.Context, emu_api, oracle, wav=sample1, frames=8)


def test_emu_resampler(emu_api, oracle):
    pc.run_resampler_parity(_capi.Context, emu_api, oracle)
