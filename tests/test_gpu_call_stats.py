"""GPU tier (H100) of the per-stream call statistics (lyra_b200_set_stats / _read_stats / _read_stats_device): every kind through
its host-buffer call, sparse ids and device twin, 4096 streams with sub-batches in both decoder modes, mixed per-stream settings,
the active mask, clear, moves, launch counts and graph replays.  The cases are in call_stats_cases.py."""
import ctypes as C

import numpy as np
import pytest

import call_stats_cases as st
import mixed_rate_cases as mc
from conftest import read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


def _wavs():
    return {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}


@pytest.mark.parametrize("call", ["dense", "sparse", "device"])
@pytest.mark.parametrize("kind", st.KINDS)
def test_call_stats_kinds(gpu_api, kind, call):
    st.run_kind(_capi.Context, gpu_api, TorchMem(), {16000: _wav16()}, kind, n=300, hops=16 if kind == "decode_plc" else 6,
                sparse=call == "sparse", device=call == "device")


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_call_stats_split_4096(gpu_api, mode):
    st.run_split_independence(_capi.Context, gpu_api, TorchMem(), _wav16(), n=4096, hops=4, mode=mode)


@pytest.mark.parametrize("kind", st.KINDS)
def test_call_stats_mixed_settings(gpu_api, kind):
    st.run_kind(_capi.Context, gpu_api, TorchMem(), _wavs(), kind, n=1200, hops=16 if kind == "decode_plc" else 6, split=2,
                ctx_rate=48000, rates=(8000, 16000, 48000), bits=184, bit_set=(64, 120, 184), dtx=[k % 3 != 1 for k in range(1200)])


@pytest.mark.parametrize("kind", st.KINDS)
def test_call_stats_active_mask(gpu_api, kind):
    st.run_kind(_capi.Context, gpu_api, TorchMem(), _wavs(), kind, n=1200, hops=16 if kind == "decode_plc" else 8, device=True,
                masked=True, split=2, ctx_rate=48000, rates=(8000, 16000, 48000))


def test_call_stats_levels(gpu_api):
    st.run_levels(_capi.Context, gpu_api)


@pytest.mark.parametrize("kind", st.KINDS)
def test_call_stats_clear(gpu_api, kind):
    st.run_clear(_capi.Context, gpu_api, TorchMem(), {16000: _wav16()}, kind, n=200, hops=14 if kind == "decode_plc" else 5)


def test_call_stats_travel(gpu_api):
    st.run_travel(_capi.Context, gpu_api, TorchMem(), _wav16(), max_streams=64)


@pytest.mark.parametrize("split", [None, 3])
def test_call_stats_off_and_launches(gpu_api, split):
    st.run_off_and_launches(_capi.Context, gpu_api, TorchMem(), _wav16(), n=2048 if split else 64, hops=2, split=split)


def test_call_stats_unaligned_rows(gpu_api):
    st.run_unaligned(_capi.Context, gpu_api, TorchMem(), _wavs(), n=300, hops=1)


def test_call_stats_argument_errors(gpu_api):
    st.run_argument_errors(_capi.Context, gpu_api, TorchMem())


def test_call_stats_graph_replays(gpu_api):
    """Dense host-buffer calls on page-locked buffers keep replaying graphs with statistics on (graphs of their own), and the
    statistics count every replayed hop: they equal those of a context without graphs."""
    import torch
    n, bits = 256, 64
    P = _capi.packet_bytes(bits)
    gr, ref = _capi.Context(n), _capi.Context(n)
    gr.set_graphs(True)
    lib = gpu_api.lib
    pin_pcm = torch.zeros((n, 320), dtype=torch.int16).pin_memory()
    pin_pk = torch.zeros((n, P), dtype=torch.uint8).pin_memory()
    pin_out = torch.zeros((n, 320), dtype=torch.int16).pin_memory()
    p = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731
    rng = np.random.default_rng(8)
    for phase in range(3):
        if phase == 1:
            gr.set_stats(1)
            ref.set_stats(1)
        r0 = gr.graph_replays()
        for f in range(4):
            pcm = rng.integers(-8000, 8000, size=(n, 320), dtype=np.int16)
            pk = ref.encode(pcm, bits)
            out = ref.decode(pk, bits)
            pin_pcm.numpy()[:] = pcm
            assert lib.lyra_b200_encode(gr.h, None, n, p(pin_pcm), bits, p(pin_pk)) == 0
            assert np.array_equal(pin_pk.numpy(), pk), (phase, f)
            assert lib.lyra_b200_decode(gr.h, None, n, p(pin_pk), None, bits, p(pin_out)) == 0
            assert np.array_equal(pin_out.numpy(), out), (phase, f)
        assert gr.graph_replays() - r0 >= 6, "phase %d: the dense calls stopped replaying graphs" % phase
        for role in ("encoder", "decoder"):
            assert np.array_equal(gr.stats(role, n=n), ref.stats(role, n=n)), "phase %d: %s statistics differ" % (phase, role)
    assert gr.stats("encoder", n=n)[:, st.HOPS].tolist() == [8] * n
    gr.close()
    ref.close()
