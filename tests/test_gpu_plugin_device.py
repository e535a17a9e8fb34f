"""GPU tier (H100) of the device twins of the plugin-level calls: the shared cases of plugin_device_cases.py at one row, a
partial last tile and a count that crosses a sub-batch edge (1540 streams = 193 tiles: at set_split 3 the parts hold 64, 64
and 65 tiles), in both decoder modes, and a check that no twin waits on the host."""
import numpy as np
import pytest

import plugin_device_cases as pd
import rate_cases as rc
from conftest import read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu

EDGE_N = 1540


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
@pytest.mark.parametrize("n,split", [(1, 3), (12, 3), (EDGE_N, 1), (EDGE_N, 3)])
def test_plugin_device_nets(gpu_api, n, split, mode):
    pd.run_nets_twin(_capi.Context, gpu_api, TorchMem(), _wav16(), n=n, hops=3, mode=mode, split=split)


@pytest.mark.parametrize("indices", [True, False])
@pytest.mark.parametrize("bits", [64, 120, 184])
@pytest.mark.parametrize("n", [1, 12, EDGE_N])
def test_plugin_device_rvq(gpu_api, n, bits, indices):
    pd.run_rvq_twin(_capi.Context, gpu_api, TorchMem(), n=n, hops=2, bits=bits, indices=indices)


@pytest.mark.parametrize("n", [1, 12, EDGE_N])
def test_plugin_device_logmel(gpu_api, n):
    pd.run_logmel_twin(_capi.Context, gpu_api, TorchMem(), _wav16(), n=n, hops=3)


@pytest.mark.parametrize("n", [1, 12, EDGE_N])
def test_plugin_device_cng(gpu_api, n):
    pd.run_cng_twin(_capi.Context, gpu_api, TorchMem(), n=n, hops=4)


@pytest.mark.parametrize("n", [1, 12, EDGE_N])
def test_plugin_device_noise_estimate(gpu_api, n):
    pd.run_noise_twin(_capi.Context, gpu_api, TorchMem(), _wav16(), n=n, hops=6)


@pytest.mark.parametrize("to_internal", [1, 0])
@pytest.mark.parametrize("rate", pd.RESAMPLE_RATES)
@pytest.mark.parametrize("n", [1, EDGE_N])
def test_plugin_device_resample(gpu_api, n, rate, to_internal):
    pd.run_resample_twin(_capi.Context, gpu_api, TorchMem(), n=n, hops=4, rate=rate, to_internal=to_internal)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
@pytest.mark.parametrize("n,split", [(12, 3), (EDGE_N, 1), (EDGE_N, 3)])
def test_plugin_device_chain(gpu_api, oracle, n, split, mode):
    pd.run_chain(_capi.Context, gpu_api, TorchMem(), _wav16(), oracle, n=n, hops=4, mode=mode, split=split,
                 oracle_rows=(0, n - 1) if n < 100 else (0, 777, n - 1))


@pytest.mark.parametrize("n", [12, EDGE_N])
def test_plugin_device_cng_chain(gpu_api, n):
    pd.run_cng_chain(_capi.Context, gpu_api, TorchMem(), _wav16(), n=n, hops=5)


def test_plugin_device_refusals(gpu_api):
    pd.run_refusals(_capi.Context, gpu_api, TorchMem())


def test_plugin_device_mask_ignored(gpu_api):
    """with an active mask that sits streams out installed, every twin gives what its host twin gives"""
    mem, wav, n = TorchMem(), _wav16(), EDGE_N
    pd.run_nets_twin(_capi.Context, gpu_api, mem, wav, n=n, hops=2, split=3, mode="tensor", mask=True)
    pd.run_rvq_twin(_capi.Context, gpu_api, mem, n=n, hops=1, bits=120, indices=True, mask=True)
    pd.run_logmel_twin(_capi.Context, gpu_api, mem, wav, n=n, hops=2, banks_bins=((0, 64), (1, 160)), mask=True)
    pd.run_cng_twin(_capi.Context, gpu_api, mem, n=n, hops=2, mask=True)
    pd.run_noise_twin(_capi.Context, gpu_api, mem, wav, n=n, hops=3, mask=True)
    pd.run_resample_twin(_capi.Context, gpu_api, mem, n=n, hops=2, rate=8000, to_internal=1, mask=True)


def test_plugin_device_no_host_wait(gpu_api):
    """With a sleep queued on the installed stream, every twin returns while an event recorded after the sleep is still pending;
    then the results equal the host twins'."""
    import torch
    n, bits = EDGE_N, 120
    P = _capi.packet_bytes(bits)
    mem = TorchMem()
    A, B = pd._pair(_capi.Context, gpu_api, mem, n, split=3)
    pcm = rc.speech_rows(_wav16(), 16000, range(n), 0)
    d_pcm = mem.zeros((n, 320), np.int16)
    mem.put(d_pcm, pcm)
    d_feat, d_lossy = mem.zeros((n, 64), np.float32), mem.zeros((n, 64), np.float32)
    d_pk, d_idx = mem.zeros((n, P), np.uint8), mem.zeros((n, 46), np.int32)
    d_out, d_mel = mem.zeros((n, 320), np.int16), mem.zeros((n, 160), np.float32)
    d_est, d_flags = mem.zeros((n, 160), np.float32), mem.zeros((n,), np.uint8)
    d_cng = mem.zeros((n, 320), np.int16)
    d_rs, d_cnt = mem.zeros((n, 961), np.int16), mem.zeros((n,), np.int32)
    torch.cuda.synchronize()
    calls = [
        ("extract_features_device", lambda: A.extract_features_device(n, d_pcm.data_ptr(), d_feat.data_ptr())),
        ("quantize_device", lambda: A.quantize_device(n, d_feat.data_ptr(), bits, d_pk.data_ptr(), d_idx.data_ptr())),
        ("dequantize_device", lambda: A.dequantize_device(n, d_pk.data_ptr(), bits, d_lossy.data_ptr())),
        ("generate_device", lambda: A.generate_device(n, d_lossy.data_ptr(), d_out.data_ptr())),
        ("logmel_device", lambda: A.logmel_device(n, d_pcm.data_ptr(), d_mel.data_ptr(), 160, 1)),
        ("noise_update_device", lambda: A.noise_update_device(n, d_pcm.data_ptr(), 0, 0, 0)),
        ("noise_estimate_device", lambda: A.noise_estimate_device(n, d_est.data_ptr(), d_flags.data_ptr())),
        ("cng_generate_device", lambda: A.cng_generate_device(n, d_est.data_ptr(), d_cng.data_ptr())),
        ("resample_device", lambda: A.resample_device(n, 48000, 0, d_pcm.data_ptr(), 320, d_rs.data_ptr(), 961, d_cnt.data_ptr())),
    ]
    with torch.cuda.stream(mem.s):
        torch.cuda._sleep(200_000_000)
        ev = torch.cuda.Event()
        ev.record(mem.s)
        for name, call in calls:
            l0 = A.launch_count
            call()
            assert A.launch_count > l0, "%s launched nothing" % name
            assert not ev.query(), "%s waited for the GPU" % name
    mem.s.synchronize()
    feats = B.extract_features(pcm)
    pk, idx = B.quantize(feats, bits, want_indices=True)
    lossy = B.dequantize(pk, bits)
    B.noise_update(pcm)
    est, flags = B.noise_estimate(n=n)
    want_rs = B.resample(pcm, 48000, False)
    got = {k: mem.get(v) for k, v in dict(feat=d_feat, pk=d_pk, idx=d_idx, lossy=d_lossy, out=d_out, mel=d_mel, est=d_est,
                                           flags=d_flags, cng=d_cng, rs=d_rs, cnt=d_cnt).items()}
    assert np.array_equal(got["feat"], feats) and np.array_equal(got["pk"], pk) and np.array_equal(got["idx"], idx)
    assert np.array_equal(got["lossy"], lossy) and np.array_equal(got["out"], B.generate(lossy))
    assert np.array_equal(got["mel"], B.logmel(pcm, 160, 1))
    assert np.array_equal(got["est"], est) and np.array_equal(got["flags"], flags.astype(np.uint8))
    assert np.array_equal(got["cng"], B.cng_generate(est))
    assert np.array_equal(got["cnt"], [len(w) for w in want_rs])
    assert all(np.array_equal(got["rs"][k, :len(w)], w) for k, w in enumerate(want_rs))
    assert np.array_equal(A.export_streams(), B.export_streams())
    pd._close(A, B)
