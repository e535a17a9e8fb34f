"""GPU tier (H100) of the fused codec calls at 8 / 32 / 48 kHz (lyra_b200_set_sample_rate): every rate, full-size dense calls with
their sub-batches engaged, both decoder modes, caller CUDA streams; against the oracle composition of tests/rate_cases.py and
against the host-buffer twins."""
import os
import sys

import numpy as np
import pytest

import parity_cases as pc
import rate_cases as rc
from conftest import ROOT, read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

sys.path.insert(0, os.path.join(ROOT, "tools"))        # duplex_schedule

pytestmark = pytest.mark.gpu


def _wav(rate):
    return read_wav_any("sample1_%dkHz.wav" % (rate // 1000), rate)


@pytest.mark.parametrize("rate", rc.RATES)
def test_fused_calls_sparse_ids(gpu_api, oracle, rate):
    rc.run_rate_parity(_capi.Context, gpu_api, oracle, _wav(rate), rate=rate, max_streams=100, stream_ids=[0, 5, 17, 31, 32, 64, 99],
                       frames=14)


@pytest.mark.parametrize("rate,mode", [(8000, "exact"), (32000, "tensor"), (48000, "exact"), (48000, "tensor")])
def test_fused_calls_dense_sub_batches(gpu_api, oracle, rate, mode):
    # 1100 streams = 138 tiles (the last one partial): split 2 engages; the checked streams sit at the edges of both sub-batches
    rc.run_rate_parity(_capi.Context, gpu_api, oracle, _wav(rate), rate=rate, max_streams=1100, n=1100, frames=12,
                       check=[0, 551, 552, 1097, 1099], decoder_mode=mode, split=2)


@pytest.mark.parametrize("rate", rc.RATES)
def test_equivalence_with_the_plugin_chain(gpu_api, rate):
    rc.run_equivalence_with_plugin_chain(_capi.Context, gpu_api, rate=rate, max_streams=64, stream_ids=(0, 7, 8, 40, 63), frames=4)


@pytest.mark.parametrize("rate,split,mode", [(48000, 2, "tensor"), (48000, 3, "exact"), (8000, 3, "tensor"), (32000, 2, "exact")])
def test_device_twins_4096(gpu_api, rate, split, mode):
    rc.run_device_twins(_capi.Context, gpu_api, TorchMem(), _wav(rate), rate=rate, n=4096, frames=5, decoder_mode=mode, split=split)


@pytest.mark.parametrize("rate", rc.RATES)
def test_dtx_estimator_at_external_rate(gpu_api, oracle, rate):
    # speech, then 5 s of low-level noise: long enough for the estimators' minimum tracking at every rate
    sizes = rc.run_dtx_at_rate(_capi.Context, gpu_api, oracle, _wav(rate), rate=rate, speech_hops=10, noise_hops=250)
    print("DTX at %d Hz: %d of %d hops empty" % (rate, sizes.count(0), len(sizes)))


def test_rate_change_and_reset(gpu_api, oracle):
    rc.run_rate_change_and_reset(_capi.Context, gpu_api, oracle, {r: _wav(r) for r in (32000, 48000)}, _capi.LyraB200Error,
                                 rates=(32000, 48000))
    rc.run_rate_change_and_reset(_capi.Context, gpu_api, oracle, {r: _wav(r) for r in (8000, 32000)}, _capi.LyraB200Error,
                                 rates=(8000, 32000))


@pytest.mark.parametrize("rate", rc.RATES)
def test_integration_criterion_through_the_rate_aware_calls(gpu_api, oracle, rate):
    worst = rc.run_integration_at_rate(_capi.Context, gpu_api, oracle, rate=rate, wav=_wav(rate))
    print("integration LSD at %d Hz through encode / decode: worst hop %.3f" % (rate, worst))
    assert worst < 2.0


@pytest.mark.parametrize("mode,split", [("exact", 2), ("tensor", 3)])
def test_bench_device_schedule_at_48khz(gpu_api, oracle, mode, split):
    """bench.py's device-resident schedule at 48 kHz: 2 context pairs of 1540 streams over slices of shared buffers, caller
    streams at priorities -1 / 0, encoder -> decoder events, 12 hops over 8 rotating slots queued with no host synchronisation.
    Every hop's output is kept; all streams are compared with host-buffer calls on one reference pair per group, the streams at
    the slice edges with the oracle composition."""
    import torch
    import duplex_schedule as ds
    rate, G, m, NBUF, hops, bits = 48000, 2, 1540, ds.NBUF, 12, 64
    n = G * m
    tol = pc.TENSOR_PCM_TOL_LSB if mode == "tensor" else 0
    rng = np.random.default_rng(23)
    host_pcm = [rng.integers(-8192, 8192, size=(n, rc.hop_of(rate)), dtype=np.int16) for _ in range(NBUF)]
    edges = [0, m - 1, m, n - 1]
    sched = ds.Schedule(host_pcm, G, split, mode, bits, rate=rate, keep_hops=hops)
    ds.run([sched], hops)
    torch.cuda.synchronize()
    outs = [x.cpu().numpy() for x in sched.out]
    pks = [x.cpu().numpy() for x in sched.kept_pks]
    refs = []
    for _ in range(G):
        re, rd = _capi.Context(m, roles="encoder"), _capi.Context(m, roles="decoder")
        rd.set_decoder_mode(mode)
        re.set_sample_rate(rate)
        rd.set_sample_rate(rate)
        refs.append((re, rd))
    oracles = {s: rc.OracleCodec(oracle, rate) for s in edges}
    for i in range(hops):
        b = i % NBUF
        for g, (re, rd) in enumerate(refs):
            sl = slice(g * m, (g + 1) * m)
            pk = re.encode(host_pcm[b][sl], bits)
            assert np.array_equal(pks[i][sl], pk), "packets of hop %d group %d" % (i, g)
            want = rd.decode(pk, bits)
            bad = np.nonzero((outs[i][sl] != want).any(axis=1))[0]
            assert bad.size == 0, "PCM of hop %d group %d differs from host-buffer calls at streams %s" % (i, g, (bad + g * m)[:8])
        for s in edges:
            opkt = oracles[s].encode(host_pcm[b][s], bits)
            assert bytes(pks[i][s]) == opkt, (i, s)
            d = int(np.abs(outs[i][s].astype(int) - oracles[s].decode(opkt, bits).astype(int)).max())
            assert d <= tol, "hop %d stream %d: max |PCM - oracle| %d" % (i, s, d)
    sched.close()
    for c in [c for r in refs for c in r]:
        c.close()
