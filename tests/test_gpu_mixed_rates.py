"""GPU tier (H100) of per-stream sample rates (lyra_b200_set_stream_sample_rates): full-size dense device calls with their
sub-batches engaged, both decoder modes, the asynchrony of the setter and bench.py's device schedule with mixed rates; against
single-rate twin contexts and the oracle composition of tests/rate_cases.py."""
import os
import sys

import numpy as np
import pytest

import mixed_rate_cases as mc
import rate_cases as rc
from conftest import ROOT, read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

sys.path.insert(0, os.path.join(ROOT, "tools"))        # duplex_schedule

pytestmark = pytest.mark.gpu


def _wavs():
    return {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}


@pytest.mark.parametrize("split,mode", [(2, "tensor"), (3, "exact")])
def test_mixed_rates_4096_device_calls(gpu_api, oracle, split, mode):
    # 4096 streams at 8 / 16 / 32 / 48 kHz interleaved in a 48 kHz context: every tile of every sub-batch mixes the four rates
    mc.run_mixed_parity(_capi.Context, gpu_api, oracle, _wavs(), ctx_rate=48000, rates=mc.ALL_RATES, max_streams=4096, n=4096,
                        frames=12, oracle_rows=(0, 1, 2, 3, 2050, 4095), decoder_mode=mode, split=split, mem=TorchMem())


@pytest.mark.parametrize("ctx_rate,rates,mode", [(48000, mc.ALL_RATES, "exact"), (16000, (8000, 16000), "tensor"),
                                                 (32000, (32000, 8000, 16000), "exact")])
def test_mixed_rates_sparse_host_calls(gpu_api, oracle, ctx_rate, rates, mode):
    mc.run_mixed_parity(_capi.Context, gpu_api, oracle, _wavs(), ctx_rate=ctx_rate, rates=rates, max_streams=100,
                        stream_ids=[0, 1, 2, 3, 5, 17, 31, 32, 33, 64, 98, 99], frames=12, oracle_rows=(0, 1, 2, 3), decoder_mode=mode)


def test_mixed_rates_dense_host_calls_split(gpu_api, oracle):
    mc.run_mixed_parity(_capi.Context, gpu_api, oracle, _wavs(), ctx_rate=48000, rates=(16000, 48000, 8000, 32000), max_streams=1100,
                        n=1100, frames=12, oracle_rows=(0, 551, 1099), split=2)


def test_rate_change_mid_call(gpu_api, oracle):
    mc.run_rate_change_mid_call(_capi.Context, gpu_api, oracle, _wavs(), max_streams=64, stream_ids=(0, 7, 8, 63))


def test_moves_carry_the_rate(gpu_api):
    mc.run_moves(_capi.Context, gpu_api, _wavs(), max_streams=40, ids=(2, 33), copy_to=(17, 39), import_to=(8, 0))


def test_validation(gpu_api):
    mc.run_validation(_capi.Context, gpu_api, _wavs(), _capi.LyraB200Error)


def test_16khz_unchanged(gpu_api):
    mc.run_16khz_unchanged(_capi.Context, gpu_api, read_wav_any("sample1_16kHz.wav", 16000), max_streams=64, stream_ids=(0, 9, 63))


def test_set_stream_sample_rates_does_not_wait_for_the_gpu(gpu_api):
    """set_stream_sample_rates is asynchronous on the installed stream: with a spin of a few tens of ms queued ahead on the caller
    stream it returns while the stream is still busy, and it takes effect in stream order - between the encode_device hop queued
    before it and the one queued after it.  The packets equal a twin that ran the same sequence with host-buffer calls."""
    import torch
    n, bits, rate = 1024, 64, 48000
    P, H = _capi.packet_bytes(bits), rc.hop_of(rate)
    wavs = _wavs()
    srate = mc.interleaved(n, mc.ALL_RATES)
    ids = np.arange(n, dtype=np.int32)
    rng = np.random.default_rng(4)
    pcm = [mc.mixed_rows(wavs, np.full(n, rate, np.int32), ids, 0, H, rng)[0], mc.mixed_rows(wavs, srate, ids, 1, H, rng)[0]]
    ctx, twin = _capi.Context(n, roles="encoder"), _capi.Context(n, roles="encoder")
    for c in (ctx, twin):
        c.set_sample_rate(rate)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    d_pcm = [torch.from_numpy(x).cuda() for x in pcm]
    d_pk = [torch.zeros((n, P), dtype=torch.uint8, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        ctx.encode_device(n, d_pcm[0].data_ptr(), bits, d_pk[0].data_ptr())
        ctx.set_stream_sample_rates(srate)
        assert not s.query(), "set_stream_sample_rates waited for the GPU"
        ctx.encode_device(n, d_pcm[1].data_ptr(), bits, d_pk[1].data_ptr())
        assert not s.query()
    s.synchronize()
    want0 = twin.encode(pcm[0], bits)
    twin.set_stream_sample_rates(srate)
    want1 = twin.encode(pcm[1], bits)
    assert np.array_equal(d_pk[0].cpu().numpy(), want0), "the hop queued before the setter must run at the old rates"
    assert np.array_equal(d_pk[1].cpu().numpy(), want1), "the hop queued after the setter must run at the new rates"
    assert np.array_equal(ctx.stream_sample_rates(), srate)
    ctx.close()
    twin.close()


@pytest.mark.parametrize("mode,split", [("tensor", 2), ("exact", 3)])
def test_bench_device_schedule_with_mixed_rates(gpu_api, mode, split):
    """bench.py's device-resident schedule with per-stream rates: 2 context pairs of 1540 streams at row rate 48 kHz, streams at
    8 / 16 / 32 / 48 kHz interleaved, caller streams at priorities -1 / 0, encoder -> decoder events, 12 hops over 8 rotating
    slots queued with no host synchronisation.  Every hop's packets and PCM equal host-buffer calls on single-rate twin pairs."""
    import torch
    import duplex_schedule as ds
    rate, G, m, NBUF, hops, bits = 48000, 2, 1540, ds.NBUF, 12, 64
    n = G * m
    srate = mc.interleaved(m, mc.ALL_RATES)
    rng = np.random.default_rng(29)
    host_pcm = [rng.integers(-8192, 8192, size=(n, rc.hop_of(rate)), dtype=np.int16) for _ in range(NBUF)]
    sched = ds.Schedule(host_pcm, G, split, mode, bits, rate=rate, stream_rates=srate, keep_hops=hops)
    ds.run([sched], hops)
    torch.cuda.synchronize()
    outs = [x.cpu().numpy() for x in sched.out]
    pks = [x.cpu().numpy() for x in sched.kept_pks]
    sel = {r: np.nonzero(srate == r)[0] for r in mc.ALL_RATES}
    refs = []
    for _ in range(G):
        pair = {}
        for r in mc.ALL_RATES:
            re, rd = _capi.Context(m, roles="encoder"), _capi.Context(m, roles="decoder")
            rd.set_decoder_mode(mode)
            re.set_sample_rate(r)
            rd.set_sample_rate(r)
            pair[r] = (re, rd)
        refs.append(pair)
    for i in range(hops):
        b = i % NBUF
        for g, pair in enumerate(refs):
            for r, (re, rd) in pair.items():
                s = sel[r]
                rows = g * m + s
                pk = re.encode(host_pcm[b][rows, :rc.hop_of(r)], bits, stream_ids=s)
                assert np.array_equal(pks[i][rows], pk), "packets of hop %d group %d at %d Hz" % (i, g, r)
                got = outs[i][rows]
                want = rd.decode(pk, bits, stream_ids=s)
                bad = np.nonzero((got[:, :rc.hop_of(r)] != want).any(axis=1))[0]
                assert bad.size == 0, "PCM of hop %d group %d at %d Hz differs at streams %s" % (i, g, r, rows[bad[:8]])
                assert not got[:, rc.hop_of(r):].any(), "row tails of hop %d group %d at %d Hz are not 0" % (i, g, r)
    sched.close()
    for c in [c for pair in refs for p in pair.values() for c in p]:
        c.close()
