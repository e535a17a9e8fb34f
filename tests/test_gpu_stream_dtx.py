"""GPU tier (H100) of per-stream DTX (lyra_b200_set_stream_dtx): full-size dense device calls with their sub-batches engaged, the
asynchrony of the setter and bench.py's device schedule with DTX on for every other stream; against the oracle and against twin
contexts that run encode_dtx for the DTX-on streams and encode for the others."""
import os
import sys

import numpy as np
import pytest

import mixed_rate_cases as mc
import rate_cases as rc
import stream_dtx_cases as dc
from conftest import ROOT, read_wav_any
from lyra_b200 import _capi
from parity_cases import TENSOR_PCM_TOL_LSB
from test_gpu_parity import TorchMem

sys.path.insert(0, os.path.join(ROOT, "tools"))        # duplex_schedule

pytestmark = pytest.mark.gpu


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("split,bits", [(2, 64), (3, 184)])
def test_mixed_dtx_4096_device_calls(gpu_api, oracle, split, bits):
    dc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, max_streams=4096, n=4096, frames=14, bits=bits,
                        oracle_rows=(0, 1, 2, 3, 6, 2050, 4095), split=split, mem=TorchMem())


def test_mixed_dtx_sparse_host_calls(gpu_api, oracle):
    dc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, max_streams=100,
                        stream_ids=[0, 1, 2, 3, 5, 17, 31, 32, 33, 64, 98, 99], frames=14)


def test_mixed_dtx_dense_host_calls_split(gpu_api, oracle):
    dc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, max_streams=1100, n=1100, frames=14, split=2,
                        oracle_rows=(0, 1, 3, 6, 551, 1099))


def test_dtx_with_stream_rates_and_bits(gpu_api, oracle):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    dc.run_mixed_parity(_capi.Context, gpu_api, oracle, wavs, max_streams=1200, n=1200, frames=14, ctx_rate=48000, rates=mc.ALL_RATES,
                        bits=184, bit_set=(64, 120, 184), oracle_rows=(0, 1, 2, 3, 4, 5, 6, 7, 1199), split=2)


def test_dtx_toggle(gpu_api, oracle):
    dc.run_toggle(_capi.Context, gpu_api, oracle, _wav16(), max_streams=64, stream_ids=(0, 9, 63))


def test_dtx_moves(gpu_api):
    dc.run_moves(_capi.Context, gpu_api, _wav16(), _capi.LyraB200Error, max_streams=40, ids=(2, 33, 34), copy_to=(17, 38, 39),
                 import_to=(8, 0, 1))


def test_dtx_validation(gpu_api):
    dc.run_validation(_capi.Context, gpu_api, _capi.LyraB200Error)


def test_dtx_unchanged_when_unused(gpu_api):
    dc.run_unchanged_when_unused(_capi.Context, gpu_api, _wav16(), max_streams=64, stream_ids=(0, 9, 63))


def test_set_stream_dtx_does_not_wait_for_the_gpu(gpu_api):
    """set_stream_dtx is asynchronous on the installed stream: with a spin queued ahead on the caller stream it returns while the
    stream is still busy, and it takes effect in stream order - between the encode_dtx_device hops queued before and after it.
    Flags and packets equal a twin that ran the same sequence with host-buffer calls."""
    import torch
    n, bits, hops = 1024, 64, 16
    P = _capi.packet_bytes(bits)
    wav = _wav16()
    pcm = [rc.speech_rows(wav, 16000, range(n), f) for f in range(hops)]
    for x in pcm[6:]:
        x[::2] = 3                                         # the even streams go quiet: DTX hops
    en = (np.arange(n) % 4 != 0).astype(np.int32)
    ctx, twin = _capi.Context(n, roles="encoder"), _capi.Context(n, roles="encoder")
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    d_pcm = [torch.from_numpy(x).cuda() for x in pcm]
    d_pk = [torch.zeros((n, P), dtype=torch.uint8, device="cuda") for _ in range(hops)]
    d_fl = [torch.zeros((n,), dtype=torch.uint8, device="cuda") for _ in range(hops)]
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        for f in range(hops):
            if f == hops // 2:
                ctx.set_stream_dtx(en)
                assert not s.query(), "set_stream_dtx waited for the GPU"
            ctx.encode_dtx_device(n, d_pcm[f].data_ptr(), bits, d_pk[f].data_ptr(), d_fl[f].data_ptr())
        assert not s.query()
    s.synchronize()
    for f in range(hops):
        if f == hops // 2:
            twin.set_stream_dtx(en)
        pk, sizes = twin.encode_dtx(pcm[f], bits)
        assert np.array_equal(d_pk[f].cpu().numpy(), pk) and np.array_equal(d_fl[f].cpu().numpy(), (sizes == 0).astype(np.uint8)), f
        if f >= hops // 2:
            assert (sizes[en == 0] > 0).all(), "hop %d: a DTX-off stream had a DTX hop" % f
    assert np.array_equal(ctx.stream_dtx(), en)
    ctx.close()
    twin.close()


def test_bench_device_schedule_with_mixed_dtx(gpu_api, oracle):
    """bench.py's device-resident schedule with DTX on for every other stream: 2 context pairs of 1540 streams, 24 hops over 8
    rotating slots of speech (every third stream silent in slots 4-7) queued with no host synchronisation; the decoders take
    DTX hops as lost packets.  Sampled rows of both groups equal the oracle hop by hop: the packets, the DTX flags and the PCM."""
    import torch
    import duplex_schedule as ds
    G, m, NBUF, hops, bits, mode = 2, 1540, ds.NBUF, 24, 64, "tensor"
    n = G * m
    wav = _wav16()
    start = (np.arange(n, dtype=np.int64) * 7919) % len(wav)
    host_pcm = [wav[(start[:, None] + b * 320 + np.arange(320)[None, :]) % len(wav)] for b in range(NBUF)]
    for x in host_pcm[NBUF // 2:]:
        x[::3] = 0
    en = (np.arange(m) % 2 == 0).astype(np.int32)
    sched = ds.Schedule(host_pcm, G, 2, mode, bits, dtx=en, keep_hops=hops)
    ds.run([sched], hops)
    torch.cuda.synchronize()
    outs = [x.cpu().numpy() for x in sched.out]
    pks = [x.cpu().numpy() for x in sched.kept_pks]
    flags = [x.cpu().numpy() for x in sched.kept_flags]
    rows = (0, 1, 2, 3, 6, m, m + 3, m + 6, 2 * m - 1)
    enc = {r: rc.OracleEncoder(oracle, 16000, dtx=bool(en[r % m])) for r in rows}
    dec = {r: rc.OracleCodec(oracle, 16000) for r in rows}
    seen = set()
    for i in range(hops):
        x = host_pcm[i % NBUF]
        for r in rows:
            want = enc[r].encode(x[r], bits)
            assert flags[i][r] == (len(want) == 0), "DTX flag of hop %d row %d" % (i, r)
            assert bytes(pks[i][r][:len(want)]) == want and not pks[i][r][len(want):].any(), "packet of hop %d row %d" % (i, r)
            d = rc._pcm_diff(outs[i][r], dec[r].decode(want or None, bits))
            assert d <= TENSOR_PCM_TOL_LSB, "PCM of hop %d row %d: max |d| %d" % (i, r, d)
            seen.add((int(en[r % m]), int(flags[i][r])))
        assert not flags[i].reshape(G, m)[:, en == 0].any(), "a DTX-off stream had a DTX hop, hop %d" % i
    assert (1, 1) in seen and (1, 0) in seen, "the DTX-on rows must produce both empty and encoded hops: %s" % seen
    sched.close()
