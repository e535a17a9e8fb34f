"""GPU tier (H100) of per-stream bit counts (lyra_b200_set_stream_bits): full-size dense device calls with their sub-batches
engaged, both decoder modes, graphs, the asynchrony of the setter and bench.py's device schedule with mixed bit counts; against
single-bit-count twin contexts and the oracle."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import mixed_rate_cases as mc
import stream_bits_cases as bc
from conftest import ROOT, read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

sys.path.insert(0, os.path.join(ROOT, "tools"))        # duplex_schedule

pytestmark = pytest.mark.gpu


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("split,mode,bit_set", [(2, "tensor", bc.COMMON), (3, "exact", bc.ODD)])
def test_mixed_bits_4096_device_calls(gpu_api, oracle, split, mode, bit_set):
    bc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, bit_set=bit_set, max_streams=4096, n=4096, frames=12,
                        oracle_rows=(0, 1, 2, 3, 2050, 4095), decoder_mode=mode, split=split, mem=TorchMem())


@pytest.mark.parametrize("bit_set,mode", [(bc.COMMON, "exact"), (bc.ODD, "tensor")])
def test_mixed_bits_sparse_host_calls(gpu_api, oracle, bit_set, mode):
    bc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, bit_set=bit_set, max_streams=100,
                        stream_ids=[0, 1, 2, 3, 5, 17, 31, 32, 33, 64, 98, 99], frames=12, oracle_rows=(0, 1, 2, 3), decoder_mode=mode)


def test_mixed_bits_dense_host_calls_split(gpu_api, oracle):
    bc.run_mixed_parity(_capi.Context, gpu_api, oracle, {16000: _wav16()}, bit_set=bc.COMMON, max_streams=1100, n=1100, frames=12,
                        oracle_rows=(0, 551, 1099), split=2)


def test_bits_with_stream_sample_rates(gpu_api, oracle):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    bc.run_mixed_parity(_capi.Context, gpu_api, oracle, wavs, bit_set=bc.COMMON, max_streams=1200, n=1200, frames=12, ctx_rate=48000,
                        rates=mc.ALL_RATES, oracle_rows=(0, 1, 2, 3, 1199), split=2)


def test_bits_change_between_hops(gpu_api):
    bc.run_bits_change(_capi.Context, gpu_api, _wav16(), max_streams=64, stream_ids=(0, 9, 63))


def test_validation(gpu_api):
    bc.run_validation(_capi.Context, gpu_api, _wav16(), _capi.LyraB200Error)


def test_moves_carry_the_words(gpu_api):
    bc.run_moves(_capi.Context, gpu_api, _wav16(), max_streams=40, ids=(2, 33), copy_to=(17, 39), import_to=(8, 0))
    bc.run_refused_after_move(_capi.Context, gpu_api, _capi.LyraB200Error)


def test_unchanged_when_unused(gpu_api):
    bc.run_unchanged_when_unused(_capi.Context, gpu_api, _wav16(), max_streams=64, stream_ids=(0, 9, 63))


def test_graphs_keep_replaying(gpu_api):
    """Dense host-buffer calls on page-locked buffers keep replaying graphs before any word is set, while words are set (graphs
    of their own) and after they are cleared; every call equals a context without graphs."""
    import torch
    n, bits = 256, 184
    P = _capi.packet_bytes(bits)
    gr, ref = _capi.Context(n), _capi.Context(n)
    gr.set_graphs(True)
    lib = gpu_api.lib
    pin_pcm = torch.zeros((n, 320), dtype=torch.int16).pin_memory()
    pin_pk = torch.zeros((n, P), dtype=torch.uint8).pin_memory()
    pin_out = torch.zeros((n, 320), dtype=torch.int16).pin_memory()
    p = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731
    sbits = mc.interleaved(n, bc.COMMON)
    rng = np.random.default_rng(8)
    for phase, words in enumerate((None, sbits, np.zeros(n, np.int32))):
        if words is not None:
            for c in (gr, ref):
                c.set_stream_bits("encoder", words)
                c.set_stream_bits("decoder", words)
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
    gr.close()
    ref.close()


def test_set_stream_bits_does_not_wait_for_the_gpu(gpu_api):
    """set_stream_bits is asynchronous on the installed stream: with a spin of a few tens of ms queued ahead on the caller stream
    it returns while the stream is still busy, and it takes effect in stream order - between the encode_device hop queued
    before it and the one queued after it.  The packets equal a twin that ran the same sequence with host-buffer calls."""
    import torch
    n, bits = 1024, 184
    P = _capi.packet_bytes(bits)
    sbits = mc.interleaved(n, bc.COMMON)
    rng = np.random.default_rng(4)
    pcm = [rng.integers(-8000, 8000, size=(n, 320), dtype=np.int16) for _ in range(2)]
    ctx, twin = _capi.Context(n, roles="encoder"), _capi.Context(n, roles="encoder")
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    d_pcm = [torch.from_numpy(x).cuda() for x in pcm]
    d_pk = [torch.zeros((n, P), dtype=torch.uint8, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        ctx.encode_device(n, d_pcm[0].data_ptr(), bits, d_pk[0].data_ptr())
        ctx.set_stream_bits("encoder", sbits)
        assert not s.query(), "set_stream_bits waited for the GPU"
        ctx.encode_device(n, d_pcm[1].data_ptr(), bits, d_pk[1].data_ptr())
        assert not s.query()
    s.synchronize()
    want0 = twin.encode(pcm[0], bits)
    twin.set_stream_bits("encoder", sbits)
    want1 = twin.encode(pcm[1], bits)
    assert np.array_equal(d_pk[0].cpu().numpy(), want0), "the hop queued before the setter must run at the call's bits"
    assert np.array_equal(d_pk[1].cpu().numpy(), want1), "the hop queued after the setter must run at the streams' own bits"
    assert not np.array_equal(want0, want1)
    assert np.array_equal(ctx.stream_bits("encoder"), sbits)
    ctx.close()
    twin.close()


@pytest.mark.parametrize("mode,split", [("tensor", 2), ("exact", 3)])
def test_bench_device_schedule_with_mixed_bits(gpu_api, mode, split):
    """bench.py's device-resident schedule with per-stream bit counts: 2 context pairs of 1540 streams called at 184 bits, the
    streams at 64 / 120 / 184 bits interleaved, 12 hops over 8 rotating slots queued with no host synchronisation.  Every hop's
    packets and PCM equal host-buffer calls on single-bit-count twin pairs."""
    import torch
    import duplex_schedule as ds
    G, m, NBUF, hops, bits = 2, 1540, ds.NBUF, 12, 184
    n = G * m
    sbits = mc.interleaved(m, bc.COMMON)
    rng = np.random.default_rng(29)
    host_pcm = [rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16) for _ in range(NBUF)]
    sched = ds.Schedule(host_pcm, G, split, mode, bits, stream_bits=sbits, keep_hops=hops)
    ds.run([sched], hops)
    torch.cuda.synchronize()
    outs = [x.cpu().numpy() for x in sched.out]
    pks = [x.cpu().numpy() for x in sched.kept_pks]
    sel = {b: np.nonzero(sbits == b)[0] for b in bc.COMMON}
    refs = []
    for _ in range(G):
        pair = {}
        for b in bc.COMMON:
            re, rd = _capi.Context(m, roles="encoder"), _capi.Context(m, roles="decoder")
            rd.set_decoder_mode(mode)
            pair[b] = (re, rd)
        refs.append(pair)
    for i in range(hops):
        buf = i % NBUF
        for g, pair in enumerate(refs):
            for b, (re, rd) in pair.items():
                s = sel[b]
                rows = g * m + s
                pk = re.encode(host_pcm[buf][rows], b, stream_ids=s)
                pb = _capi.packet_bytes(b)
                assert np.array_equal(pks[i][rows, :pb], pk) and not pks[i][rows, pb:].any(), \
                    "packets of hop %d group %d at %d bits" % (i, g, b)
                bad = np.nonzero((outs[i][rows] != rd.decode(pk, b, stream_ids=s)).any(axis=1))[0]
                assert bad.size == 0, "PCM of hop %d group %d at %d bits differs at streams %s" % (i, g, b, rows[bad[:8]])
    sched.close()
    for c in [c for pair in refs for p in pair.values() for c in p]:
        c.close()
