"""GPU tier (H100) of the active mask of the *_device codec calls (lyra_b200_set_active_mask): 4096-stream device twins with their
sub-batches engaged in both decoder modes, mixed per-stream settings, an all-ones / all-zero mask, the oracle, and a mask
rewritten on the device between queued calls."""
import numpy as np
import pytest

import active_mask_cases as am
import mixed_rate_cases as mc
import rate_cases as rc
from conftest import read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("split,mode", [(2, "exact"), (3, "tensor")])
@pytest.mark.parametrize("kind", am.KINDS)
def test_active_mask_twin_4096(gpu_api, kind, split, mode):
    am.run_twin(_capi.Context, gpu_api, TorchMem(), {16000: _wav16()}, kind, n=4096, hops=18 if kind == "decode_plc" else 10,
                split=split, mode=mode)


@pytest.mark.parametrize("kind", am.KINDS)
def test_active_mask_mixed_settings(gpu_api, kind):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    am.run_twin(_capi.Context, gpu_api, TorchMem(), wavs, kind, n=1200, hops=18 if kind == "decode_plc" else 10, split=2,
                ctx_rate=48000, rates=(8000, 16000, 48000), bits=184, bit_set=(64, 120, 184), dtx=[k % 3 != 1 for k in range(1200)])


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_active_mask_ones_zeros_and_launches(gpu_api, mode):
    am.run_ones_zeros_and_launches(_capi.Context, gpu_api, TorchMem(), _wav16(), n=4096, split=3, mode=mode)


def test_active_mask_oracle(gpu_api, oracle):
    am.run_oracle_spot(_capi.Context, gpu_api, oracle, TorchMem(), _wav16(), n=1024, hops=10, rows=(0, 5, 511, 1023))


def test_active_mask_setter(gpu_api):
    am.run_setter(_capi.Context, gpu_api, _capi.LyraB200Error)


def test_active_mask_rewritten_in_stream_order(gpu_api):
    """The mask is read when the kernels run: with a spin queued ahead on the installed stream, every hop's mask is copied into
    the one installed buffer by cudaMemcpyAsync between the queued encode_device / decode_device calls, and nothing waits for the
    GPU.  Packets and PCM equal a twin that ran each hop's active ids through the host-buffer calls."""
    import torch
    n, bits, hops = 2048, 64, 8
    P = _capi.packet_bytes(bits)
    wav = _wav16()
    rng = np.random.default_rng(6)
    pcm = [rc.speech_rows(wav, 16000, range(n), f) for f in range(hops)]
    masks = [am.hop_mask(f, n, rng) for f in range(hops)]
    ctx, twin = _capi.Context(n), _capi.Context(n)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    d_mask = torch.ones((n,), dtype=torch.uint8, device="cuda")
    ctx.set_active_mask(d_mask)
    h_masks = [torch.from_numpy(m).pin_memory() for m in masks]
    d_pcm = [torch.from_numpy(x).cuda() for x in pcm]
    d_pk = [torch.zeros((n, P), dtype=torch.uint8, device="cuda") for _ in range(hops)]
    d_out = [torch.zeros((n, 320), dtype=torch.int16, device="cuda") for _ in range(hops)]
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        for f in range(hops):
            d_mask.copy_(h_masks[f], non_blocking=True)
            ctx.encode_device(n, d_pcm[f].data_ptr(), bits, d_pk[f].data_ptr())
            ctx.decode_device(n, d_pk[f].data_ptr(), 0, bits, d_out[f].data_ptr())
        assert not s.query(), "a call or the mask copy waited for the GPU"
    s.synchronize()
    for f in range(hops):
        act = np.nonzero(masks[f])[0].astype(np.int32)
        pk, out = d_pk[f].cpu().numpy(), d_out[f].cpu().numpy()
        off = masks[f] == 0
        assert not pk[off].any() and not out[off].any(), "hop %d: a stream that sat out has a nonzero row" % f
        if len(act):
            w_pk = twin.encode(pcm[f][act], bits, stream_ids=act)
            assert np.array_equal(pk[act], w_pk), "hop %d: packets differ from the host-buffer twin" % f
            assert np.array_equal(out[act], twin.decode(w_pk, bits, stream_ids=act)), "hop %d: PCM differs from the twin" % f
    assert np.array_equal(ctx.export_streams(), twin.export_streams()), "stream records differ from the twin's"
    ctx.set_active_mask(None)
    ctx.close()
    twin.close()
