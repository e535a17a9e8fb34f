"""GPU tier (H100): moving live streams (lyra_b200_export_streams / _import_streams / _copy_streams) at full size, the
asynchrony of copy_streams and a move between two GPUs."""
import numpy as np
import pytest

import stream_state_cases as sc
from conftest import read_wav_any
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu

# 1100 streams: tiles 0..136 and a partial tile 137 (1096..1099).  1 -> 1096 and 1093 -> 1098: other lanes of the partial last
# tile, next to B's live streams 1097 / 1099; 6 -> 3, 14 -> 7: tile 0, shared with B's live stream 4; 517 -> 64: tile 8, shared
# with B's live stream 66
MOVE = dict(max_streams=1100, a_ids=[1, 6, 9, 14, 100, 517, 1090, 1093], a_fill=[0, 16, 700, 1099],
            b_ids=[1096, 3, 12, 7, 1001, 64, 250, 1098], b_live=[4, 1097, 66, 1099], hops=10, after=4)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_move_between_contexts(gpu_api, sample1, mode):
    sc.run_move_between_contexts(_capi.Context, gpu_api, sample1, mode=mode, **MOVE)


def test_move_at_48k(gpu_api):
    sc.run_move_at_48k(_capi.Context, gpu_api, read_wav_any("sample1_48kHz.wav", 48000), _capi.LyraB200Error, max_streams=1100,
                       a_ids=(2, 9, 13, 600, 1099), b_ids=(11, 0, 1097, 5, 640))


def test_compaction_on_the_device_path(gpu_api, sample1):
    sc.run_compaction_on_the_device_path(_capi.Context, gpu_api, TorchMem(), sample1, n0=1100, hops=14,
                                         churn={3: (40, 0), 6: (0, 12), 9: (25, 6), 11: (10, 3)})


def test_round_trip_and_reset(gpu_api, sample1):
    sc.run_round_trip_and_reset(_capi.Context, gpu_api, sample1, max_streams=1100, ids=(3, 8, 12, 1099, 500),
                                moved_to=(10, 1, 1098, 15, 77))


def test_validation(gpu_api, sample1):
    sc.run_validation(_capi.Context, gpu_api, sample1, _capi.LyraB200Error, max_streams=1100, ids=(2, 5, 11, 1099))


def test_copy_streams_is_asynchronous_and_ordered(gpu_api):
    """copy_streams returns while a spin queued ahead still occupies the caller stream; its effect lands after the device call
    queued before it and before the one queued after it: the packets equal a twin that ran the same steps synchronously."""
    import torch
    n, bits = 1024, 64
    rng = np.random.default_rng(17)
    pcm = [rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16) for _ in range(2)]
    src, dst = [5, 700, 1023, -1, 8], [900, 3, 12, 800, 9]
    enc = _capi.Context(n, roles="encoder")
    twin = _capi.Context(n, roles="encoder")
    s = torch.cuda.Stream()
    enc.set_stream(s.cuda_stream)
    enc.set_split(2)
    d_pcm = [torch.from_numpy(x).cuda() for x in pcm]
    d_pk = [torch.zeros((n, 8), dtype=torch.uint8, device="cuda") for _ in range(2)]
    for c in (enc, twin):                 # first launches (module loading) outside the checked window
        c.copy_streams([-1], [0])
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        enc.encode_device(n, d_pcm[0].data_ptr(), bits, d_pk[0].data_ptr())
        enc.copy_streams(src, dst)
        assert not s.query(), "copy_streams waited for the GPU"
        enc.encode_device(n, d_pcm[1].data_ptr(), bits, d_pk[1].data_ptr())
    s.synchronize()
    want0 = twin.encode(pcm[0], bits)
    twin.copy_streams(src, dst)
    want1 = twin.encode(pcm[1], bits)
    assert np.array_equal(d_pk[0].cpu().numpy(), want0)
    assert np.array_equal(d_pk[1].cpu().numpy(), want1), "copy_streams was not ordered between the device calls"
    enc.close()
    twin.close()


def test_move_between_gpus(gpu_api, sample1):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("a move between GPUs needs two CUDA devices; this machine has %d" % torch.cuda.device_count())
    sc.run_move_between_contexts(_capi.Context, gpu_api, sample1, devices=(0, 1), **MOVE)
