"""GPU tier (H100) of the tensor-mode decoder's error profile (tensor_accuracy_cases): dense decoder-only contexts of 4100 streams
(the last tile holds 4) with their sub-batches engaged, split 2 and 3; decode_plc, sparse calls, replaced states and lanes that
sit out at full size.  The measured clean numbers are in tensor_accuracy_cases' docstring."""
import pytest

import tensor_accuracy_cases as ta
from conftest import read_wav
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu

N = 4100


@pytest.fixture(scope="module")
def wavs():
    return [read_wav("sample1_16kHz.wav"), read_wav("sample2_16kHz.wav")]


@pytest.mark.parametrize("split", [2, 3])
def test_tensor_profile_decode(gpu_api, oracle, wavs, split):
    ta.check_profile("decode / decode_device, split %d" % split,
                     ta.run_decode(_capi.Context, gpu_api, oracle, TorchMem(), wavs, n=N, hops=24, split=split))


def test_tensor_profile_decode_plc(gpu_api, oracle, wavs):
    ta.check_profile("decode_plc", ta.run_decode_plc(_capi.Context, gpu_api, oracle, wavs, n=N, hops=20))


def test_tensor_profile_sparse_and_replaced(gpu_api, wavs):
    ta.check_profile("sparse calls, replaced states", ta.run_sparse_and_replaced(_capi.Context, gpu_api, wavs, max_streams=N, hops=10))


def test_tensor_profile_sat_out_lanes(gpu_api, wavs):
    ta.check_profile("decode_device, lanes sitting out", ta.run_sat_out_lanes(_capi.Context, gpu_api, TorchMem(), wavs, n=N, hops=8))
