"""CPU tier of the tensor-mode decoder's error profile (tensor_accuracy_cases): the product kernels on the block simulator, at
a few tiles.  The simulator's MMA model adds each k8 step in double, so it is more accurate than the hardware; the thresholds are
the GPU tier's."""
import pytest

import tensor_accuracy_cases as ta
from conftest import read_wav
from lyra_b200 import _capi
from parity_cases import HostMem


@pytest.fixture(scope="module")
def wavs():
    return [read_wav("sample1_16kHz.wav"), read_wav("sample2_16kHz.wav")]


def test_emu_tensor_profile_decode(emu_api, oracle, wavs):
    # two tiles, the last holding 4 streams
    ta.check_profile("decode / decode_device", ta.run_decode(_capi.Context, emu_api, oracle, HostMem(), wavs, n=12, hops=24))


def test_emu_tensor_profile_decode_plc(emu_api, oracle, wavs):
    ta.check_profile("decode_plc", ta.run_decode_plc(_capi.Context, emu_api, oracle, wavs, n=8, hops=14))


def test_emu_tensor_profile_sparse_and_replaced(emu_api, wavs):
    ta.check_profile("sparse calls, replaced states", ta.run_sparse_and_replaced(_capi.Context, emu_api, wavs, max_streams=28, hops=8))


def test_emu_tensor_profile_sat_out_lanes(emu_api, wavs):
    ta.check_profile("decode_device, lanes sitting out", ta.run_sat_out_lanes(_capi.Context, emu_api, HostMem(), wavs, n=8, hops=6))
