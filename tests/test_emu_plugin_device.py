"""CPU tier of the device twins of the plugin-level calls: the product kernels on the block emulator, a few tiles.  The cases are
in plugin_device_cases.py; the GPU tier runs them at full size with sub-batches engaged."""
import pytest

import plugin_device_cases as pd
import parity_cases as pc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("n", [1, 12])
@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_emu_plugin_device_nets(emu_api, n, mode):
    pd.run_nets_twin(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=n, hops=3, mode=mode)


@pytest.mark.parametrize("indices", [True, False])
@pytest.mark.parametrize("bits", [64, 120, 184])
def test_emu_plugin_device_rvq(emu_api, bits, indices):
    pd.run_rvq_twin(_capi.Context, emu_api, pc.HostMem(), n=12, hops=2, bits=bits, indices=indices)


def test_emu_plugin_device_rvq_one_row_decoder_context(emu_api):
    pd.run_rvq_twin(_capi.Context, emu_api, pc.HostMem(), n=1, hops=2, bits=120, indices=True, roles="decoder")


@pytest.mark.parametrize("n", [1, 12])
def test_emu_plugin_device_logmel(emu_api, n):
    pd.run_logmel_twin(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=n, hops=3)


@pytest.mark.parametrize("n", [1, 12])
def test_emu_plugin_device_cng(emu_api, n):
    pd.run_cng_twin(_capi.Context, emu_api, pc.HostMem(), n=n, hops=3)


@pytest.mark.parametrize("n", [1, 12])
def test_emu_plugin_device_noise_estimate(emu_api, n):
    pd.run_noise_twin(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=n, hops=6)


@pytest.mark.parametrize("to_internal", [1, 0])
@pytest.mark.parametrize("rate", pd.RESAMPLE_RATES)
def test_emu_plugin_device_resample(emu_api, rate, to_internal):
    pd.run_resample_twin(_capi.Context, emu_api, pc.HostMem(), n=12, hops=4, rate=rate, to_internal=to_internal)


@pytest.mark.parametrize("mode", ["exact", "tensor"])
def test_emu_plugin_device_chain(emu_api, oracle, mode):
    pd.run_chain(_capi.Context, emu_api, pc.HostMem(), _wav16(), oracle, n=12, hops=3, mode=mode, oracle_rows=(0, 11))


def test_emu_plugin_device_cng_chain(emu_api):
    pd.run_cng_chain(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=12, hops=4)


def test_emu_plugin_device_refusals(emu_api):
    pd.run_refusals(_capi.Context, emu_api, pc.HostMem())


def test_emu_plugin_device_mask_ignored(emu_api):
    """with an active mask that sits streams out installed, every twin gives what its host twin gives"""
    mem, wav = pc.HostMem(), _wav16()
    pd.run_nets_twin(_capi.Context, emu_api, mem, wav, n=12, hops=2, mask=True)
    pd.run_rvq_twin(_capi.Context, emu_api, mem, n=12, hops=1, bits=64, indices=True, mask=True)
    pd.run_logmel_twin(_capi.Context, emu_api, mem, wav, n=12, hops=2, banks_bins=((1, 160),), mask=True)
    pd.run_cng_twin(_capi.Context, emu_api, mem, n=12, hops=2, mask=True)
    pd.run_noise_twin(_capi.Context, emu_api, mem, wav, n=12, hops=3, mask=True)
    pd.run_resample_twin(_capi.Context, emu_api, mem, n=12, hops=2, rate=32000, to_internal=0, mask=True)
