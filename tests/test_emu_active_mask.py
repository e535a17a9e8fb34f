"""CPU tier of the active mask of the *_device codec calls (lyra_b200_set_active_mask): the product kernels on the block emulator,
small sizes.  The cases are in active_mask_cases.py; the GPU tier runs them at full size."""
import pytest

import active_mask_cases as am
import mixed_rate_cases as mc
import parity_cases as pc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


@pytest.mark.parametrize("kind", am.KINDS)
def test_emu_active_mask_twin(emu_api, kind):
    am.run_twin(_capi.Context, emu_api, pc.HostMem(), {16000: _wav16()}, kind, n=16, hops=20 if kind == "decode_plc" else 12)


@pytest.mark.parametrize("kind", ["encode", "decode_plc"])
def test_emu_active_mask_twin_split_tensor(emu_api, kind):
    # the emulated contexts are too small for sub-batches: split 3 falls back to one part, like any call under 64 tiles per part
    am.run_twin(_capi.Context, emu_api, pc.HostMem(), {16000: _wav16()}, kind, n=16, hops=18, split=3, mode="tensor")


@pytest.mark.parametrize("kind", am.KINDS)
def test_emu_active_mask_mixed_settings(emu_api, kind):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    am.run_twin(_capi.Context, emu_api, pc.HostMem(), wavs, kind, n=12, hops=20 if kind == "decode_plc" else 12, ctx_rate=48000,
                rates=(8000, 16000, 48000), bits=184, bit_set=(64, 120, 184), dtx=[k % 3 != 1 for k in range(12)])


def test_emu_active_mask_ones_zeros_and_launches(emu_api):
    am.run_ones_zeros_and_launches(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=16)


def test_emu_active_mask_oracle(emu_api, oracle):
    am.run_oracle_spot(_capi.Context, emu_api, oracle, pc.HostMem(), _wav16(), n=10, hops=8, rows=(0, 3, 9))


def test_emu_active_mask_setter(emu_api):
    am.run_setter(_capi.Context, emu_api, _capi.LyraB200Error)
