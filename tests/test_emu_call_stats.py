"""CPU tier of the per-stream call statistics (lyra_b200_set_stats / _read_stats / _read_stats_device): the product kernels on the
block emulator, small sizes.  The cases are in call_stats_cases.py; the GPU tier runs them at full size."""
import pytest

import call_stats_cases as st
import mixed_rate_cases as mc
import parity_cases as pc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


def _wavs():
    return {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}


@pytest.mark.parametrize("call", ["dense", "sparse", "device"])
@pytest.mark.parametrize("kind", st.KINDS)
def test_emu_call_stats_kinds(emu_api, kind, call):
    st.run_kind(_capi.Context, emu_api, pc.HostMem(), {16000: _wav16()}, kind, n=10, hops=16 if kind == "decode_plc" else 6,
                sparse=call == "sparse", device=call == "device")


@pytest.mark.parametrize("kind", st.KINDS)
def test_emu_call_stats_mixed_settings(emu_api, kind):
    st.run_kind(_capi.Context, emu_api, pc.HostMem(), _wavs(), kind, n=12, hops=16 if kind == "decode_plc" else 6, ctx_rate=48000,
                rates=(8000, 16000, 48000), bits=184, bit_set=(64, 120, 184), dtx=[k % 3 != 1 for k in range(12)])


@pytest.mark.parametrize("kind", st.KINDS)
def test_emu_call_stats_active_mask(emu_api, kind):
    st.run_kind(_capi.Context, emu_api, pc.HostMem(), _wavs(), kind, n=12, hops=16 if kind == "decode_plc" else 8, device=True,
                masked=True, ctx_rate=48000, rates=(8000, 16000, 48000))


def test_emu_call_stats_tensor_mode(emu_api):
    st.run_kind(_capi.Context, emu_api, pc.HostMem(), {16000: _wav16()}, "decode_plc", n=8, hops=16, device=True, mode="tensor")


def test_emu_call_stats_levels(emu_api):
    st.run_levels(_capi.Context, emu_api)


@pytest.mark.parametrize("kind", ["encode_dtx", "decode_plc"])
def test_emu_call_stats_clear(emu_api, kind):
    st.run_clear(_capi.Context, emu_api, pc.HostMem(), {16000: _wav16()}, kind, n=6, hops=14 if kind == "decode_plc" else 5)


def test_emu_call_stats_travel(emu_api):
    st.run_travel(_capi.Context, emu_api, pc.HostMem(), _wav16())


def test_emu_call_stats_off_and_launches(emu_api):
    st.run_off_and_launches(_capi.Context, emu_api, pc.HostMem(), _wav16(), n=8, hops=2)


def test_emu_call_stats_unaligned_rows(emu_api):
    st.run_unaligned(_capi.Context, emu_api, pc.HostMem(), _wavs(), n=6, hops=1)


def test_emu_call_stats_argument_errors(emu_api):
    st.run_argument_errors(_capi.Context, emu_api, pc.HostMem())
