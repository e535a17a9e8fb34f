"""CPU tier of the fused codec calls at 8 / 32 / 48 kHz (lyra_b200_set_sample_rate): the product kernels on the block emulator
against the oracle composition of tests/rate_cases.py.  One rate per call kind here (the emulator is slow); the GPU tier runs
every rate."""
import parity_cases as pc
import rate_cases as rc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav(rate):
    return read_wav_any("sample1_%dkHz.wav" % (rate // 1000), rate)


def test_emu_fused_calls_at_48khz(emu_api, oracle):
    # sparse ids over two tiles (3 streams), every fused call, loss, bursts into comfort noise and back, bit-rate changes
    rc.run_rate_parity(_capi.Context, emu_api, oracle, _wav(48000), rate=48000, max_streams=16, stream_ids=[2, 7, 12], frames=12)


def test_emu_fused_calls_at_8khz_dense(emu_api, oracle):
    rc.run_rate_parity(_capi.Context, emu_api, oracle, _wav(8000), rate=8000, max_streams=10, n=10, frames=12, check=[0, 3, 8, 9],
                       calls=("plc", "dtx"))


def test_emu_equivalence_with_the_plugin_chain(emu_api):
    rc.run_equivalence_with_plugin_chain(_capi.Context, emu_api, rate=32000)


def test_emu_device_twins_at_32khz(emu_api):
    rc.run_device_twins(_capi.Context, emu_api, pc.HostMem(), _wav(32000), rate=32000, n=10, frames=4)


def test_emu_dtx_estimator_at_8khz(emu_api, oracle):
    rc.run_dtx_at_rate(_capi.Context, emu_api, oracle, _wav(8000), rate=8000, speech_hops=10, noise_hops=22)


def test_emu_rate_change_and_reset(emu_api, oracle):
    rc.run_rate_change_and_reset(_capi.Context, emu_api, oracle, {r: _wav(r) for r in (48000, 8000)}, _capi.LyraB200Error)


def test_emu_integration_criterion_at_8khz(emu_api, oracle):
    worst = rc.run_integration_at_rate(_capi.Context, emu_api, oracle, rate=8000, wav=_wav(8000), hops=14)
    assert worst < 2.0, worst
