"""CPU tier of per-stream sample rates (lyra_b200_set_stream_sample_rates): the product kernels on the block emulator, small
sizes.  The cases are in mixed_rate_cases.py; the GPU tier runs them at full size."""
import mixed_rate_cases as mc
import parity_cases as pc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wavs():
    return {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}


def test_emu_mixed_rates_at_48khz_sparse(emu_api, oracle):
    # tiles 0 and 1 each mix all four rates; rows 0-3 (one per rate) are also checked against the oracle
    mc.run_mixed_parity(_capi.Context, emu_api, oracle, _wavs(), ctx_rate=48000, rates=mc.ALL_RATES, max_streams=16,
                        stream_ids=[0, 1, 2, 3, 9, 12, 14, 15], frames=10, oracle_rows=range(4))


def test_emu_8khz_streams_in_a_16khz_context_dense(emu_api, oracle):
    mc.run_mixed_parity(_capi.Context, emu_api, oracle, _wavs(), ctx_rate=16000, rates=(8000, 16000), max_streams=10, n=10,
                        frames=10, oracle_rows=(0, 1))


def test_emu_mixed_rates_device_twins(emu_api, oracle):
    # guarded caller buffers; the GPU tier runs the device calls at 4096 streams in both decoder modes
    mc.run_mixed_parity(_capi.Context, emu_api, oracle, _wavs(), ctx_rate=48000, rates=(48000, 8000, 32000, 16000), max_streams=10,
                        n=10, frames=10, oracle_rows=(1,), mem=pc.HostMem())


def test_emu_rate_change_mid_call(emu_api, oracle):
    mc.run_rate_change_mid_call(_capi.Context, emu_api, oracle, _wavs())


def test_emu_moves_carry_the_rate(emu_api):
    mc.run_moves(_capi.Context, emu_api, _wavs())


def test_emu_validation(emu_api):
    mc.run_validation(_capi.Context, emu_api, _wavs(), _capi.LyraB200Error)


def test_emu_16khz_unchanged(emu_api):
    mc.run_16khz_unchanged(_capi.Context, emu_api, read_wav_any("sample1_16kHz.wav", 16000))
