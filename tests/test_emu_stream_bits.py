"""CPU tier of per-stream bit counts (lyra_b200_set_stream_bits): the product kernels on the block emulator, small sizes.  The
cases are in stream_bits_cases.py; the GPU tier runs them at full size."""
import mixed_rate_cases as mc
import parity_cases as pc
import stream_bits_cases as bc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


def test_emu_mixed_bits_sparse(emu_api, oracle):
    # tiles 0 and 1 each mix 64 / 120 / 184 bits; rows 0-2 (one per count) are also checked against the oracle
    bc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, bit_set=bc.COMMON, max_streams=16,
                        stream_ids=[0, 1, 2, 3, 9, 12, 14, 15], frames=10, oracle_rows=range(3))


def test_emu_odd_bits_dense(emu_api, oracle):
    bc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, bit_set=bc.ODD, max_streams=10, n=10, frames=10,
                        oracle_rows=(0, 1))


def test_emu_mixed_bits_device_twins(emu_api, oracle):
    bc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, bit_set=(184, 60, 120, 4), max_streams=10, n=10,
                        frames=10, oracle_rows=(1,), mem=pc.HostMem())


def test_emu_bits_with_stream_sample_rates(emu_api, oracle):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    bc.run_mixed_parity(_capi.Context, emu_api, oracle, wavs, bit_set=bc.COMMON, max_streams=12, n=12, frames=10, ctx_rate=48000,
                        rates=mc.ALL_RATES, oracle_rows=(0, 1, 2, 3))


def test_emu_bits_change_between_hops(emu_api):
    bc.run_bits_change(_capi.Context, emu_api, _wav16())


def test_emu_validation(emu_api):
    bc.run_validation(_capi.Context, emu_api, _wav16(), _capi.LyraB200Error)


def test_emu_moves_carry_the_words(emu_api):
    bc.run_moves(_capi.Context, emu_api, _wav16())
    bc.run_refused_after_move(_capi.Context, emu_api, _capi.LyraB200Error)


def test_emu_unchanged_when_unused(emu_api):
    bc.run_unchanged_when_unused(_capi.Context, emu_api, _wav16())
