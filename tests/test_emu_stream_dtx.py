"""CPU tier of per-stream DTX (lyra_b200_set_stream_dtx): the product kernels on the block emulator, small sizes.  The cases are
in stream_dtx_cases.py; the GPU tier runs them at full size."""
import mixed_rate_cases as mc
import parity_cases as pc
import stream_dtx_cases as dc
from conftest import read_wav_any
from lyra_b200 import _capi


def _wav16():
    return read_wav_any("sample1_16kHz.wav", 16000)


def test_emu_mixed_dtx_sparse(emu_api, oracle):
    # tiles 0 and 1 each mix DTX-on and DTX-off streams
    dc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, max_streams=16, stream_ids=[0, 1, 2, 3, 9, 12, 14, 15],
                        frames=12)


def test_emu_mixed_dtx_dense_split(emu_api, oracle):
    dc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, max_streams=10, n=10, frames=12, split=2, bits=120)


def test_emu_mixed_dtx_device_twin(emu_api, oracle):
    dc.run_mixed_parity(_capi.Context, emu_api, oracle, {16000: _wav16()}, max_streams=10, n=10, frames=12, mem=pc.HostMem())


def test_emu_dtx_with_stream_rates_and_bits(emu_api, oracle):
    wavs = {r: read_wav_any("sample1_%dkHz.wav" % (r // 1000), r) for r in mc.ALL_RATES}
    dc.run_mixed_parity(_capi.Context, emu_api, oracle, wavs, max_streams=12, n=12, frames=12, ctx_rate=48000, rates=mc.ALL_RATES,
                        bits=184, bit_set=(64, 120, 184), oracle_rows=(0, 1, 2, 3, 4, 5))


def test_emu_dtx_toggle(emu_api, oracle):
    dc.run_toggle(_capi.Context, emu_api, oracle, _wav16())


def test_emu_dtx_moves(emu_api):
    dc.run_moves(_capi.Context, emu_api, _wav16(), _capi.LyraB200Error)


def test_emu_dtx_validation(emu_api):
    dc.run_validation(_capi.Context, emu_api, _capi.LyraB200Error)


def test_emu_dtx_unchanged_when_unused(emu_api):
    dc.run_unchanged_when_unused(_capi.Context, emu_api, _wav16())
