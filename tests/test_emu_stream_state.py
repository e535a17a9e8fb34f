"""CPU tier: moving live streams (lyra_b200_export_streams / _import_streams / _copy_streams) on the emulated kernels, small
sizes.  The cases are in stream_state_cases.py; the GPU tier runs them at full size."""
import parity_cases as pc
import stream_state_cases as sc
from conftest import read_wav_any
from lyra_b200 import _capi


def test_emu_move_between_contexts(emu_api, sample1):
    # 20 streams = tiles 0, 1 and a partial tile 2 (16..19).  1 -> 18: another lane in the partial last tile, next to B's live
    # stream 19; 6 -> 3 and 14 -> 7: tile 0, shared with B's live stream 4; 9 -> 12: the same tile, another lane
    sc.run_move_between_contexts(_capi.Context, emu_api, sample1, max_streams=20, a_ids=[1, 6, 9, 14], a_fill=[0, 16],
                                 b_ids=[18, 3, 12, 7], b_live=[4, 19], hops=9, after=2)


def test_emu_move_between_contexts_tensor_mode(emu_api, sample1):
    sc.run_move_between_contexts(_capi.Context, emu_api, sample1, max_streams=16, a_ids=[2, 9], a_fill=[5], b_ids=[13, 0],
                                 b_live=[14], hops=9, after=2, mode="tensor")


def test_emu_move_at_48k(emu_api):
    sc.run_move_at_48k(_capi.Context, emu_api, read_wav_any("sample1_48kHz.wav", 48000), _capi.LyraB200Error, hops=10, after=2)


def test_emu_compaction_on_the_device_path(emu_api, sample1):
    sc.run_compaction_on_the_device_path(_capi.Context, emu_api, pc.HostMem(), sample1, n0=20, hops=12,
                                         churn={3: (4, 0), 5: (0, 2), 8: (3, 2)})


def test_emu_round_trip_and_reset(emu_api, sample1):
    sc.run_round_trip_and_reset(_capi.Context, emu_api, sample1)


def test_emu_validation(emu_api, sample1):
    sc.run_validation(_capi.Context, emu_api, sample1, _capi.LyraB200Error)


def test_emu_record_size_follows_the_roles(emu_api):
    sizes = {r: _capi.Context(8, capi=emu_api, roles=r).stream_state_bytes() for r in ("both", "encoder", "decoder")}
    assert sizes["both"] > sizes["encoder"] > 64 and sizes["both"] > sizes["decoder"] > 64
    assert emu_api.lib.lyra_b200_stream_state_bytes(None) == 0

