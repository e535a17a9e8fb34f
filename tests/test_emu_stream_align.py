"""CPU tier: lyra_b200_align_streams on the emulated kernels, small sizes.  The cases are in stream_align_cases.py; the GPU tier
runs them at full size."""
import numpy as np
import pytest

import parity_cases as pc
import stream_align_cases as ac
from conftest import read_wav_any
from lyra_b200 import _capi


@pytest.mark.parametrize("roles,mode", [("both", "exact"), ("both", "tensor"), ("encoder", "exact"), ("decoder", "exact")])
def test_emu_continuation_every_rotation(emu_api, sample1, roles, mode):
    ac.run_continuation(_capi.Context, emu_api, sample1, n=24, roles=roles, mode=mode)


def test_emu_continuation_at_48k_with_stream_rates_and_bits(emu_api):
    n = 24

    def setup(c):
        c.set_sample_rate(48000)
        c.set_stream_sample_rates(np.asarray([8000, 16000, 32000, 48000] * (n // 4), np.int32))
        c.set_stream_bits("encoder", np.asarray([64, 0, 120] * (n // 3), np.int32))
        c.set_stream_bits("decoder", np.asarray([0, 120, 64] * (n // 3), np.int32))
    ac.run_continuation(_capi.Context, emu_api, read_wav_any("sample1_48kHz.wav", 48000), n=n, bits=120, hop=960, setup=setup)


def test_emu_records(emu_api, sample1):
    ac.run_records(_capi.Context, emu_api, sample1)


def test_emu_realign_after_skipped_hops(emu_api, sample1):
    ac.run_realign_after_skips(_capi.Context, emu_api, sample1)


def test_emu_compaction_with_alignment(emu_api, sample1):
    ac.run_compaction_with_alignment(_capi.Context, emu_api, pc.HostMem(), sample1, n0=20, hops=12,
                                     churn={3: (4, 0), 5: (0, 2), 8: (3, 2)})


def test_emu_validation(emu_api, sample1):
    ac.run_validation(_capi.Context, emu_api, sample1, _capi.LyraB200Error)
