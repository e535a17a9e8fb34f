"""CPU tier of the fused codec calls' launch counts and argument checks: the product kernels on the block emulator, small sizes,
one sub-batch.  The cases are in call_schedule_cases.py; the GPU tier adds dense calls over several sub-batches."""
import pytest

import call_schedule_cases as cs
import parity_cases as pc
from lyra_b200 import _capi


@pytest.mark.parametrize("setting", cs.SETTINGS)
def test_emu_launch_counts(emu_api, setting):
    cs.run_launch_counts(_capi.Context, emu_api, pc.HostMem(), setting=setting, max_streams=16, n=10, sparse_ids=[1, 4, 9, 14])


def test_emu_rejected_calls(emu_api):
    cs.run_rejections(_capi.Context, emu_api, pc.HostMem())
