"""GPU tier (H100) of the fused codec calls' launch counts and argument checks (call_schedule_cases.py): the CPU tier's cases at
a larger size, and dense calls over 4096 streams cut into 1, 2 and 3 sub-batches."""
import pytest

import call_schedule_cases as cs
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("setting", cs.SETTINGS)
def test_launch_counts(gpu_api, setting):
    cs.run_launch_counts(_capi.Context, gpu_api, TorchMem(), setting=setting, max_streams=100, n=100, sparse_ids=[0, 1, 17, 63, 99])


@pytest.mark.parametrize("setting", cs.SETTINGS)
def test_launch_counts_4096_streams_split(gpu_api, setting):
    cs.run_launch_counts(_capi.Context, gpu_api, TorchMem(), setting=setting, max_streams=4096, n=4096, splits=(1, 2, 3))


def test_rejected_calls(gpu_api):
    cs.run_rejections(_capi.Context, gpu_api, TorchMem())
