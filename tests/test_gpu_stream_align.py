"""GPU tier (H100): lyra_b200_align_streams at full size.  4096 streams on every counter residue are aligned like one stream in
one call (four launches of 1024 ids) and continue bit for bit against a twin that was not aligned, in both decoder modes and at
split 2 and 3; the records, compaction and validation cases of the CPU tier at full size."""
import numpy as np
import pytest

import stream_align_cases as ac
from lyra_b200 import _capi
from test_gpu_parity import TorchMem

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,split", [("exact", 2), ("tensor", 3)])
def test_continuation_every_rotation(gpu_api, sample1, mode, split):
    ac.run_continuation(_capi.Context, gpu_api, sample1, n=4096, mode=mode, split=split, like=1000)


@pytest.mark.parametrize("roles", ["encoder", "decoder"])
def test_continuation_one_role(gpu_api, sample1, roles):
    ac.run_continuation(_capi.Context, gpu_api, sample1, n=1100, roles=roles, split=2)


def test_records(gpu_api, sample1):
    ac.run_records(_capi.Context, gpu_api, sample1, n=1100, x=1083, y=7, spare=1099)


def test_realign_after_skipped_hops(gpu_api, sample1):
    ac.run_realign_after_skips(_capi.Context, gpu_api, sample1, n=1100, dtx=(3, 12, 1093), lossy=(5, 9, 1090))


def test_compaction_with_alignment(gpu_api, sample1):
    ac.run_compaction_with_alignment(_capi.Context, gpu_api, TorchMem(), sample1, n0=1100, hops=14,
                                     churn={3: (40, 0), 6: (0, 12), 9: (25, 6), 11: (10, 3)})


def test_validation(gpu_api, sample1):
    ac.run_validation(_capi.Context, gpu_api, sample1, _capi.LyraB200Error, max_streams=1100, ids=(2, 5, 1099))
