#!/usr/bin/env python3
"""Dev tool (GPU): per-kernel serialized device times (engine CUDA events, split = 1) for both decoder modes."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lyra_b200 import _capi  # noqa

def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    rng = np.random.default_rng(0)
    pcm = rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16)
    for mode in ("exact", "tensor"):
        ctx = _capi.Context(n)
        ctx.set_decoder_mode(mode)
        ctx.set_split(1)
        for _ in range(3):
            pk = ctx.encode(pcm, 64)
            ctx.decode(pk, 64)
        ctx.profile_enable(True)
        for _ in range(20):
            pk = ctx.encode(pcm, 64)
            out = ctx.decode(pk, 64)
        prof = {k: v for k, v in ctx.profile_read().items() if v[1]}
        print(mode, " ".join("%s %.1fus" % (k, 1e3 * v[0] / v[1]) for k, v in prof.items()),
              "| sum %.1fus" % sum(1e3 * v[0] / v[1] for v in prof.values()), "checksum", int(out.astype(np.int64).sum()))
        ctx.close()


if __name__ == "__main__":
    main()
