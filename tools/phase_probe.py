#!/usr/bin/env python3
"""Dev tool (GPU): per-phase clock64() breakdown of the four conv-net kernels using the -DLYRA_PHASE_PROF build
(devtools_build/liblyra_b200_phase.so: tools/build_variant.sh phase -DLYRA_PHASE_PROF).

usage: tools/phase_probe.py [streams] [split] [exact|tensor]    (decoder mode, default exact)"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa
from lyra_b200 import _capi  # noqa

NAMES = {
    0: ["loads(X,prefix,state)", "first_layer", "u0.dw", "u0.pw1", "u0.pw2", "u1.dw", "u1.pw1", "u1.pw2", "u2.dw", "u2.pw1", "u2.pw2", "down0.state", "down0 gemm+end"],
    1: ["loads", "r0.dw", "r0.pw1", "r0.pw2", "r1.dw", "r1.pw1", "r1.pw2", "r2.dw", "r2.pw1", "r2.pw2", "down1 state", "down1", "m.dw+pw1+pw2",
        "q0.dw", "q0.pw1", "q0.pw2", "q1.dw", "q1.pw1", "q1.pw2", "down2 state+gemm", "bott state", "bott"],
    2: ["loads", "bott", "up0", "lrelu+quant", "m.dw+pw1+pw2", "q0.dw", "q0.pw1", "q0.pw2", "q1.dw", "q1.pw1", "q1.pw2", "up1 prep", "up1",
        "r0.dw", "r0.pw1", "r0.pw2", "r1.dw", "r1.pw1", "r1.pw2", "r2.dw", "r2.pw1", "r2.pw2", "store"],
    3: ["loads", "up2", "u0.dw", "u0.pw1", "u0.pw2", "u1.dw", "u1.pw1", "u1.pw2", "u2.dw", "u2.pw1", "u2.pw2", "last+store"],
}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    api = _capi.CApi(os.environ.get("LYRA_PHASE_LIB", os.path.join(ROOT, "devtools_build", "liblyra_b200_phase.so")))
    api.lib.lyra_b200_debug_phases.restype = C.c_int
    api.lib.lyra_b200_debug_phases.argtypes = [C.c_void_p, C.c_void_p]
    ctx = _capi.Context(n, capi=api)
    if len(sys.argv) > 2:
        ctx.set_split(int(sys.argv[2]))          # 1 = one launch per kernel for the whole batch (no concurrent sub-batches)
    du = len(sys.argv) > 3 and sys.argv[3] == "tensor"
    if du:
        ctx.set_decoder_mode("tensor")           # kernel 3 is then DecoderKernelDW
    buf = np.zeros((4, 1024, 48), dtype=np.int64)
    api.lib.lyra_b200_debug_phases(ctx.h, buf.ctypes.data_as(C.c_void_p))      # arms the buffer
    rng = np.random.default_rng(0)
    pcm = rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16)
    for _ in range(3):
        pk = ctx.encode(pcm, 64)
        ctx.decode(pk, 64)
    api.lib.lyra_b200_debug_phases(ctx.h, buf.ctypes.data_as(C.c_void_p))
    nblk = min(1024, n // ctx.tile_streams)
    if du:
        NAMES[3] = ["loads+X", "up2 split (weight stream)", "up2 mma tail", "up2 epi"] + sum([["u%d ring wait" % i, "u%d dw" % i, "u%d ring upd" % i, "u%d pw1 mma" % i, "u%d epi1" % i,
                                                          "u%d pw2 mma" % i, "u%d epi2" % i] for i in range(3)], []) + ["last (4 taps)", "last epi+store"]
    for k in range(4):
        t = buf[k, :nblk]
        t = t[t[:, 0] != 0]                     # blocks that really stamped (sub-batches launch fewer blocks than the buffer holds)
        if not len(t):
            continue
        nph = int((t[0] != 0).sum())
        d = np.diff(t[:, :nph], axis=1).astype(np.float64)
        tot = d.sum(axis=1).mean()
        print("kernel %d: %d phases, mean block cycles %.0f" % (k, nph, tot))
        for i in range(nph - 1):
            nm = NAMES[k][i] if i < len(NAMES[k]) else "?"
            print("   %-24s %9.0f cyc  %5.1f%%" % (nm, d[:, i].mean(), 100 * d[:, i].mean() / tot))


if __name__ == "__main__":
    main()
