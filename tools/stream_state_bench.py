"""Cost of moving live streams (lyra_b200_copy_streams / _align_streams / _export_streams / _import_streams): copy_streams (up to
half the streams: the top k into the bottom k) and align_streams of 1, 64, 1024 and 4096 streams inside a 4096-stream context
(CUDA events around --reps calls on the installed stream), and export / import of 4096 streams to / from page-locked host memory (host clock; both calls end in a device
synchronise).  Algorithmic bytes = record payload x streams, read + write, for a copy; for an align, the ring words it rotates
(every ring of the four networks, read + write).  What a move leaves behind, tiles whose streams run on different hop
counters, is the mixed-counters configuration of tools/schedule_bench.py; aligned-counters is the same after align_streams.

  python tools/stream_state_bench.py [--streams 4096] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lyra_b200 import _capi  # noqa: E402
from schedule_bench import power_limit  # noqa: E402

HBM_TBPS = 3.35          # H100 SXM data sheet


# 4-byte ring words per stream that an align moves (kDwRings in net_kernels.cuh: the 6- and 18-row rings; every layer runs an
# even number of rows per hop, so the 2-row rings never rotate): encoder_0, encoder_1, quant_encoder_2, quant_decoder_0,
# decoder_1, decoder_2
RING_WORDS = (6 + 18) * (64 + 128 + 64 + 64 + 128 + 64)


def move_times(n_streams, sizes, reps, what):
    """what = "copy": the top k streams into the bottom k.  what = "align": streams 2 .. k + 1 of a context of n_streams + 2
    like stream 0 and like stream 1 in turn, which sit one hop apart in every network, so every call rotates every ring."""
    ctx = _capi.Context(n_streams if what == "copy" else n_streams + 2)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    per_stream = ctx.stream_state_bytes() - 64 if what == "copy" else 4 * RING_WORDS
    if what == "align":
        ctx.encode(np.zeros((1, 320), np.int16), 64, stream_ids=[1])
        ctx.decode(np.zeros((1, 8), np.uint8), 64, stream_ids=[1])
    out = {}
    for k in sizes:
        if what == "copy":
            src, dst = np.arange(n_streams - k, n_streams, dtype=np.int32), np.arange(k, dtype=np.int32)
            call = lambda: ctx.copy_streams(src, dst)                                        # noqa: E731
        else:
            dst, like, turn = np.arange(2, k + 2, dtype=np.int32), [np.zeros(k, np.int32), np.ones(k, np.int32)], [0]

            def call():
                ctx.align_streams(dst, like[turn[0]])
                turn[0] ^= 1
        call()                                                         # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(reps):
            call()
        e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        nbytes = 2 * per_stream * k
        out[k] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6, "share_of_hbm": nbytes / ms / 1e9 / HBM_TBPS}
        print("%s_streams %5d streams: %.4f ms, %.1f MB read+write, %.1f GB/s (%.2f %% of %.2f TB/s)" % (
            what, k, ms, nbytes / 1e6, out[k]["GB_per_s"], 100 * out[k]["share_of_hbm"], HBM_TBPS), flush=True)
    ctx.close()
    return out


def export_import_times(n_streams, reps):
    ctx = _capi.Context(n_streams)
    rb = ctx.stream_state_bytes()
    host = torch.empty(n_streams * rb, dtype=torch.uint8, pin_memory=True)
    ptr = C.c_void_p(host.data_ptr())
    lib = ctx.api.lib
    res = {}
    for name, fn in (("export", lambda: lib.lyra_b200_export_streams(ctx.h, None, n_streams, ptr)),
                     ("import", lambda: lib.lyra_b200_import_streams(ctx.h, None, n_streams, ptr))):
        assert fn() == 0, ctx.api.lib.lyra_b200_last_error(ctx.h)       # warm-up (allocates the staging)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            assert fn() == 0
            ts.append(time.perf_counter() - t0)
        ms = 1e3 * float(np.median(ts))
        nbytes = 2 * rb * n_streams
        res[name] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6, "share_of_hbm": nbytes / ms / 1e9 / HBM_TBPS}
        print("%s_streams %d streams to/from pinned host memory: %.2f ms, %.1f MB read+write, %.1f GB/s (%.3f %% of %.2f TB/s)" % (
            name, n_streams, ms, nbytes / 1e6, res[name]["GB_per_s"], 100 * res[name]["share_of_hbm"], HBM_TBPS), flush=True)
    ctx.close()
    return res, rb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--sizes", default="1,64,1024,4096", help="streams per copy_streams / align_streams call")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_state_bench needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "streams": args.streams}
    print("GPU %s, power limit %s" % (res["gpu"], res["power_limit"]), flush=True)
    sizes = [int(x) for x in args.sizes.split(",")]
    res["copy_streams"] = move_times(args.streams, [k for k in sizes if k <= args.streams // 2], args.reps, "copy")
    res["align_streams"] = move_times(args.streams, sizes, args.reps, "align")
    res["export_import"], res["record_bytes"] = export_import_times(args.streams, 3)
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_state_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
