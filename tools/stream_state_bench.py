"""Cost of moving live streams (lyra_b200_copy_streams / _export_streams / _import_streams): copy_streams of 1, 64 and 1024
streams inside a 4096-stream context (CUDA events around --reps calls on the installed stream), and export / import of 4096
streams to / from page-locked host memory (host clock; both calls end in a device synchronise).  Algorithmic bytes = record
payload x streams, read + write.  What a move leaves behind, tiles whose streams run on different hop counters, is the
mixed-counters configuration of tools/schedule_bench.py.

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


def copy_times(n_streams, sizes, reps):
    ctx = _capi.Context(n_streams)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    payload = ctx.stream_state_bytes() - 64
    out = {}
    for k in sizes:
        src = np.arange(n_streams - k, n_streams, dtype=np.int32)      # the top k streams into the bottom k
        dst = np.arange(k, dtype=np.int32)
        ctx.copy_streams(src, dst)                                     # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(reps):
            ctx.copy_streams(src, dst)
        e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        nbytes = 2 * payload * k
        out[k] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6, "share_of_hbm": nbytes / ms / 1e9 / HBM_TBPS}
        print("copy_streams %5d streams: %.4f ms, %.1f MB read+write, %.1f GB/s (%.2f %% of %.2f TB/s)" % (
            k, ms, nbytes / 1e6, out[k]["GB_per_s"], 100 * out[k]["share_of_hbm"], HBM_TBPS), flush=True)
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
    ap.add_argument("--copy-sizes", default="1,64,1024")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_state_bench needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "streams": args.streams}
    print("GPU %s, power limit %s" % (res["gpu"], res["power_limit"]), flush=True)
    res["copy_streams"] = copy_times(args.streams, [int(x) for x in args.copy_sizes.split(",")], args.reps)
    res["export_import"], res["record_bytes"] = export_import_times(args.streams, 3)
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_state_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
