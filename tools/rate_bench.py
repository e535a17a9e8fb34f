"""Throughput of the fused codec calls at external sample rates (lyra_b200_set_sample_rate).

Runs bench.py's device-resident duplex schedule (encoder-only / decoder-only context pairs over slices of shared buffers, caller
streams at priorities -1 / 0, encoder -> decoder events, 8 rotating slots, no host synchronisation inside a step) at each rate,
alternating the rates run by run in one process so clock and thermal drift hit them alike.  Then a torch.profiler pass at every
rate other than 16 kHz gives ResampleKernel's device time per launch.  Prints one line per run and a JSON summary.

  python tools/rate_bench.py [--streams 4096] [--steps 4] [--runs 3] [--rates 16000,48000,8000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lyra_b200 import _capi  # noqa: E402

NBUF = 8


class Schedule:
    """G encoder/decoder context pairs at one rate with their buffers."""

    def __init__(self, rate, n, groups, split, bits, mode):
        self.rate, self.n, self.bits, self.hop = rate, n, bits, rate // 50
        self.P = (bits + 7) // 8
        self.m = n // groups
        rng = np.random.default_rng(1234)
        self.pcm = [torch.from_numpy(rng.integers(-8192, 8192, size=(n, self.hop), dtype=np.int16)).cuda() for _ in range(NBUF)]
        self.pks = [torch.zeros((n, self.P), dtype=torch.uint8, device="cuda") for _ in range(NBUF)]
        self.out = torch.zeros((n, self.hop), dtype=torch.int16, device="cuda")
        self.groups = []
        for _ in range(groups):
            e_ = _capi.Context(self.m, roles="encoder")
            d_ = _capi.Context(self.m, roles="decoder")
            d_.set_decoder_mode(mode)
            gx, gy = torch.cuda.Stream(priority=-1), torch.cuda.Stream(priority=0)
            for c, prio, st in ((e_, -1, gx), (d_, 0, gy)):
                c.set_sample_rate(rate)
                c.set_priority(prio)
                c.set_stream(st.cuda_stream)
                c.set_split(split)
            self.groups.append((e_, d_, gx, gy))
        self.ev_pk = [[torch.cuda.Event() for _ in range(NBUF)] for _ in range(groups)]
        self.ev_free = [[torch.cuda.Event() for _ in range(NBUF)] for _ in range(groups)]

    def run(self, hops):
        """bench.py run_device: hop i's encode waits until the ring slot's previous packets are decoded."""
        row = 2 * self.hop
        for i in range(hops):
            b = i % NBUF
            for g, (e_, d_, gx, gy) in enumerate(self.groups):
                off = g * self.m
                if i >= NBUF:
                    gx.wait_event(self.ev_free[g][b])
                e_.encode_device(self.m, self.pcm[b].data_ptr() + off * row, self.bits, self.pks[b].data_ptr() + off * self.P)
                self.ev_pk[g][b].record(gx)
                gy.wait_event(self.ev_pk[g][b])
                d_.decode_device(self.m, self.pks[b].data_ptr() + off * self.P, 0, self.bits, self.out.data_ptr() + off * row)
                self.ev_free[g][b].record(gy)

    def timed(self, hops):
        timer = torch.cuda.Stream()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(timer)
        for _, _, gx, gy in self.groups:
            gx.wait_stream(timer)
            gy.wait_stream(timer)
        self.run(hops)
        for _, _, gx, gy in self.groups:
            timer.wait_stream(gx)
            timer.wait_stream(gy)
        e1.record(timer)
        torch.cuda.synchronize()
        return self.n * hops / (e0.elapsed_time(e1) / 1e3)

    def close(self):
        for e_, d_, _, _ in self.groups:
            e_.close()
            d_.close()


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def resample_kernel_us(sched, hops):
    """Mean device time of one ResampleKernel launch (torch.profiler, CUDA activity) over `hops` hops of the schedule."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sched.run(hops)
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.events():            # CUDA activity only: kernel and copy records, named after the kernel
        if "ResampleKernel" in ev.name:
            total += ev.time_range.elapsed_us()
            count += 1
    return (total / count if count else None), count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=4, help="timed steps per run; one step = --hops-per-step hops")
    ap.add_argument("--hops-per-step", type=int, default=50)
    ap.add_argument("--runs", type=int, default=3, help="runs per rate, alternating the rates")
    ap.add_argument("--rates", default="16000,48000,8000")
    ap.add_argument("--groups", type=int, default=2)
    ap.add_argument("--split", type=int, default=2)
    ap.add_argument("--bits", type=int, default=64, help="64 bits per 20 ms hop = 3.2 kbps")
    ap.add_argument("--decoder-mode", default="tensor", choices=["exact", "tensor"])
    ap.add_argument("--profile-hops", type=int, default=10)
    args = ap.parse_args()
    rates = [int(r) for r in args.rates.split(",")]
    scheds = {r: Schedule(r, args.streams, args.groups, args.split, args.bits, args.decoder_mode) for r in rates}
    for s in scheds.values():
        s.run(NBUF + 2)                      # warm-up: first launches, stream maps
    torch.cuda.synchronize()
    hops = args.steps * args.hops_per_step
    fps = {r: [] for r in rates}
    for run in range(args.runs):
        for r in rates:
            v = scheds[r].timed(hops)
            fps[r].append(v)
            print("run %d  %5d Hz  %.3f M frames/s" % (run, r, v / 1e6), flush=True)
    base = rates[0]
    med = {r: float(np.median(v)) for r, v in fps.items()}
    kernel = {}
    for r in rates:
        if r != 16000:
            us, cnt = resample_kernel_us(scheds[r], args.profile_hops)
            kernel[r] = {"ms_per_launch": None if us is None else us / 1e3, "launches": cnt}
    for s in scheds.values():
        s.close()
    res = {
        "gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "streams": args.streams, "bits": args.bits,
        "decoder_mode": args.decoder_mode, "split": args.split, "groups": args.groups, "hops_per_run": hops,
        "frames_per_s": {str(r): v for r, v in fps.items()}, "median_frames_per_s": {str(r): v for r, v in med.items()},
        "ratio_to_%d" % base: {str(r): med[r] / med[base] for r in rates},
        "resample_kernel": {str(r): v for r, v in kernel.items()},
    }
    for r in rates:
        print("%5d Hz: median %.3f M frames/s, %.3f x %d Hz" % (r, med[r] / 1e6, med[r] / med[base], base))
    for r, v in kernel.items():
        if v["ms_per_launch"] is not None:
            print("ResampleKernel at %d Hz: %.1f us per launch (%d launches of %d streams / group / part)" % (
                r, v["ms_per_launch"] * 1e3, v["launches"], args.streams // args.groups))
    print("GPU %s, power limit %s" % (res["gpu"], res["power_limit"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
