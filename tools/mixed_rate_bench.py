"""Throughput of the fused codec calls with per-stream sample rates (lyra_b200_set_stream_sample_rates).

Runs bench.py's device-resident duplex schedule (encoder-only / decoder-only context pairs, caller streams at priorities -1 / 0,
encoder -> decoder events, 8 rotating slots, no host synchronisation inside a step) in three configurations, alternating them
run by run in one process so clock and thermal drift hit them alike:
  16k    the streams at 16 kHz in `--groups` context pairs (the benchmark's workload);
  mixed  the same context pairs at row rate 48 kHz, the streams in equal shares at 8 / 16 / 32 / 48 kHz, interleaved so that
         every tile mixes the four rates;
  split  the same traffic split by rate: one context pair per rate, each with a quarter of the streams (what a server without
         per-stream rates runs).
The card's name, power limit and the median SM clock sampled during the timed runs are recorded with the numbers.  Prints one
line per run and a JSON summary.

  python tools/mixed_rate_bench.py [--streams 4096] [--hops 200] [--runs 5]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lyra_b200 import _capi  # noqa: E402

NBUF = 8
RATES = (8000, 16000, 32000, 48000)


class Pair:
    """One encoder-only / decoder-only context pair at row rate `rate` over m streams with its own buffers; stream_rates: the
    streams' own rates (None: all at `rate`)."""

    def __init__(self, rate, m, split, bits, mode, stream_rates=None):
        self.m, self.bits, self.hop, self.P = m, bits, rate // 50, (bits + 7) // 8
        rng = np.random.default_rng(1234)
        self.pcm = [torch.from_numpy(rng.integers(-8192, 8192, size=(m, self.hop), dtype=np.int16)).cuda() for _ in range(NBUF)]
        self.pks = [torch.zeros((m, self.P), dtype=torch.uint8, device="cuda") for _ in range(NBUF)]
        self.out = torch.zeros((m, self.hop), dtype=torch.int16, device="cuda")
        self.enc, self.dec = _capi.Context(m, roles="encoder"), _capi.Context(m, roles="decoder")
        self.dec.set_decoder_mode(mode)
        self.gx, self.gy = torch.cuda.Stream(priority=-1), torch.cuda.Stream(priority=0)
        for c, prio, st in ((self.enc, -1, self.gx), (self.dec, 0, self.gy)):
            c.set_sample_rate(rate)
            c.set_priority(prio)
            c.set_stream(st.cuda_stream)
            c.set_split(split)
            if stream_rates is not None:
                c.set_stream_sample_rates(stream_rates)
        self.ev_pk = [torch.cuda.Event() for _ in range(NBUF)]
        self.ev_free = [torch.cuda.Event() for _ in range(NBUF)]

    def hop_(self, i):
        """bench.py run_device: hop i's encode waits until the ring slot's previous packets are decoded"""
        b = i % NBUF
        if i >= NBUF:
            self.gx.wait_event(self.ev_free[b])
        self.enc.encode_device(self.m, self.pcm[b].data_ptr(), self.bits, self.pks[b].data_ptr())
        self.ev_pk[b].record(self.gx)
        self.gy.wait_event(self.ev_pk[b])
        self.dec.decode_device(self.m, self.pks[b].data_ptr(), 0, self.bits, self.out.data_ptr())
        self.ev_free[b].record(self.gy)

    def close(self):
        self.enc.close()
        self.dec.close()


class Config:
    def __init__(self, pairs):
        self.pairs = pairs
        self.n = sum(p.m for p in pairs)

    def run(self, hops):
        for i in range(hops):
            for p in self.pairs:
                p.hop_(i)

    def timed(self, hops):
        timer = torch.cuda.Stream()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(timer)
        for p in self.pairs:
            p.gx.wait_stream(timer)
            p.gy.wait_stream(timer)
        self.run(hops)
        for p in self.pairs:
            timer.wait_stream(p.gx)
            timer.wait_stream(p.gy)
        e1.record(timer)
        torch.cuda.synchronize()
        return self.n * hops / (e0.elapsed_time(e1) / 1e3)

    def close(self):
        for p in self.pairs:
            p.close()


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


class ClockSampler:
    """SM clock (MHz) read with nvidia-smi every `period` s while the timed runs go on (read-only queries)"""

    def __init__(self, period=0.25):
        self.period, self.samples, self.stop = period, [], threading.Event()
        self.thread = threading.Thread(target=self._loop, daemon=True)

    def _loop(self):
        while not self.stop.wait(self.period):
            v = smi("clocks.sm")
            if v and v.replace(".", "").isdigit():
                self.samples.append(float(v))

    def __enter__(self):
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--hops", type=int, default=200, help="hops per timed run")
    ap.add_argument("--runs", type=int, default=5, help="runs per configuration, alternating the configurations")
    ap.add_argument("--groups", type=int, default=2)
    ap.add_argument("--split", type=int, default=2)
    ap.add_argument("--bits", type=int, default=64, help="64 bits per 20 ms hop = 3.2 kbps")
    ap.add_argument("--decoder-mode", default="tensor", choices=["exact", "tensor"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mixed_rate_bench needs a CUDA device")
    m = args.streams // args.groups
    q = args.streams // len(RATES)
    mix = np.array([RATES[k % len(RATES)] for k in range(m)], dtype=np.int32)
    mk = lambda rate, n, sr=None: Pair(rate, n, args.split, args.bits, args.decoder_mode, sr)   # noqa: E731
    configs = {
        "16k": Config([mk(16000, m) for _ in range(args.groups)]),
        "mixed": Config([mk(48000, m, mix) for _ in range(args.groups)]),
        "split": Config([mk(r, q) for r in RATES]),
    }
    for c in configs.values():
        c.run(NBUF + 2)                      # warm-up: first launches, stream maps
    torch.cuda.synchronize()
    fps = {k: [] for k in configs}
    with ClockSampler() as clocks:
        for run in range(args.runs):
            for k, c in configs.items():
                v = c.timed(args.hops)
                fps[k].append(v)
                print("run %d  %-5s  %.3f M frames/s" % (run, k, v / 1e6), flush=True)
    for c in configs.values():
        c.close()
    med = {k: float(np.median(v)) for k, v in fps.items()}
    res = {
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"),
        "median_sm_clock_mhz": float(np.median(clocks.samples)) if clocks.samples else None, "clock_samples": len(clocks.samples),
        "streams": args.streams, "bits": args.bits, "decoder_mode": args.decoder_mode, "split": args.split, "groups": args.groups,
        "hops_per_run": args.hops, "frames_per_s": fps, "median_frames_per_s": med,
        "spread": {k: [min(v) / med[k], max(v) / med[k]] for k, v in fps.items()},
        "ratio_to_16k": {k: v / med["16k"] for k, v in med.items()},
    }
    for k in configs:
        print("%-5s: median %.3f M frames/s (%.3f-%.3f), %.3f x 16k" % (k, med[k] / 1e6, min(fps[k]) / 1e6, max(fps[k]) / 1e6,
                                                                     med[k] / med["16k"]))
    print("GPU %s, power limit %s W, median SM clock %s MHz" % (res["gpu"], res["power_limit_w"], res["median_sm_clock_mhz"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
