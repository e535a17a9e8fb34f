"""Throughput of bench.py's device-resident duplex schedule (tools/duplex_schedule.py) in named configurations, alternated run by
run in one process so that clock and thermal drift hit them alike:
  16k, 8k, 32k, 48k  every stream at that context rate (lyra_b200_set_sample_rate) in --groups context pairs; 16k is the
                     benchmark's workload;
  mixed              --groups pairs at row rate 48 kHz, the streams at 8 / 16 / 32 / 48 kHz interleaved
                     (lyra_b200_set_stream_sample_rates) so that every tile mixes the four rates;
  split              the same traffic split by rate: one context pair per rate with a quarter of the streams each (what a
                     server without per-stream rates runs);
  bits-184           every stream at 184 bits (9.2 kbps) in --groups pairs called at 184 bits;
  bits-mixed         --groups pairs called at 184 bits, the streams at 64 / 120 / 184 bits interleaved
                     (lyra_b200_set_stream_bits) so that every tile and every RVQ block mixes them;
  bits-split         the same traffic split by bit rate: one context pair per bit rate with a tile-aligned third of the streams
                     each (what a server without per-stream bit rates runs);
  mixed-counters     16k with the odd lanes of every context set back to their state at creation (copy_streams from -1) after
                     the warm-up, so odd and even lanes stay 10 hops apart and every tile takes the per-stream hop-counter path
                     of the depthwise convolutions instead of the shared-counter fast path;
  aligned-counters   mixed-counters followed by align_streams(odd lanes, like = the even lane before each) on both contexts
                     of every pair: the same streams in the same states, every tile back on one counter;
  dtx                speech input (tests/data/sample1_16kHz.wav tiled, stream i from offset (i * 7919) mod len), the encoders
                     running encode_dtx_device with DTX on for every stream and the decoders taking DTX hops as lost packets;
  dtx-mixed          dtx with DTX off for every other stream (lyra_b200_set_stream_dtx), so every tile mixes the two kinds;
  dtx-split          the same traffic split by kind: half the streams in encode_dtx_device pairs, half in encode_device pairs
                     (what a server without per-stream DTX runs);
  dtx-off            dtx with DTX off for every stream, to compare with 16k;
  mask-ones          16k with an all-ones active mask installed (lyra_b200_set_active_mask), to compare with 16k;
  mask-tiles         16k with the tiles alternating hop by hop: the even tiles run on even hops, the odd tiles on odd hops (a
                     server that ticks every 10 ms and staggers the 20 ms hop phase of its calls tile by tile);
  mask-lanes         16k with a rotating quarter of the lanes of every tile sitting out (lanes 2k, 2k + 1 on hops i = k mod 4),
                     every stream aligned with the first lane of its tile every 25 hops (lyra_b200_align_streams);
  stats              shorthand for the four configurations below, alternated like any others:
  stats-off-16k,     16k and 48k with the per-stream call statistics off (the default) and on (lyra_b200_set_stats: one
  stats-on-16k,      CallStatsKernel launch per sub-batch of every codec call), to compare pairwise.
  stats-off-48k,
  stats-on-48k
Frames/s counts every stream's hops, also those it sits out; the mask configurations also report the active fraction.
The dtx configurations also report the fraction of DTX hops over the timed runs.
Prints one line per run, then every configuration's median, spread and ratio to the first configuration, the card's name,
power limit and median SM clock over the timed runs, and a JSON line.  --profile-hops adds a torch.profiler pass per
configuration, separate from the timed runs: the mean device time per launch of ResampleKernel, RvqEncodeKernel,
RvqDecodeKernel and CallStatsKernel.

  python tools/schedule_bench.py [--configs 16k,48k,8k,mixed,split,bits-184,bits-mixed,bits-split,mixed-counters,aligned-counters,
                                            dtx,dtx-mixed,dtx-split,dtx-off,mask-ones,mask-tiles,mask-lanes,stats]
                                 [--streams 4096]
                                 [--hops 200] [--runs 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
import duplex_schedule as ds  # noqa: E402

RATES = (8000, 16000, 32000, 48000)
BIT_RATES = (64, 120, 184)
CONFIGS = ("16k", "8k", "32k", "48k", "mixed", "split", "bits-184", "bits-mixed", "bits-split", "mixed-counters", "aligned-counters",
           "dtx", "dtx-mixed", "dtx-split", "dtx-off", "mask-ones", "mask-tiles", "mask-lanes", "stats-off-16k", "stats-on-16k",
           "stats-off-48k", "stats-on-48k")
STATS = ("stats-off-16k", "stats-on-16k", "stats-off-48k", "stats-on-48k")
PROFILED = ("ResampleKernel", "RvqEncodeKernel", "RvqDecodeKernel", "CallStatsKernel")
# active-mask patterns of the mask-* configurations (rows of all groups, 8-stream tiles), applied hop by hop in turn
MASKS = {
    "mask-ones": lambda n: [np.ones(n, np.uint8)],
    "mask-tiles": lambda n: [((np.arange(n) // 8) % 2 == h).astype(np.uint8) for h in range(2)],
    "mask-lanes": lambda n: [((np.arange(n) % 8) // 2 != k).astype(np.uint8) for k in range(4)],
}


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def speech_slots(streams):
    """ds.NBUF hops of speech for the given stream indices: tests/data/sample1_16kHz.wav tiled, stream i from offset
    (i * 7919) mod len (SURVEY.md section 8d)"""
    import wave
    with wave.open(os.path.join(bench.ROOT, "tests", "data", "sample1_16kHz.wav")) as w:
        clip = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)
    start = (np.asarray(streams, np.int64) * 7919) % len(clip)
    return [clip[(start[:, None] + b * 320 + np.arange(320)[None, :]) % len(clip)] for b in range(ds.NBUF)]


def make(name, args):
    """The schedules of one configuration."""
    def sched(n, groups, rate=16000, stream_rates=None, bits=None, stream_bits=None, dtx=None, speech=None, mask=None, realign=0):
        if speech is None:
            rng = np.random.default_rng(1234)
            pcm = [rng.integers(-8192, 8192, size=(n, rate // 50), dtype=np.int16) for _ in range(ds.NBUF)]
        else:
            pcm = speech_slots(speech)
        return ds.Schedule(pcm, groups, args.split, args.decoder_mode, bits or args.bits, rate=rate, stream_rates=stream_rates,
                           stream_bits=stream_bits, dtx=dtx, mask=mask, realign=realign)

    n, g = args.streams, args.groups
    if name in STATS:
        s = sched(n, g, int(name[-3:-1]) * 1000)
        if name.startswith("stats-on"):
            for enc, dec, _, _ in s.groups:
                enc.set_stats(1)
                dec.set_stats(1)
        return [s]
    if name.startswith("mask-"):
        return [sched(n, g, mask=MASKS[name](n), realign=25 if name == "mask-lanes" else 0)]
    if name in ("dtx", "dtx-mixed", "dtx-off"):
        m = n // g
        dtx = {"dtx": np.ones(m, np.int32), "dtx-mixed": (np.arange(m) % 2 == 0).astype(np.int32), "dtx-off": np.zeros(m, np.int32)}[name]
        return [sched(n, g, dtx=dtx, speech=np.arange(n))]
    if name == "dtx-split":
        # the streams of dtx-mixed, each kind in context pairs of its own: DTX on (the even streams) and encode_device (the odd)
        return [sched(n // 2, g, dtx=np.ones(n // 2 // g, np.int32), speech=np.arange(0, n, 2)), sched(n // 2, g, speech=np.arange(1, n, 2))]
    if name == "bits-184":
        return [sched(n, g, bits=184)]
    if name == "bits-mixed":
        return [sched(n, g, bits=184, stream_bits=np.array([BIT_RATES[k % len(BIT_RATES)] for k in range(n // g)], dtype=np.int32))]
    if name == "bits-split":
        t = 8                                        # lyra_b200_tile_streams
        cut = [0, (n // 3) // t * t, (2 * n // 3) // t * t, n]
        return [sched(cut[i + 1] - cut[i], 1, bits=b) for i, b in enumerate(BIT_RATES)]
    if name == "mixed":
        return [sched(n, g, 48000, np.array([RATES[k % len(RATES)] for k in range(n // g)], dtype=np.int32))]
    if name == "split":
        return [sched(n // len(RATES), 1, r) for r in RATES]
    return [sched(n, g, 16000 if name.endswith("-counters") else int(name[:-1]) * 1000)]


def kernel_us(scheds, hops):
    """{kernel: (mean device time of one launch, launch count)} of the PROFILED kernels (torch.profiler, CUDA activity) over
    `hops` hops."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ds.run(scheds, hops)
        torch.cuda.synchronize()
    res = {}
    for k in PROFILED:
        times = [ev.time_range.elapsed_us() for ev in prof.events() if k in ev.name]
        res[k] = {"us_per_launch": sum(times) / len(times) if times else None, "launches": len(times)}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0], formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="16k,48k,8k,mixed,split,mixed-counters", help="comma-separated, from " + ",".join(CONFIGS))
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--hops", type=int, default=200, help="hops per timed run")
    ap.add_argument("--runs", type=int, default=5, help="runs per configuration, alternating the configurations")
    ap.add_argument("--groups", type=int, default=2)
    ap.add_argument("--split", type=int, default=2)
    ap.add_argument("--bits", type=int, default=64, help="64 bits per 20 ms hop = 3.2 kbps")
    ap.add_argument("--decoder-mode", default="tensor", choices=["exact", "tensor"])
    ap.add_argument("--profile-hops", type=int, default=0, help="hops of the per-kernel profiler pass (0: none)")
    args = ap.parse_args()
    names = [k for c in args.configs.split(",") for k in (STATS if c == "stats" else (c,))]
    bad = [k for k in names if k not in CONFIGS]
    if bad:
        ap.error("unknown configuration %s" % ", ".join(bad))
    if not torch.cuda.is_available():
        raise SystemExit("schedule_bench needs a CUDA device")
    configs = {k: make(k, args) for k in names}
    for scheds in configs.values():
        ds.run(scheds, ds.NBUF + 2)          # warm-up: first launches, stream maps; every stream at hop counter 10
    torch.cuda.synchronize()
    for k in ("mixed-counters", "aligned-counters"):
        if k not in configs:
            continue
        s = configs[k][0]
        odd = np.arange(1, s.m, 2, dtype=np.int32)
        for e_, d_, _, _ in s.groups:
            for c in (e_, d_):
                c.copy_streams(np.full(odd.size, -1, np.int32), odd)   # odd lanes back to hop counter 0
                if k == "aligned-counters":
                    c.align_streams(odd, odd - 1)                      # and onto their even neighbours' counters
        torch.cuda.synchronize()
    fps = {k: [] for k in names}
    sampler = bench.ClockSampler(0, "GPU-%s" % torch.cuda.get_device_properties(0).uuid)
    sampler.start()
    for run in range(args.runs):
        for k, scheds in configs.items():
            v = ds.timed(scheds, args.hops)
            fps[k].append(v)
            print("run %d  %-14s  %.3f M frames/s" % (run, k, v / 1e6), flush=True)
    clocks = sampler.stop()
    dtx_frac = {}
    for k, scheds in configs.items():      # each slot holds the flags of its latest hop: the last ds.NBUF hops of the timed runs
        if k.startswith("dtx"):
            torch.cuda.synchronize()
            dtx_frac[k] = sum(int(f.sum()) for s in scheds if s.dtx for f in s.dtx_flags) / (ds.NBUF * sum(s.n for s in scheds))
    kernel = {}
    if args.profile_hops:
        for k, scheds in configs.items():
            kernel[k] = kernel_us(scheds, args.profile_hops)
    for scheds in configs.values():
        for s in scheds:
            s.close()
    base = names[0]
    med = {k: float(np.median(v)) for k, v in fps.items()}
    res = {
        "gpu": torch.cuda.get_device_name(), "power_limit": power_limit(), "clocks": clocks, "streams": args.streams,
        "bits": args.bits, "decoder_mode": args.decoder_mode, "split": args.split, "groups": args.groups, "hops_per_run": args.hops,
        "frames_per_s": fps, "median_frames_per_s": med, "spread": {k: [min(v) / med[k], max(v) / med[k]] for k, v in fps.items()},
        "ratio_to_" + base: {k: v / med[base] for k, v in med.items()}, "kernels": kernel, "dtx_hop_fraction": dtx_frac,
        "active_fraction": {k: float(np.mean([p.mean() for p in MASKS[k](args.streams)])) for k in names if k in MASKS},
    }
    for k in names:
        print("%-14s: median %.3f M frames/s (runs %.3f-%.3f), %.3f x %s%s" % (
            k, med[k] / 1e6, min(fps[k]) / 1e6, max(fps[k]) / 1e6, med[k] / med[base], base,
            ", DTX hops %.3f" % dtx_frac[k] if k in dtx_frac else ""))
    for k, per in kernel.items():
        for name, v in per.items():
            if v["launches"]:
                print("%s in %s: %.1f us per launch (%d launches)" % (name, k, v["us_per_launch"], v["launches"]))
    print("GPU %s, power limit %s, median SM clock %s MHz" % (res["gpu"], res["power_limit"], clocks["sm_mhz"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
