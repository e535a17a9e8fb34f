#!/usr/bin/env python3
"""Dev tool (GPU): the device twins of the plugin-level calls against their host-buffer twins, at 1024 and 4096 streams, and the
chain extract -> quantize -> dequantize -> generate on device buffers against the same chain of host-buffer calls and against the
fused encode_device + decode_device.

Host-buffer calls: wall clock per call (each copies in, runs, copies out and synchronises).  Device twins and the fused pair:
CUDA events around a window of calls queued back to back on the installed stream, per call.  Every figure is the median of
`--rounds` rounds; the rounds alternate the contenders.  Prints one JSON line per (call, streams) and, first, the GPU's name and
power limit.  Usage: tools/plugin_device_bench.py [--streams 1024 4096] [--iters 50] [--warmup 5] [--rounds 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from lyra_b200 import _capi  # noqa: E402

BITS = 64


def gpu_info(torch):
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unknown"
    return info


def device_ms(torch, s, fn, iters, warmup):
    """ms per call of fn queued `iters` times on stream s, by CUDA events"""
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(iters):
            fn()
        b.record(s)
    b.synchronize()
    return a.elapsed_time(b) / iters


def host_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return 1e3 * (time.perf_counter() - t0) / iters


def run(torch, n, iters, warmup, rounds):
    s = torch.cuda.Stream()
    D, H, F = _capi.Context(n), _capi.Context(n), _capi.Context(n)     # device twins, host twins, fused pair
    for c in (D, F):
        c.set_stream(s.cuda_stream)
    rng = np.random.default_rng(n)
    h_pcm = rng.integers(-8192, 8192, size=(n, 320), dtype=np.int16)
    h_feat = H.extract_features(h_pcm)
    h_pk = H.quantize(h_feat, BITS)
    h_cn = rng.uniform(0.62, 1.3, size=(n, 160)).astype(np.float32)
    P = _capi.packet_bytes(BITS)
    with torch.cuda.stream(s):
        t = lambda a: torch.from_numpy(a).cuda()     # noqa: E731
        d_pcm, d_feat, d_pk, d_cnf = t(h_pcm), t(h_feat), t(h_pk), t(h_cn)
        d_out = torch.zeros((n, 320), dtype=torch.int16, device="cuda")
        d_feat2 = torch.zeros((n, 64), dtype=torch.float32, device="cuda")
        d_pk2 = torch.zeros((n, P), dtype=torch.uint8, device="cuda")
        d_mel = torch.zeros((n, 160), dtype=torch.float32, device="cuda")
        d_flags = torch.zeros((n,), dtype=torch.uint8, device="cuda")
        d_rs = torch.zeros((n, 961), dtype=torch.int16, device="cuda")
        d_cnt = torch.zeros((n,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    p = lambda x: x.data_ptr()                      # noqa: E731

    def dev_chain():
        D.extract_features_device(n, p(d_pcm), p(d_feat2))
        D.quantize_device(n, p(d_feat2), BITS, p(d_pk2))
        D.dequantize_device(n, p(d_pk2), BITS, p(d_feat2))
        D.generate_device(n, p(d_feat2), p(d_out))

    def host_chain():
        f = H.extract_features(h_pcm)
        H.generate(H.dequantize(H.quantize(f, BITS), BITS))

    def fused():
        F.encode_device(n, p(d_pcm), BITS, p(d_pk2))
        F.decode_device(n, p(d_pk2), 0, BITS, p(d_out))

    cases = [
        ("extract_features", lambda: D.extract_features_device(n, p(d_pcm), p(d_feat2)), lambda: H.extract_features(h_pcm)),
        ("quantize", lambda: D.quantize_device(n, p(d_feat), BITS, p(d_pk2)), lambda: H.quantize(h_feat, BITS)),
        ("dequantize", lambda: D.dequantize_device(n, p(d_pk), BITS, p(d_feat2)), lambda: H.dequantize(h_pk, BITS)),
        ("generate", lambda: D.generate_device(n, p(d_feat), p(d_out)), lambda: H.generate(h_feat)),
        ("logmel", lambda: D.logmel_device(n, p(d_pcm), p(d_mel), 160, 0), lambda: H.logmel(h_pcm, 160, 0)),
        ("noise_estimate", lambda: D.noise_estimate_device(n, p(d_mel), p(d_flags)), lambda: H.noise_estimate(n=n)),
        ("cng_generate", lambda: D.cng_generate_device(n, p(d_cnf), p(d_out)), lambda: H.cng_generate(h_cn)),
        ("resample_16k_to_48k", lambda: D.resample_device(n, 48000, 0, p(d_pcm), 320, p(d_rs), 961, p(d_cnt)),
         lambda: H.resample(h_pcm, 48000, False)),
        ("chain_extract_quantize_dequantize_generate", dev_chain, host_chain),
    ]
    out = []
    for name, dev, host in cases:
        dv, hv, fv = [], [], []
        for _ in range(rounds):
            dv.append(device_ms(torch, s, dev, iters, warmup))
            hv.append(host_ms(host, max(3, iters // 5), 1))
            if name.startswith("chain"):
                fv.append(device_ms(torch, s, fused, iters, warmup))
        r = {"call": name, "streams": n, "device_ms": round(float(np.median(dv)), 4), "host_ms": round(float(np.median(hv)), 4),
             "device_ms_spread": [round(min(dv), 4), round(max(dv), 4)]}
        if fv:
            r["fused_encode_decode_device_ms"] = round(float(np.median(fv)), 4)
            r["fused_spread"] = [round(min(fv), 4), round(max(fv), 4)]
        out.append(r)
        print(json.dumps(r), flush=True)
    for c in (D, H, F):
        c.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("plugin_device_bench needs a CUDA device")
    info = gpu_info(torch)
    print(json.dumps(info), flush=True)
    res = [r for n in a.streams for r in run(torch, n, a.iters, a.warmup, a.rounds)]
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"info": info, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
