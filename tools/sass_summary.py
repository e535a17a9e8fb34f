#!/usr/bin/env python
"""Per-kernel SASS evidence for profiles/: resource usage, opcode histogram, and the instructions that prove which
hardware path a kernel uses (HGMMA = wgmma, UBLKCP = TMA bulk copies, SYNCS = mbarriers,
IMMA / HMMA = mma.sync).  Runs cuobjdump on the built library (no GPU needed).

usage: tools/sass_summary.py <tag>          -> profiles/<tag>_sass_<kernel>.txt
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lyra_b200", "liblyra_b200.so")

# mangled-name patterns (DecoderKernelC<true> feeds DecoderKernelDW in the tensor mode, DecoderKernelC<false> DecoderKernelD in the
# exact mode)
KERNELS = {
    "EncoderKernelA": r"EncoderKernelAE",
    "EncoderKernelB": r"EncoderKernelBE",
    "DecoderKernelC_tensor": r"DecoderKernelCILb1E",
    "DecoderKernelC_exact": r"DecoderKernelCILb0E",
    "DecoderKernelD_exact": r"DecoderKernelDE",
    "DecoderKernelDW": r"DecoderKernelDWE",
    "RvqEncodeKernel": r"RvqEncodeKernelE",
    "RvqDecodeKernel": r"RvqDecodeKernelE",
    "LogMelKernel": r"LogMelKernelE",
    "NoiseEstimatorKernel": r"NoiseEstimatorKernelE",
    "ComfortNoiseKernel": r"ComfortNoiseKernelE",
    "PlcMixKernel": r"PlcMixKernelE",
    "PlcPlanKernel": r"PlcPlanKernelE",
    "ResampleKernel": r"ResampleKernelE",
}
PROOF = ("HGMMA", "WARPGROUP", "UBLKCP", "UTMALDG", "SYNCS", "IMMA", "HMMA", "BAR", "DFMA", "CALL")
FULL_LISTING = ("DecoderKernelDW",)      # small enough to commit whole (instruction text only)


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "rX"
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            usage[cur] = line.strip()
            cur = None
    chunks = re.split(r"\n\s*Function : ", sass)
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    for name, pat in KERNELS.items():
        body = next((c for c in chunks[1:] if re.match(r"\S*" + pat, c)), None)
        if body is None:
            print("missing", name)
            continue
        mangled = body.split("\n", 1)[0].strip()
        insts = []
        for line in body.splitlines():
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if m:
                insts.append((m.group(1), m.group(2).strip()))
        hist = collections.Counter()
        for _, text in insts:
            t = text.split()
            op = t[1] if t[0].startswith("@") and len(t) > 1 else t[0]
            hist[op.split(".")[0]] += 1
        out = [f"# {name}: {mangled}", f"# library: lyra_b200/liblyra_b200.so (nvcc -gencode arch=compute_90a,code=sm_90a), cuobjdump -sass",
               f"# resources: {usage.get(mangled, '?')}", f"# instructions: {len(insts)}", "", "## opcode histogram"]
        for op, n in hist.most_common():
            out.append(f"{n:8d}  {op}")
        out += ["", "## evidence instructions (count, first occurrences)"]
        for p in PROOF:
            hits = [(a, t) for a, t in insts if re.search(r"(^|\s)" + p + r"(\.|\s|$)", t)]
            if not hits:
                continue
            out.append(f"{p}: {len(hits)}")
            for a, t in hits[:6]:
                out.append(f"    /*{a}*/  {t}")
        if name in FULL_LISTING:
            out += ["", "## full listing (instruction text)"]
            out += [f"/*{a}*/  {t}" for a, t in insts]
        path = os.path.join(ROOT, "profiles", f"{tag}_sass_{name}.txt")
        with open(path, "w") as f:
            f.write("\n".join(out) + "\n")
        print(path, len(insts), {p: hist[p] for p in ("HGMMA", "UBLKCP", "IMMA", "HMMA", "FFMA") if hist[p]})


if __name__ == "__main__":
    main()
