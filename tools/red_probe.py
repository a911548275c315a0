#!/usr/bin/env python
"""Time the moment reductions of one backward render alone: tools/red_probe.cu, built here with nvcc for sm_90a and run on
GPU 0.  Prints the probe's RESULT lines, per row pattern the time of (a) ten scalar reductions minus the faster four-operation
split (d1 / d2), and the card's name, power limit and SM clock read while the probe runs.

    python tools/red_probe.py [--pairs 590000] [--rows 100000] [--launches 200]

--pairs: (record, sub-tile) pairs of the bench view's backward (tools/bwd_reduction_count.py prints it).
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))


def nvidia_smi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=590000)
    ap.add_argument("--rows", type=int, default=100000)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "red_probe")
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe, os.path.join(HERE, "red_probe.cu")],
                       check=True)
        print("gpu (name, power limit, max SM clock):", nvidia_smi("name,power.limit,clocks.max.sm"), flush=True)
        proc = subprocess.Popen([exe, str(a.pairs), str(a.rows), str(a.launches)], stdout=subprocess.PIPE, text=True)
        samples = []
        while proc.poll() is None:                     # SM clock sampled while the probe runs
            time.sleep(0.5)
            if proc.poll() is None:
                samples.append(nvidia_smi("clocks.sm,power.draw"))
        out = proc.stdout.read()
        print(out, end="")
        print("SM clock, power draw during the run:", "; ".join(samples[:12]) or "run too short to sample")
        if proc.returncode != 0:
            sys.exit(proc.returncode)
    res = {}
    for m in re.finditer(r"RESULT pattern=(\S+) pass=(\d) variant=(\S+) ops_per_pair=\d+ us=([\d.]+)", out):
        res.setdefault((m.group(1), m.group(3)), []).append(float(m.group(4)))
    for pat in ("contended", "random"):
        t = {v: min(us) for (p, v), us in res.items() if p == pat}
        if not t:
            continue
        best_d = min(("d1_v4v4f32f32", "d2_v4v2v2v2"), key=lambda v: t[v])
        print("%s: a %.2f us, c %.2f us, d1 %.2f us, d2 %.2f us; a - %s = %.2f us" % (
            pat, t["a_10xf32"], t["c_v4v4v2"], t["d1_v4v4f32f32"], t["d2_v4v2v2v2"], best_d, t["a_10xf32"] - t[best_d]))


if __name__ == "__main__":
    main()
