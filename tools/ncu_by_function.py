#!/usr/bin/env python
"""Aggregate an ncu source-page (SASS) capture of k_run by __noinline__ device function.

usage: tools/ncu_by_function.py <report.ncu-rep> <libgrasp_engine.so> [kernel-substring]
Needs ncu, cuobjdump and nvdisasm on PATH (no GPU).  Prints executed warp instructions, stall samples and the top stall
reason per function, i.e. where the sub-step's time goes.
"""
import collections
import csv
import io
import os
import re
import subprocess
import sys
import tempfile


def function_ranges(so, kernel):
    d = tempfile.mkdtemp()
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=d, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    txt = ""
    for cubin in sorted(f for f in os.listdir(d) if f.endswith(".cubin")):  # one cubin per translation unit (engine variants)
        t = subprocess.run(["nvdisasm", os.path.join(d, cubin)], capture_output=True, text=True).stdout
        if any(l.startswith(".text.") and kernel in l for l in t.splitlines()):
            txt = t
            break
    ranges, on, name = [], False, "(kernel body)"
    for line in txt.splitlines():
        if line.startswith(".text."):
            on = kernel in line
            name = "(kernel body)"
            continue
        if not on:
            continue
        if line.startswith("$"):
            name = line.strip().rstrip(":").split("$")[-1]
            m = re.search(r"_ZN\d+ge(?:_warp|_cta)?\d+([A-Za-z_0-9]+?)E", name)
            name = m.group(1) if m else name
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/", line)
        if m:
            addr = int(m.group(1), 16)
            if not ranges or ranges[-1][1] != name:
                ranges.append((addr, name))
    return ranges


def main():
    rep, so = sys.argv[1], sys.argv[2]
    kernel = sys.argv[3] if len(sys.argv) > 3 else "k_run"
    ranges = function_ranges(so, kernel)
    starts = [r[0] for r in ranges]
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hi = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
    H = rows[hi]
    ci = {n: H.index(n) for n in ("Address", "Warp Stall Sampling (All Samples)", "Instructions Executed", "Thread Instructions Executed")}
    stall_cols = [(i, h) for i, h in enumerate(H) if h.startswith("stall_") and "Not Issued" not in h]
    base = None
    agg = collections.defaultdict(lambda: [0, 0, 0, collections.Counter()])
    import bisect

    for r in rows[hi + 1:]:
        if len(r) < len(H):
            continue
        try:
            a = int(r[ci["Address"]], 16)
        except ValueError:
            continue
        if base is None:
            base = a
        k = bisect.bisect_right(starts, a - base) - 1
        name = ranges[max(k, 0)][1]
        e = agg[name]
        e[0] += int(float(r[ci["Instructions Executed"]] or 0))
        e[1] += int(float(r[ci["Thread Instructions Executed"]] or 0))
        e[2] += int(float(r[ci["Warp Stall Sampling (All Samples)"]] or 0))
        for i, h in stall_cols:
            v = r[i]
            if v and v != "0":
                try:
                    e[3][h] += int(float(v))
                except ValueError:
                    pass
    ti = sum(e[0] for e in agg.values()) or 1
    ts = sum(e[2] for e in agg.values()) or 1
    print(f"{'function':22s} {'warp-inst':>12s} {'%inst':>6s} {'thr/inst':>8s} {'samples':>9s} {'%time':>6s}  top stalls")
    for name, e in sorted(agg.items(), key=lambda x: -x[1][2]):
        top = ", ".join(f"{k.replace('stall_', '')}:{v * 100 // max(e[2], 1)}%" for k, v in e[3].most_common(3))
        print(f"{name:22s} {e[0]:12d} {100 * e[0] / ti:6.1f} {e[1] / max(e[0], 1):8.1f} {e[2]:9d} {100 * e[2] / ts:6.1f}  {top}")
    print(f"total warp instructions {ti}, samples {ts}")


if __name__ == "__main__":
    main()
