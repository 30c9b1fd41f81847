"""SASS footprint of the engine kernels (CPU only: nvcc / cuobjdump / nvdisasm, no GPU).

    python tools/sass_footprint.py                   # compile both engine variants of this tree for sm_90a and report
    python tools/sass_footprint.py --src DIR         # ... of another checkout (DIR holds mujoco_rl_ur5_b200/csrc)
    python tools/sass_footprint.py --obj a.o [b.o]   # report already compiled objects (registers / stack from the cubin)

Per kernel: SASS bytes and instructions, registers, stack frame, spill stores / loads (only for objects compiled here: ptxas -v),
LDL / STL and CALL instructions.  For k_run also the bytes of every device function it calls: without -rdc each non-inlined callee
is a labelled subroutine inside the kernel's own text section, so its bytes are the distance to the next label.  HOT is the list of
functions that run on every scene-A sub-step; their sum is the code a warp walks per sub-step.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-diag-suppress", "550"]
HOT = ["build_hessian", "solve_newton", "nt_update", "group_chol_solve", "stage_collision", "stage_constraints", "mpr_w", "stage_fk",
       "cholesky_solve", "stage_rne", "support_w", "sim_step", "forward", "mass_block_solve", "rows_cost", "stage_crb", "mul_M"]


def compile_variant(src, variant, out):
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + FLAGS + ["-Xptxas", "-v", "-DGE_VARIANT=%d" % variant, "-c", "-o", out,
                                                        os.path.join(src, "mujoco_rl_ur5_b200", "csrc", "grasp_engine.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.exit(r.stderr)
    return r.stderr


def ptxas_spills(log):
    """{mangled kernel: (spill store bytes, spill load bytes)} from ptxas -v"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def demangled_tail(name):
    """_ZN7ge_warp5k_runE9EnvArrays... -> k_run;  __internal_accurate_pow -> itself"""
    m = re.match(r"_ZN\d+\w+?(\d+)(\w+)", name)
    if not m or not name.startswith("_ZN"):
        return name
    parts, s = [], name[3:]
    while s and s[0].isdigit():
        n = re.match(r"\d+", s).group(0)
        parts.append(s[len(n):len(n) + int(n)])
        s = s[len(n) + int(n):]
    return parts[-1] if parts else name


def analyse(obj, spills):
    with tempfile.TemporaryDirectory() as td:
        subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(obj)], cwd=td, check=True,
                       capture_output=True)
        cubin = [f for f in os.listdir(td) if f.endswith(".cubin")][0]
        res = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", os.path.join(td, cubin)], capture_output=True,
                             text=True, check=True).stdout
        dis = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), os.path.join(td, cubin)], capture_output=True, text=True,
                             check=True).stdout
    usage, fn = {}, None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            usage[fn] = (int(m.group(1)), int(m.group(2)))
    kernels = {}  # kernel -> {"n": instructions, "ldl", "stl", "call", "sub": {callee: instructions}}
    k = sub = None
    for line in dis.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            k, sub = m.group(1), None
            kernels[k] = {"n": 0, "ldl": 0, "stl": 0, "call": 0, "sub": {}}
            continue
        if k is None:
            continue
        m = re.match(r"^\$" + re.escape(k) + r"\$(\S+):", line)
        if m:
            sub = demangled_tail(m.group(1))
            kernels[k]["sub"].setdefault(sub, 0)
            continue
        if re.match(r"\s*\.section\s", line):
            k = None
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*)", line)
        if not m:
            continue
        ins = m.group(1)
        d = kernels[k]
        d["n"] += 1
        if sub:
            d["sub"][sub] += 1
        op = re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0] if ins.split() else ""
        if op.startswith("LDL"):
            d["ldl"] += 1
        elif op.startswith("STL"):
            d["stl"] += 1
        elif op.startswith("CALL"):
            d["call"] += 1
    return kernels, usage, spills


def report(title, kernels, usage, spills):
    print("== %s" % title)
    print("%-16s %9s %7s %5s %6s %13s %6s %6s %5s" % ("kernel", "bytes", "instr", "regs", "stack", "spill st/ld", "LDL", "STL", "CALL"))
    for k, d in sorted(kernels.items(), key=lambda kv: -kv[1]["n"]):
        reg, stk = usage.get(k, ("?", "?"))
        sp = spills.get(k)
        print("%-16s %9d %7d %5s %6s %13s %6d %6d %5d" % (demangled_tail(k), 16 * d["n"], d["n"], reg, stk,
                                                          "%d/%d" % sp if sp else "n/a", d["ldl"], d["stl"], d["call"]))
    run = [k for k in kernels if demangled_tail(k) == "k_run"]
    if not run:
        return
    d = kernels[run[0]]
    own = d["n"] - sum(d["sub"].values())
    print("k_run by function (bytes):")
    rows = sorted(d["sub"].items(), key=lambda kv: -kv[1]) + [("(k_run body)", own)]
    for name, n in rows:
        print("  %-28s %8d%s" % (name, 16 * n, "  *" if name in HOT else ""))
    hot = sum(n for name, n in d["sub"].items() if name in HOT)
    print("hot path (* : functions run on every scene-A sub-step): %d bytes in %d functions" %
          (16 * hot, sum(1 for name in d["sub"] if name in HOT)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--src", default=ROOT, help="source tree to compile (default: this checkout)")
    ap.add_argument("--obj", nargs="*", help="report these objects instead of compiling")
    a = ap.parse_args()
    if a.obj:
        for o in a.obj:
            report(o, *analyse(o, {}))
        return
    with tempfile.TemporaryDirectory() as td:
        outs = [os.path.join(td, "v%d.o" % v) for v in (0, 1)]
        with ThreadPoolExecutor(2) as ex:
            logs = list(ex.map(lambda v: compile_variant(a.src, v, outs[v]), (0, 1)))
        for v in (0, 1):
            report("GE_VARIANT=%d (%s)" % (v, "warp per env" if v == 0 else "CTA per env"), *analyse(outs[v], ptxas_spills(logs[v])))


if __name__ == "__main__":
    main()
