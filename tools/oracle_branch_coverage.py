#!/usr/bin/env python
"""Branch coverage of the fp64 oracle's solver and narrow phase over the states of fixture files (CPU only).

The CUDA stages mirror oracle/grasp_oracle.c branch for branch, so an oracle branch that no fixture state takes is a device branch that
no parity test compares.  This builds the oracle with `gcc --coverage` in a temporary directory (the repository is not written), loads
that build through GRASP_ORACLE_SO, runs one forward() on every stored state and prints, for impedance, make_constraint, solve_newton,
every col_* function, support and mpr_penetration, the branches taken out of those compiled, and the source lines that hold an untaken
branch or never ran.

States: every array `qpos*` of a fixture .npz (its last axis is nq: 50 = scene A, 288 = scene B), with the `qvel*` array of the same
suffix when it has the matching shape, else zero velocity.  --attempts N also replays N grasp attempts spread over the records of a
scene-A fixture that has a .json next to it with `records` (coords and action per attempt, as success_64.json), from its states
`qpos0` / `qvel0`.

  python tools/oracle_branch_coverage.py tests/golden/limits_contacts.npz
  python tools/oracle_branch_coverage.py tests/golden/scene_a_edges.npz tests/golden/success_64.npz --attempts 11
"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ("impedance", "make_constraint", "solve_newton", "support", "mpr_penetration")
CFLAGS = ["-O0", "--coverage", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-D_GNU_SOURCE"]


def _wanted(name):
    return name in FUNCS or name.startswith("col_")


def _states(path, nq_scene):
    d = np.load(path)
    for k in sorted(d.files):
        if not k.startswith("qpos"):
            continue
        q = np.asarray(d[k], np.float64)
        scene = nq_scene.get(q.shape[-1])
        if scene is None:
            continue
        q = q.reshape(-1, q.shape[-1])
        kv = "qvel" + k[4:]
        v = np.asarray(d[kv], np.float64).reshape(len(q), -1) if kv in d.files and d[kv].size % len(q) == 0 else None
        yield scene, q, v


def _drive(paths, attempts):
    """runs in a child process: the coverage build must be the one oracle_py loads"""
    sys.path.insert(0, ROOT)
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob
    from oracle.oracle_py import OracleEnv

    blobs = {s: load_scene_blob(s) for s in "AB"}
    nq_scene = {int(np.asarray(load_scene(s)[0]["nq"]).ravel()[0]): s for s in "AB"}
    nfwd = nstep = 0
    for path in paths:
        for scene, qs, vs in _states(path, nq_scene):
            o = OracleEnv(blobs[scene])
            for i, q in enumerate(qs):
                o.reset(q, None if vs is None or vs.shape[1] != o.nv else vs[i])
                o.forward()
                nfwd += 1
            o.close()
        js = os.path.splitext(path)[0] + ".json"
        if attempts and os.path.exists(js):
            recs = json.load(open(js)).get("records", [])
            d = np.load(path)
            if not recs or "qpos0" not in d.files or d["qpos0"].shape[-1] not in nq_scene or nq_scene[d["qpos0"].shape[-1]] != "A" \
                    or not all(k in recs[0] for k in ("coords", "action")):
                continue
            o = OracleEnv(blobs["A"])
            for i in np.unique(np.linspace(0, len(recs) - 1, attempts).astype(int)):
                r = recs[i]
                o.reset(d["qpos0"][i], d["qvel0"][i] if "qvel0" in d.files else None)
                s0 = o.substeps
                o.move_and_grasp(r["coords"], int(r["action"][1]), 0.91)
                nstep += o.substeps - s0
            o.close()
    print("%d forward() calls, %d sub-steps of grasp attempts" % (nfwd, nstep))


def _report(gcov_json, source):
    lines = open(source).read().split("\n")
    rows = []
    for f in gcov_json["files"]:
        if not f["file"].endswith("grasp_oracle.c"):
            continue
        funcs = [fn for fn in f["functions"] if _wanted(fn["name"])]
        by_line = {ln["line_number"]: ln for ln in f["lines"]}
        for fn in sorted(funcs, key=lambda fn: fn["start_line"]):
            total = taken = 0
            missed = []
            for no in range(fn["start_line"], fn["end_line"] + 1):
                ln = by_line.get(no)
                if ln is None:
                    continue
                br = ln.get("branches", [])
                total += len(br)
                taken += sum(1 for b in br if b["count"] > 0)
                if ln["count"] == 0 or any(b["count"] == 0 for b in br):
                    missed.append((no, ln["count"], sum(1 for b in br if b["count"] > 0), len(br)))
            rows.append((fn["name"], fn["start_line"], taken, total, fn["execution_count"], missed))
    print("%-22s %6s %14s %12s" % ("function", "line", "branches taken", "calls"))
    for name, start, taken, total, calls, _ in rows:
        print("%-22s %6d %7d / %-5d %12d" % (name, start, taken, total, calls))
    print("\nlines with an untaken branch, or never run (times run, branches taken / compiled):")
    for name, _, _, _, _, missed in rows:
        for no, count, taken, total in missed:
            print("  %-20s %5d %9d %3d / %-3d %s" % (name, no, count, taken, total, lines[no - 1].strip()[:100]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("fixtures", nargs="+", help=".npz files under tests/golden/")
    ap.add_argument("--attempts", type=int, default=0, help="grasp attempts to replay from fixtures with a records .json")
    ap.add_argument("--drive", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    paths = [os.path.abspath(p) for p in a.fixtures]
    if a.drive:
        _drive(paths, a.attempts)
        return
    src = os.path.join(ROOT, "oracle", "grasp_oracle.c")
    with tempfile.TemporaryDirectory(prefix="oracle_cov_") as tmp:
        for f in ("grasp_oracle.c", "orc_math.h"):
            with open(os.path.join(ROOT, "oracle", f)) as fi, open(os.path.join(tmp, f), "w") as fo:
                fo.write(fi.read())
        so = os.path.join(tmp, "liboracle_cov.so")
        subprocess.check_call(["gcc"] + CFLAGS + ["-o", so, "grasp_oracle.c", "-lm"], cwd=tmp)
        env = dict(os.environ, GRASP_ORACLE_SO=so)
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--drive", "--attempts", str(a.attempts)] + paths, env=env)
        gcda = [f for f in os.listdir(tmp) if f.endswith(".gcda")]
        subprocess.check_call(["gcov", "--json-format", "--branch-probabilities", "--branch-counts", gcda[0]], cwd=tmp,
                              stdout=subprocess.DEVNULL)
        out = [f for f in os.listdir(tmp) if f.endswith(".gcov.json.gz")]
        with gzip.open(os.path.join(tmp, out[0])) as fi:
            _report(json.load(fi), src)


if __name__ == "__main__":
    main()
