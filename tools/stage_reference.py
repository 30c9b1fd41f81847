#!/usr/bin/env python
"""Stages the UNMODIFIED reference scripts the acceptance test runs (tests/test_reference_scripts_gpu.py) into baseline/_ref/.

/root/reference exists only in the development container; the GPU box gets a snapshot of /root/repo.  baseline/_ref/ is
git-ignored (never committed: the repository holds no reference source) but travels with the snapshot, which is what the bench
contract reserves it for.  Staged byte for byte: example_agent.py, Grasping_Agent_multidiscrete.py, Modules.py (the agent's
network + replay buffer) and the pickled `mean_and_std`.  The reference's gym_grasper package is NOT staged: the scripts import
`gym_grasper` / `gym` from mujoco_rl_ur5_b200/compat, i.e. they run against the H100 engine.

  python tools/stage_reference.py [/root/reference]
"""
import hashlib
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ["example_agent.py", "Grasping_Agent_multidiscrete.py", "Modules.py", "mean_and_std"]


def main():
    src = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    dst = os.path.join(ROOT, "baseline", "_ref")
    os.makedirs(dst, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(src, f), os.path.join(dst, f))
        print(f, hashlib.sha256(open(os.path.join(dst, f), "rb").read()).hexdigest()[:16])
    print("staged into", dst)


if __name__ == "__main__":
    main()
