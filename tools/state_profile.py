#!/usr/bin/env python
"""Cost of environment state records (ge_snapshot / ge_restore / ge_clone) next to what they save: a 4096-env stay(1000).

  python tools/state_profile.py [--envs 4096] [--reps 50] [--scenes A,B]

Per scene: envs reset by the scene's rule, settled with stay(1000) (timed: the settle a snapshot lets a grasp-labelling run skip), then
snapshot, restore and clone timed with CUDA events over `reps` back-to-back calls after a warm-up.  restore and clone include their one
host synchronisation (the record check).  Bytes moved: snapshot reads the rows and writes R per env (2 R); restore reads the headers and
then the records and writes the rows (about 2 R); clone is a snapshot into the engine's scratch plus a restore from it (4 R).  GB/s is
over the H100 SXM's 3.35 TB/s HBM3; the card's name and power limit are printed with the numbers.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"(nvidia-smi unavailable: {e})"


def timed(fn, reps):
    import torch

    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3  # seconds per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--scenes", default="A,B")
    args = ap.parse_args()
    import numpy as np
    import torch

    from mujoco_rl_ur5_b200.batched_env import scene_a_reset_qpos, scene_b_reset_qpos
    from mujoco_rl_ur5_b200.engine import BatchedEngine
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    if not torch.cuda.is_available():
        raise SystemExit("state_profile needs a CUDA device")
    print(f"card: {card()}")
    print(f"{'scene':5} {'call':9} {'envs':>5} {'R':>5} {'MB moved':>9} {'time':>11} {'GB/s':>7} {'of 3.35 TB/s':>12}")
    n = args.envs
    for scene in args.scenes.split(","):
        arrays, _ = load_scene(scene)
        rule = scene_b_reset_qpos if scene == "B" else scene_a_reset_qpos
        eng = BatchedEngine(load_scene_blob(scene), n, 0)
        eng.set_state(np.stack([rule(arrays, 20000 + i) for i in range(n)]))
        a, b = torch.cuda.Event(True), torch.cuda.Event(True)
        eng.stay(1000)
        a.record()
        eng.run()
        b.record()
        torch.cuda.synchronize()
        t_stay = a.elapsed_time(b) * 1e-3
        R = eng.state_bytes
        s = eng.snapshot()
        src = torch.arange(n - 1, -1, -1, dtype=torch.int32, device=eng.device)
        rows = {"snapshot": (lambda: eng.snapshot(), 2), "restore": (lambda: eng.restore(s), 2), "clone": (lambda: eng.clone(src), 4)}
        for name, (fn, k) in rows.items():
            t = timed(fn, args.reps)
            moved = k * n * R
            print(f"{scene:5} {name:9} {n:5d} {R:5d} {moved / 1e6:9.2f} {t * 1e6:8.1f} us {moved / t / 1e9:7.0f} {moved / t / 3.35e12:11.1%}")
        print(f"{scene:5} {'stay 1000':9} {n:5d} {'':5} {'':9} {t_stay * 1e3:8.1f} ms   ({n * 500 / t_stay / 1e6:.2f} M sub-steps/s)")
        eng.close()


if __name__ == "__main__":
    main()
