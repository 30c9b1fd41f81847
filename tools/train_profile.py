#!/usr/bin/env python
"""Where a batched step of the online trainer (mujoco_rl_ur5_b200.batched_train) spends its time: scene A, one GPU, CUDA events around
  env.step | acting (keyed transform + Q-net forward + arg-max + gq_sample_actions) | replay push | one learner update (batch 12)
per batched step, and gq_sample_actions against BatchedGreedyAgent.random_table_actions (the torch-op rejection loop with a host
synchronisation per round) on the same observations, the two alternated in one process.  Prints the card name and power limit.
usage: python tools/train_profile.py [--envs 4096] [--steps 3] [--updates 8] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    import torch

    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--updates", type=int, default=8, help="learner updates timed per batched step")
    ap.add_argument("--reps", type=int, default=20, help="sampler comparison repetitions")
    a = ap.parse_args()
    import torch

    from mujoco_rl_ur5_b200.batched_agent import BatchedGreedyAgent
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    tr = BatchedTrainer(a.envs, "A", 0, seed=0, updates_per_step=a.updates)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows = []
    try:
        tr.env.reset()
        for s in range(a.steps + 1):  # the first step is warm-up
            e = {}

            def mark(name):
                e[name] = ev()
                e[name].record()

            rec = tr.step(mark)  # the trainer's own step, CUDA events between its phases
            torch.cuda.synchronize()
            if s == 0:
                continue
            r = {"act_ms": e["start"].elapsed_time(e["act"]), "env_step_ms": e["act"].elapsed_time(e["env_step"]),
                 "push_ms": e["env_step"].elapsed_time(e["push"]), "update_ms": e["push"].elapsed_time(e["learn"]) / rec["updates"],
                 "n_random": rec["n_random"]}
            rows.append(r)
            print(json.dumps({"step": s, **{k: round(v, 3) if isinstance(v, float) else v for k, v in r.items()}}), flush=True)
        med = {k: float(np.median([r[k] for r in rows])) for k in ("act_ms", "env_step_ms", "push_ms", "update_ms")}
        full = med["act_ms"] + med["env_step_ms"] + med["push_ms"] + a.envs * med["update_ms"]
        print(json.dumps({"median": {k: round(v, 3) for k, v in med.items()}, "envs": a.envs,
                          "step_ms_at_one_update_per_transition": round(full, 1),
                          "learner_share_at_one_update_per_transition": round(a.envs * med["update_ms"] / full, 4)}), flush=True)

        # sampler: both at eps = 1 (every env random), on the current observations, alternated
        agent = BatchedGreedyAgent(tr.env, tr.learner.model_state_dict(), seed=0)
        obs = tr.env.current_observation
        idx = torch.zeros(a.envs, dtype=torch.int32, device=tr.dev)
        eps = torch.ones(a.envs, dtype=torch.float64)
        fw = tr.learner.fw
        kernel = lambda: fw.sample_actions(obs["depth"], idx, eps, tr.genv, 0, tr.seed, tr.camera, tr.z_min, 6, tr.max_draws)
        torch_loop = lambda: agent.random_table_actions(obs)
        kernel(); torch_loop(); torch.cuda.synchronize()
        t_k, t_t = [], []
        for _ in range(a.reps):
            for fn, out in ((kernel, t_k), (torch_loop, t_t)):
                e0, e1 = ev(), ev()
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                out.append(e0.elapsed_time(e1))
        mk, mt = float(np.median(t_k)), float(np.median(t_t))
        print(json.dumps({"sampler": {"gq_sample_actions_ms": round(mk, 4), "random_table_actions_ms": round(mt, 3), "speedup": round(mt / mk, 1),
                                      "envs": a.envs, "reps": a.reps}}), flush=True)
    finally:
        tr.close()
    print(f"card: {name}, power limit {power}", flush=True)


if __name__ == "__main__":
    main()
