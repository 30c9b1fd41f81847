#!/usr/bin/env python
"""Where a batched step of the online trainer (mujoco_rl_ur5_b200.batched_train) spends its time: scene A, one GPU, CUDA events around
  env.step | acting (keyed transform + Q-net forward + arg-max + gq_sample_actions) | replay push | one learner update (batch 12)
per batched step, and gq_sample_actions against BatchedGreedyAgent.random_table_actions (the torch-op rejection loop with a host
synchronisation per round) on the same observations, the two alternated in one process.  Prints the card name and power limit.
With --gamma G > 0 it instead alternates a gamma = 0 trainer and a gamma = G trainer on the same replay contents and times, per
repetition: one learner update of each (the gamma = G one including its target forward), a target-network sync, the target forward
alone (QNetForward.max_target on the batch's next states) and gq_head_max_target against gq_head_up2 + gq_argmax on the same head input.
usage: python tools/train_profile.py [--envs 4096] [--steps 3] [--updates 8] [--reps 20] [--gamma G --target-update K]
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
    ap.add_argument("--gamma", type=float, default=0.0, help="> 0: compare the bootstrapped update with the gamma = 0 one instead")
    ap.add_argument("--target-update", type=int, default=100, help="target sync period of the gamma > 0 trainer")
    a = ap.parse_args()
    import torch

    from mujoco_rl_ur5_b200.batched_agent import BatchedGreedyAgent
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    if a.gamma > 0:
        gamma_profile(a)
        print(f"card: {name}, power limit {power}", flush=True)
        return
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


def timed(fn):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def gamma_profile(a):
    import torch

    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    trs = {"gamma0": BatchedTrainer(a.envs, "A", 0, seed=0, updates_per_step=0),
           "gamma": BatchedTrainer(a.envs, "A", 0, seed=0, updates_per_step=0, gamma=a.gamma, target_update=a.target_update)}
    try:
        for tr in trs.values():  # fill the replays (no updates), then one untimed update of each: warm-up
            tr.env.reset()
            for _ in range(a.steps):
                tr.step()
            tr.update()
        tg = trs["gamma"]
        L = tg.learner
        B = tg.batch_size
        _, _, r, s2 = tg.replay.sample(B, L.fw, tg.seed, tg.depth_threshold, tg.noise_std)
        tgt = L.target
        x, h, w = tgt._trunk(s2)
        r = r.reshape(B).contiguous()
        qmax, y = torch.empty(B, device=tg.dev), torch.empty(B, device=tg.dev)
        idx = torch.empty(B, dtype=torch.int32, device=tg.dev)

        def head_max():
            tgt._ck(tgt.L.gq_head_max_target(tgt._p(x), tgt._p(tgt.w_head), tgt._p(tgt.b_head), tgt._p(r), float(a.gamma), tgt._p(qmax), tgt._p(y), B, h, w,
                                             tgt.A, tgt._stream()), "gq_head_max_target")

        def head_up2_argmax():
            q = tgt._head(x, h, w)
            tgt._ck(tgt.L.gq_argmax(tgt._p(q), B, q[0].numel(), tgt._p(idx), tgt._p(qmax), tgt._stream()), "gq_argmax")

        fns = {"update_gamma0_ms": trs["gamma0"].update, "update_gamma_ms": tg.update, "sync_target_ms": L.sync_target,
               "target_forward_ms": lambda: L.target.max_target(s2, r, a.gamma), "gq_head_max_target_ms": head_max,
               "gq_head_up2_plus_argmax_ms": head_up2_argmax}
        for fn in fns.values():
            fn()
        times = {k: [] for k in fns}
        for _ in range(a.reps):
            for k, fn in fns.items():
                times[k].append(timed(fn))
        med = {k: round(float(np.median(v)), 4) for k, v in times.items()}
        spread = {k: [round(float(np.percentile(v, 10)), 4), round(float(np.percentile(v, 90)), 4)] for k, v in times.items()}
        print(json.dumps({"gamma_profile": {"median": med, "p10_p90": spread, "envs": a.envs, "batch": B, "gamma": a.gamma, "reps": a.reps,
                                            "update_overhead": round(med["update_gamma_ms"] / med["update_gamma0_ms"] - 1, 4)}}), flush=True)
    finally:
        for tr in trs.values():
            tr.close()


if __name__ == "__main__":
    main()
