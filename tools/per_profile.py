#!/usr/bin/env python
"""What prioritized replay costs the online trainer: CUDA-event times of the three sum-tree kernels (gq_per_push of 4096 slots,
gq_per_sample and gq_per_update at B = 12) at replay sizes 2000, 16 384 and 1 048 576; the uniform path's per-update draw
(ObservationReplay.sample_indices, Python's random.sample) plus its host-to-device index copy; and one batched trainer step with and
without prioritized replay (--updates learner updates each), the two trainers alternated in one process.  Prints the card name and
power limit.
usage: python tools/per_profile.py [--envs 4096] [--steps 3] [--updates 8] [--reps 200]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from train_profile import card  # noqa: E402


def fill(rp, n, chunk=1 << 16):
    import torch

    for k in range(0, n, chunk):
        m = min(chunk, n - k)
        rp.push_batch(torch.zeros((m, 2, 2, 3), dtype=torch.uint8, device="cuda"), torch.zeros((m, 2, 2), device="cuda"), torch.zeros(m, dtype=torch.int64),
                      torch.zeros(m), torch.arange(k, k + m), torch.zeros(m, dtype=torch.int64))


def event_ms(fn, reps):
    """mean device time of fn() over `reps` back-to-back calls between two CUDA events (after one warm-up call)"""
    import torch

    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(reps):
    import torch

    from mujoco_rl_ur5_b200.replay_buffer import ObservationReplay, PrioritizedObservationReplay

    out = []
    for size in (2000, 16384, 1048576):
        rp = PrioritizedObservationReplay(size, (2, 2), device="cuda")
        fill(rp, size)
        L, st = rp.L, torch.cuda.current_stream().cuda_stream
        slots = (size // 3 + torch.arange(min(4096, size), device="cuda")) % size  # a push's run of ring slots (the whole ring at 2000)
        idx = torch.empty(12, dtype=torch.int64, device="cuda")
        w = torch.empty(12, dtype=torch.float32, device="cuda")
        q, r = torch.rand(12, device="cuda"), (torch.rand(12, device="cuda") < 0.2).float()
        ptr = lambda x: x.data_ptr()
        push = lambda: L.gq_per_push(ptr(rp.tree), ptr(rp.pmax), ptr(slots), int(slots.numel()), rp.cap, st)
        upd = [0]

        def sample():
            upd[0] += 1
            return L.gq_per_sample(ptr(rp.tree), rp.cap, len(rp), 12, 0.4, 0, upd[0], 0, ptr(idx), ptr(w), st)

        update = lambda: L.gq_per_update(ptr(rp.tree), ptr(rp.pmax), ptr(idx), ptr(q), ptr(r), 12, 0.6, 1e-6, rp.cap, st)
        row = {"size": size, "push_slots": int(slots.numel()), "gq_per_push_us": 1e3 * event_ms(push, reps), "gq_per_sample_us": 1e3 * event_ms(sample, reps),
               "gq_per_update_us": 1e3 * event_ms(update, reps)}
        # the uniform path: Python's random.sample on the host, then the index tensor copied to the device (one update's draw)
        ur = ObservationReplay(size, (2, 2), device="cuda", rng=random.Random(0))
        ur.length = size
        torch.cuda.synchronize()
        for _ in range(10):
            torch.as_tensor(ur.sample_indices(12), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            torch.as_tensor(ur.sample_indices(12), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        row["uniform_draw_and_copy_us"] = 1e6 * (time.perf_counter() - t0) / reps
        row = {k: round(v, 2) if isinstance(v, float) else v for k, v in row.items()}
        out.append(row)
        print(json.dumps({"kernels": row}), flush=True)
        del rp, ur
        torch.cuda.empty_cache()
    return out


def trainer_steps(envs, steps, updates):
    import torch

    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    ev = lambda: torch.cuda.Event(enable_timing=True)
    trs = {"uniform": BatchedTrainer(envs, "A", 0, seed=0, updates_per_step=updates),
           "prioritized": BatchedTrainer(envs, "A", 0, seed=0, updates_per_step=updates,
                                         prioritized=dict(alpha=0.6, beta0=0.4, beta_updates=(steps + 1) * updates, eps=1e-6))}
    rows = {k: [] for k in trs}
    try:
        for tr in trs.values():
            tr.env.reset()
        for s in range(steps + 1):  # the first step of each is warm-up
            for name, tr in trs.items():
                e = {}

                def mark(m):
                    e[m] = ev()
                    e[m].record()

                t0 = time.perf_counter()
                rec = tr.step(mark)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if s == 0:
                    continue
                r = {"step_ms": 1e3 * wall, "push_ms": e["env_step"].elapsed_time(e["push"]), "update_ms": e["push"].elapsed_time(e["learn"]) / rec["updates"],
                     "mean_loss": rec["mean_loss"]}
                rows[name].append(r)
                print(json.dumps({"trainer": name, "step": s, **{k: round(v, 3) for k, v in r.items()}}), flush=True)
        med = {name: {k: round(float(np.median([r[k] for r in rs])), 3) for k in ("step_ms", "push_ms", "update_ms")} for name, rs in rows.items()}
        med["envs"], med["updates_per_step"] = envs, updates
        print(json.dumps({"trainer_median": med}), flush=True)
        return med
    finally:
        for tr in trs.values():
            tr.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--updates", type=int, default=8, help="learner updates per batched step")
    ap.add_argument("--reps", type=int, default=200, help="kernel launches per timing")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("per_profile needs a CUDA device")
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    kernels(a.reps)
    trainer_steps(a.envs, a.steps, a.updates)
    print(f"card: {name}, power limit {power}", flush=True)


if __name__ == "__main__":
    main()
