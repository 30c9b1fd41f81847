#!/usr/bin/env python
"""What the learner's optimizer passes cost next to its forward/backward, on one GPU:
  (1) gq_adam, gq_sgd and gq_grad_accumulate on the Q-network's flat fp32 parameter buffer (7.32 M values), CUDA events over back-to-back
      launches, with the bytes each pass must move and the resulting GB/s against the H100 SXM's 3.35 TB/s HBM3;
  (2) one QNetLearner.learn_step at accumulate K = 1 and K = 2 (12 K rows of 200 x 200) for Adam and for SGD, the four learners alternated
      in one process: median and 10th-90th percentile.
Prints the card's name, power limit and SM clocks (read in the same run) and one JSON line per part.
usage: python tools/optimizer_profile.py [--launches 200] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS = 3350.0  # H100 SXM data sheet


def card():
    import torch

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{torch.cuda.get_device_name(0)}, power limit / SM clock / max SM clock: {q}"


def batch(B, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, 4, 200, 200), generator=g).cuda(), torch.randint(0, 6 * 200 * 200, (B, 1), generator=g).cuda(),
            (torch.arange(B) % 2 == 0).float().reshape(B, 1).cuda())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200, help="back-to-back launches per kernel timing")
    ap.add_argument("--reps", type=int, default=20, help="learn steps timed per configuration")
    a = ap.parse_args()
    import torch

    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    if not torch.cuda.is_available():
        raise SystemExit("optimizer_profile needs a CUDA device")
    print("card: " + card(), flush=True)
    ev = lambda: torch.cuda.Event(enable_timing=True)

    # (1) the optimizer passes on the flat buffer
    L = QNetLearner(seed=0)
    n = L.flat.numel()
    g = torch.Generator(device="cuda").manual_seed(1)
    p, grad, m, v, buf, acc = (torch.randn(n, generator=g, device="cuda") * 0.01 for _ in range(6))
    v.abs_()
    st = L._st()
    P = L._p
    kernels = {  # name -> (launch, bytes moved per launch)
        "gq_adam": (lambda: L.L.gq_adam(P(p), P(grad), P(m), P(v), n, 1e-3, 0.9, 0.999, 1e-8, 2e-5, 5, st), 7 * 4 * n),
        "gq_sgd": (lambda: L.L.gq_sgd(P(p), P(grad), P(buf), n, 1e-3, 0.9, 2e-5, 0, st), 5 * 4 * n),
        "gq_grad_accumulate": (lambda: L.L.gq_grad_accumulate(P(acc), P(grad), n, 0, st), 3 * 4 * n),
    }
    res = {}
    for name, (fn, nbytes) in kernels.items():
        for _ in range(10):
            assert fn() == 0, name
        times = []
        for _ in range(5):
            e0, e1 = ev(), ev()
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / a.launches)
        us = float(np.median(times))
        res[name] = {"us": round(us, 2), "MB_moved": round(nbytes / 1e6, 1), "GB_per_s": round(nbytes / us / 1e3, 0),
                     "share_of_3350_GBps": round(nbytes / us / 1e3 / HBM_GBS, 3)}
    print(json.dumps({"optimizer_passes": res, "n_params": n, "launches": a.launches}), flush=True)
    del p, grad, m, v, buf, acc

    # (2) learn steps, four configurations alternated
    cfgs = {f"{o}_K{K}": QNetLearner(seed=0, optimizer=o, accumulate=K) for o in ("adam", "sgd") for K in (1, 2)}
    data = {k: batch(12 * c.accumulate, 7) for k, c in cfgs.items()}
    for k, c in cfgs.items():  # warm-up
        c.learn_step(*data[k])
    torch.cuda.synchronize()
    times = {k: [] for k in cfgs}
    for _ in range(a.reps):
        for k, c in cfgs.items():
            e0, e1 = ev(), ev()
            e0.record()
            c.learn_step(*data[k])
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    med = {k: round(float(np.median(t)), 3) for k, t in times.items()}
    spread = {k: [round(float(np.percentile(t, 10)), 3), round(float(np.percentile(t, 90)), 3)] for k, t in times.items()}
    print(json.dumps({"learn_step_ms": {"median": med, "p10_p90": spread, "reps": a.reps, "rows_per_micro_batch": 12,
                                        "K2_over_K1": {o: round(med[f"{o}_K2"] / med[f"{o}_K1"], 3) for o in ("adam", "sgd")}}}), flush=True)
    print("card: " + card(), flush=True)


if __name__ == "__main__":
    main()
