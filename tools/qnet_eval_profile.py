#!/usr/bin/env python
"""Eval-mode Q-net forward (BatchNorm running statistics folded into the weights, batchnorm="running") against the default training-mode
forward (batchnorm="batch", per-image statistics) at the bench's Q-net size, timed alternately in one process with CUDA events after
warm-up; then one offline-training epoch (mujoco_rl_ur5_b200.offline_train) on a seeded synthetic transition file, as transitions/s.
Prints the card's name and power limit (read-only nvidia-smi query) with the numbers.

usage: python tools/qnet_eval_profile.py [images=512] [chunk=64] [rounds=5] [transitions=600] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mujoco_rl_ur5_b200.qnet import QNetForward, make_torch_qnet

FLOP_PER_IMAGE = 41.99424e9  # the forward's convolution work per 200 x 200 image (same figure as tools/qnet_profile.py)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("images", type=int, nargs="?", default=512)
    ap.add_argument("chunk", type=int, nargs="?", default=64)
    ap.add_argument("rounds", type=int, nargs="?", default=5)
    ap.add_argument("transitions", type=int, nargs="?", default=600)
    ap.add_argument("--out", default=None, help="directory for a JSON record of the numbers")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    info = card()
    print("card:", info)
    # non-trivial running statistics: a few seeded training-mode forwards of the fp32 module
    torch.manual_seed(0)
    net = make_torch_qnet(6).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(2)
    with torch.no_grad():
        for _ in range(3):
            net(torch.rand((4, 4, 200, 200), generator=g, device="cuda"))
    sd = {k: v.cpu() for k, v in net.state_dict().items()}
    del net
    fwd = {"running": QNetForward(sd, 0, max_batch=a.chunk, batchnorm="running"), "batch": QNetForward(sd, 0, max_batch=a.chunk)}
    state = torch.rand((a.images, 4, 200, 200), generator=g, device="cuda")
    for f in fwd.values():  # warm-up of every shape (module load, tensor-map encoders, allocator)
        f.forward(state)
    torch.cuda.synchronize()
    times = {k: [] for k in fwd}
    launches = {}
    for _ in range(a.rounds):
        for k, f in fwd.items():
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            n0 = f.launches
            e0.record()
            f.forward(state)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            launches[k] = f.launches - n0
    res = {"card": info, "images": a.images, "chunk": a.chunk, "rounds": a.rounds}
    for k, ts in times.items():
        med = float(np.median(ts))
        res[k] = dict(ms_median=med, ms_min=float(min(ts)), ms_max=float(max(ts)), images_per_s=a.images / med * 1e3,
                      tflops=a.images * FLOP_PER_IMAGE / med / 1e9, launches_per_forward=launches[k])
        print(f"batchnorm={k:8s} {a.images} images, chunks of {a.chunk}: median {med:.2f} ms (min {min(ts):.2f}, max {max(ts):.2f}) "
              f"= {a.images / med * 1e3:.0f} images/s = {a.images * FLOP_PER_IMAGE / med / 1e9:.1f} TFLOP/s, {launches[k]} launches")
    res["running_over_batch_time"] = res["running"]["ms_median"] / res["batch"]["ms_median"]
    print(f"running / batch time: {res['running_over_batch_time']:.3f}")
    del fwd, state
    torch.cuda.empty_cache()

    # one offline-training epoch on a seeded synthetic file (train.py's defaults: batch 15, 80/20 split)
    from mujoco_rl_ur5_b200 import offline_data as od
    from mujoco_rl_ur5_b200.offline_train import OfflineTrainer

    r = np.random.RandomState(0)
    n = a.transitions
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "data.pt")
        od.save_transitions(path, r.randint(0, 256, (n, 200, 200, 3)).astype(np.uint8), (0.7 + 0.5 * r.rand(n, 200, 200)).astype(np.float32),
                            r.randint(0, 6 * 40000, n), r.randint(0, 2, n))
        tr = OfflineTrainer(path, 0, epochs=2)
    tr.run(epochs=1)  # warm-up epoch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr.run(epochs=1)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res["offline_epoch"] = dict(transitions=n, seconds=dt, transitions_per_s=n / dt, train=int(0.8 * n), test=n - int(0.8 * n))
    print(f"offline training epoch: {n} transitions ({int(0.8 * n)} trained, {n - int(0.8 * n)} evaluated) in {dt:.2f} s = {n / dt:.0f} transitions/s")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "qnet_eval_profile.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
