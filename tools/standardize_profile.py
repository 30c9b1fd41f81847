#!/usr/bin/env python
"""What the standardised observation path costs on one GPU, on 4096 seeded 200 x 200 observations:
  gq_obs_channel_stats over all of them, gq_obs_to_state_standard on 4096 rows (f32 out, and f32 + bf16 NHWC out) and
  gq_obs_to_state_keyed (the min-max training transform) on the same rows, the four alternated in one process.  CUDA events around
  back-to-back launches; median and 10th-90th percentile over the rounds; bytes moved over time against the H100 SXM's 3.35 TB/s.
Bytes per observation or row: the statistics read rgb + depth = 280 000 B (their second pass reads the depth, 160 000 B, again);
the transforms read 280 000 B and write 640 000 B of f32 state (+ 320 000 B of bf16).  Prints the card's name, power limit and SM
clocks, read in the same run, and one JSON line.
usage: python tools/standardize_profile.py [--rows 4096] [--launches 20] [--rounds 15]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.optimizer_profile import HBM_GBS, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4096)
    ap.add_argument("--launches", type=int, default=20, help="back-to-back launches per timing")
    ap.add_argument("--rounds", type=int, default=15, help="alternated rounds of every kernel")
    a = ap.parse_args()
    import torch

    from mujoco_rl_ur5_b200.qnet import QNetForward, make_torch_qnet

    if not torch.cuda.is_available():
        raise SystemExit("standardize_profile needs a CUDA device")
    print("card: " + card(), flush=True)
    torch.manual_seed(0)
    fw = QNetForward(make_torch_qnet(6).state_dict(), 0)
    L, P, st = fw.L, fw._p, fw._stream()
    B, H, W = a.rows, 200, 200
    HW = H * W
    g = torch.Generator(device="cuda").manual_seed(3)
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    depth = 0.9 + 0.9 * torch.rand((B, H, W), generator=g, device="cuda")
    env = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 1234, dtype=torch.int32, device="cuda")
    ms = np.array([108.3, 120.3, 132.3, 1.53, 67.9, 57.2, 48.9, 0.43], dtype=np.float32)
    state = torch.empty((B, 4, H, W), device="cuda")
    nhwc = torch.empty((B, H, W, 4), dtype=torch.bfloat16, device="cuda")
    red, fac = torch.empty((B, 4), device="cuda"), torch.empty((B, 4), device="cuda")
    order = torch.empty((B, 4), dtype=torch.int32, device="cuda")
    scratch = torch.empty(L.gq_obs_channel_stats_scratch_bytes(B * HW), dtype=torch.uint8, device="cuda")
    out = torch.empty(8, dtype=torch.float64, device="cuda")
    msp = ms.ctypes.data_as(C.c_void_p)
    obs_in = (3 + 4) * HW
    kernels = {  # name -> (launch, bytes moved per launch)
        "gq_obs_channel_stats": (lambda: L.gq_obs_channel_stats(P(rgb), P(depth), B, HW, P(scratch), P(out), st), B * obs_in),
        "gq_obs_to_state_standard_f32": (lambda: L.gq_obs_to_state_standard(P(rgb), P(depth), None, P(env), P(steps), 0, msp, 1.1, 0.001, 5, P(state), None,
                                                                            B, HW, st), B * (obs_in + 16 * HW)),
        "gq_obs_to_state_standard_f32_bf16": (lambda: L.gq_obs_to_state_standard(P(rgb), P(depth), None, P(env), P(steps), 0, msp, 1.1, 0.001, 5, P(state),
                                                                                 P(nhwc), B, HW, st), B * (obs_in + 24 * HW)),
        "gq_obs_to_state_keyed_f32": (lambda: L.gq_obs_to_state_keyed(P(rgb), P(depth), None, P(env), P(steps), 1.1, 0.001, 5, P(red), P(fac), P(order),
                                                                      P(state), None, B, HW, st), B * (obs_in + 16 * HW)),
    }
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for name, (fn, _) in kernels.items():
        for _ in range(3):
            assert fn() == 0, (name, L.gq_last_error())
    torch.cuda.synchronize()
    times = {k: [] for k in kernels}
    for _ in range(a.rounds):
        for name, (fn, _) in kernels.items():
            e0, e1 = ev(), ev()
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / a.launches)
    res = {}
    for name, (_, nbytes) in kernels.items():
        us = float(np.median(times[name]))
        res[name] = {"us": round(us, 1), "p10_p90_us": [round(float(np.percentile(times[name], q)), 1) for q in (10, 90)], "MB_moved": round(nbytes / 1e6, 1),
                     "GB_per_s": round(nbytes / us / 1e3, 0), "share_of_3350_GBps": round(nbytes / us / 1e3 / HBM_GBS, 3)}
    print(json.dumps({"rows": B, "launches": a.launches, "rounds": a.rounds, "kernels": res}), flush=True)
    print("card: " + card(), flush=True)


if __name__ == "__main__":
    main()
