#!/usr/bin/env python
"""Generates tests/golden/reference_io.json by running two of the REFERENCE's own classes, unmodified, on inputs the tests rebuild:

  * `Modules.ReplayBuffer(size, simple=True)` driven like Grasping_Agent_multidiscrete.py:396-401 (one push per step, a sample of B as
    soon as 2 B transitions are stored) for three (size, B, pushes) cases: the stored value of every sampled transition, in order
    (tests/test_replay_buffer.py::test_same_samples_as_the_reference_class);
  * `Offline RL/grasping_dataset.Grasping_Dataset` on a file written by mujoco_rl_ur5_b200.offline_data from a seeded batch: its length,
    item 1's action and reward, and item 1's depth channel (the min-max normalised, noise-added depth of transform_observation after
    np.random.seed(0)) as a seeded sample of pixels (tests/test_offline_data.py::test_reference_dataset_class_reads_our_file).

Run where the reference checkout exists:  python tests/golden/make_reference_io_golden.py [reference dir]
"""
import importlib.util
import json
import os
import sys
import tempfile
import types
from collections import namedtuple

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("GRASP_REFERENCE_DIR", "/root/reference")

from tests.test_offline_data import DATASET_CASE, _batch  # noqa: E402
from tests.test_replay_buffer import REPLAY_CASES, _drive  # noqa: E402
from mujoco_rl_ur5_b200 import offline_data as od  # noqa: E402


def _load(name, path, stubs):
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def replay_sequences():
    mod = _load("ref_modules", os.path.join(REF, "Modules.py"), {"prettytable": types.SimpleNamespace(PrettyTable=object)})
    out = []
    for size, B, n in REPLAY_CASES:
        rb = mod.ReplayBuffer(size, simple=True)  # seeds the global `random` with 20
        seq = _drive(lambda k: rb.push(torch.full((1, 1, 2, 2), float(k)), torch.tensor([[k * 3]]), torch.tensor([[k % 2]])),
                     lambda B_: [int(t.state[0, 0, 0, 0]) for t in rb.sample(B_)], lambda: len(rb), n, size, B)
        out.append({"size": size, "B": B, "pushes": n, "samples": seq})
    return out


def dataset_item():
    mod = _load("ref_grasping_dataset", os.path.join(REF, "Offline RL", "grasping_dataset.py"),
                {"Modules": types.SimpleNamespace(simple_Transition=namedtuple("simple_Transition", ("state", "action", "reward")))})
    rgb, depth, act, rew = _batch(DATASET_CASE["n"], seed=DATASET_CASE["seed"])
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "grasping_data_1.pt")
        od.save_transitions(p, rgb, depth, od.flat_action(act), rew)
        _orig = torch.load
        torch.load = lambda f, *a, **k: _orig(f, *a, **{**k, "weights_only": False})  # the reference predates the weights_only default
        try:
            ds = mod.Grasping_Dataset(p)
        finally:
            torch.load = _orig
        np.random.seed(0)
        state, a, r = ds[DATASET_CASE["item"]]
    dch = state[3].numpy().reshape(-1)
    idx = np.random.RandomState(DATASET_CASE["sample_seed"]).choice(dch.size, DATASET_CASE["samples"], replace=False)
    return {"len": len(ds), "state_shape": list(state.shape), "action": int(a), "reward": int(r), "depth_min": float(dch.min()),
            "depth_max": float(dch.max()), "depth_sum": float(dch.astype(np.float64).sum()), "depth_idx": idx.tolist(),
            "depth_values": dch[idx].astype(np.float64).tolist()}


if __name__ == "__main__":
    out = {"generator": "tests/golden/make_reference_io_golden.py", "replay_buffer": replay_sequences(), "grasping_dataset": dataset_item()}
    json.dump(out, open(os.path.join(HERE, "reference_io.json"), "w"), indent=1)
    print("wrote", os.path.join(HERE, "reference_io.json"))
