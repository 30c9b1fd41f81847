#!/usr/bin/env python
"""Generates tests/golden/standardize.json and standardize.npz by running the REFERENCE's own code, unmodified:

  * `Grasp_Agent.transform_observation(obs, normalize=False)` (Grasping_Agent_multidiscrete.py:301-368) on the seeded observations of
    tests/test_standardize.py::STATE_CASES, called on a stub `self` (depth_threshold = 1.1, depth_only = False, get_mean_std the
    class's own) in a temporary directory holding a `mean_and_std` with the shipped values, and with torch.randn_like patched to
    zeros: the noise-free standardised states [1,4,H,W] f32 (npz, state_<seed>);
  * normalize.py, executed as it is with a stub `gym` whose env.reset() returns the observations of
    tests/test_standardize.py::normalize_observations one by one: the pickle it writes (hex), its values and element types;
  * the shipped `mean_and_std`: its bytes, values and element types.

Values are stored as float.hex strings.  Run where the reference checkout exists:
    python tests/golden/make_standardize_golden.py [reference dir]
"""
import contextlib
import importlib.util
import io
import json
import os
import pickle
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("GRASP_REFERENCE_DIR", "/root/reference")

from tests.test_standardize import NORMALIZE_CASE, STATE_CASES, normalize_observations, synthetic_obs  # noqa: E402


@contextlib.contextmanager
def stubbed(stubs):
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def entry(values):
    return {"values": [float(v).hex() for v in values], "types": [type(v).__name__ for v in values]}


def agent_class():
    modules = types.ModuleType("Modules")
    for name in ("ReplayBuffer", "Transition", "simple_Transition", "MULTIDISCRETE_RESNET"):
        setattr(modules, name, object)
    tb = types.ModuleType("torch.utils.tensorboard")
    tb.SummaryWriter = object
    stubs = {"gym": types.ModuleType("gym"), "Modules": modules, "torch.utils.tensorboard": tb,
             "termcolor": types.SimpleNamespace(colored=lambda s, *a, **k: s)}
    with stubbed(stubs):
        spec = importlib.util.spec_from_file_location("ref_agent", os.path.join(REF, "Grasping_Agent_multidiscrete.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    return mod.Grasp_Agent


def reference_states(ship_bytes):
    Agent = agent_class()
    out = {}
    cwd = os.getcwd()
    real_randn_like = torch.randn_like
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "mean_and_std"), "wb") as f:
            f.write(ship_bytes)
        os.chdir(tmp)
        torch.randn_like = torch.zeros_like
        try:
            stub = types.SimpleNamespace(depth_threshold=np.round(1.1, decimals=3), depth_only=False)
            stub.get_mean_std = lambda: Agent.get_mean_std(stub)
            for seed, H, W in STATE_CASES:
                rgb, depth = synthetic_obs(seed, H, W)
                s = Agent.transform_observation(stub, {"rgb": rgb.copy(), "depth": depth.copy()}, normalize=False)
                out[f"state_{seed}"] = s.numpy().astype(np.float32)
                assert out[f"state_{seed}"].shape == (1, 4, H, W)
        finally:
            torch.randn_like = real_randn_like
            os.chdir(cwd)
    return out


def run_normalize_py():
    rgb, depth = normalize_observations()
    it = iter(range(NORMALIZE_CASE["n"]))

    class Env:
        def reset(self):
            i = next(it)
            return {"rgb": rgb[i].copy(), "depth": depth[i].copy()}

    gym = types.ModuleType("gym")
    gym.make = lambda name: Env()
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        shutil.copy(os.path.join(REF, "normalize.py"), tmp)
        os.chdir(tmp)
        try:
            with stubbed({"gym": gym, "termcolor": types.SimpleNamespace(colored=lambda s, *a, **k: s)}), contextlib.redirect_stdout(io.StringIO()):
                src = open("normalize.py").read()
                exec(compile(src, os.path.join(REF, "normalize.py"), "exec"), {"__name__": "__main__"})
            with open("mean_and_std", "rb") as f:
                raw = f.read()
        finally:
            os.chdir(cwd)
    return raw


def main():
    with open(os.path.join(REF, "mean_and_std"), "rb") as f:
        ship_bytes = f.read()
    shipped = pickle.loads(ship_bytes)
    states = reference_states(ship_bytes)
    norm_raw = run_normalize_py()
    norm = pickle.loads(norm_raw)
    meta = {
        "shipped": {**entry(shipped), "pickle_hex": ship_bytes.hex()},
        "used": entry(shipped),
        "depth_threshold": float(np.round(1.1, 3)).hex(),
        "states": [{"seed": s, "H": H, "W": W} for s, H, W in STATE_CASES],
        "normalize": {**NORMALIZE_CASE, **entry(norm), "pickle_hex": norm_raw.hex()},
    }
    with open(os.path.join(HERE, "standardize.json"), "w") as f:
        json.dump(meta, f, indent=1)
    np.savez_compressed(os.path.join(HERE, "standardize.npz"), **states)
    print("wrote standardize.json / standardize.npz:", {k: v.shape for k, v in states.items()}, "normalize.py:", [float(v) for v in norm])


if __name__ == "__main__":
    main()
