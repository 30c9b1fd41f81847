#!/usr/bin/env python
"""Generates tests/golden/offline_train_rng.json from the REFERENCE's own code, unmodified, on inputs the tests rebuild:

  * the random-number plan of `Offline RL/train.py`: its `Grasping_Dataset` and `Modules.MULTIDISCRETE_RESNET` driven in train.py's
    order (manual_seed(30) :28-31, random_split 80/20 :69-71, DataLoader(shuffle=True) x 2 :73-74, network :76, then per epoch the
    training loader and the test loader) for 2 epochs of batch 15 over a small synthetic file whose actions equal the transition index.
    Per epoch: every batch's transition indices and every sample's ColorJitter parameters, captured by wrapping
    torchvision's ColorJitter.get_params (tests/test_offline_train.py::test_trainer_rng_plan_matches_the_reference);
  * `binary_accuracy` and `AverageMeter` of train.py (:198-252), taken out of the script with `ast` (it trains at import), on seeded
    batches including ones without positives or without negatives (tests/test_offline_train.py::test_metrics_match_the_reference).

Run where the reference checkout exists:  python tests/golden/make_offline_train_golden.py [reference dir]
"""
import ast
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("GRASP_REFERENCE_DIR", "/root/reference")

from tests.test_offline_train import METRIC_CASES, RNG_CASE, metric_batches, synthetic_file  # noqa: E402


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


def rng_plan():
    import random

    import torchvision.transforms as T
    from torch.utils.data import DataLoader, random_split

    modules = _load("ref_modules", os.path.join(REF, "Modules.py"), {"prettytable": types.SimpleNamespace(PrettyTable=object)})
    gd = _load("ref_grasping_dataset", os.path.join(REF, "Offline RL", "grasping_dataset.py"), {"Modules": modules})
    captured = []
    orig = T.ColorJitter.get_params

    def spy(*a):
        r = orig(*a)
        captured.append((r[0].tolist(), [float(v) for v in r[1:]]))
        return r

    T.ColorJitter.get_params = staticmethod(spy)
    _orig_load = torch.load
    torch.load = lambda f, *a, **k: _orig_load(f, *a, **{**k, "weights_only": False})  # the reference predates the weights_only default
    try:
        with tempfile.TemporaryDirectory() as d:
            path = synthetic_file(d, RNG_CASE["n"], RNG_CASE["size"])
            seed, bs = RNG_CASE["seed"], RNG_CASE["batch_size"]
            torch.manual_seed(seed)                                   # train.py:28-31
            np.random.seed(seed)
            random.seed(seed)
            ds = gd.Grasping_Dataset(path)                            # :67
            train_size = int(0.8 * len(ds))                           # :69-71
            trainset, testset = random_split(ds, [train_size, len(ds) - train_size])
            train_loader = DataLoader(dataset=trainset, batch_size=bs, shuffle=True)  # :73-74
            test_loader = DataLoader(dataset=testset, batch_size=bs, shuffle=True)
            modules.MULTIDISCRETE_RESNET(6)                           # :76 (training itself draws no random numbers)
            epochs = []
            for _ in range(RNG_CASE["epochs"]):
                ep = {}
                for name, loader in (("train", train_loader), ("test", test_loader)):
                    batches = []
                    for data in loader:
                        idx = data[1].tolist()                        # the action of transition k is k
                        jit = captured[:len(idx)]
                        del captured[:len(idx)]
                        batches.append({"idx": idx, "order": [j[0] for j in jit], "factors": [j[1] for j in jit]})
                    ep[name] = batches
                epochs.append(ep)
            assert not captured
    finally:
        T.ColorJitter.get_params = staticmethod(orig)
        torch.load = _orig_load
    return epochs


def metrics():
    src = open(os.path.join(REF, "Offline RL", "train.py")).read()
    keep = [n for n in ast.parse(src).body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in ("binary_accuracy", "AverageMeter")]
    ns = {"torch": torch}
    exec(compile(ast.Module(body=keep, type_ignores=[]), "train.py", "exec"), ns)
    out = []
    for case in METRIC_CASES:
        pos, neg, loss = ns["AverageMeter"]("p"), ns["AverageMeter"]("n"), ns["AverageMeter"]("l")
        per_batch = []
        for pred, target, lv in metric_batches(case):
            pa, npos, na, nneg = ns["binary_accuracy"](pred, target)
            pos.update(pa, npos)
            neg.update(na, nneg)
            loss.update(lv, len(pred))
            per_batch.append([float(pa), float(npos), float(na), float(nneg)])
        out.append({"batches": per_batch, "pos_avg": float(pos.avg), "neg_avg": float(neg.avg), "loss_avg": float(loss.avg)})
    return out


if __name__ == "__main__":
    out = {"generator": "tests/golden/make_offline_train_golden.py", "torch": torch.__version__, "rng": rng_plan(), "metrics": metrics()}
    json.dump(out, open(os.path.join(HERE, "offline_train_rng.json"), "w"), indent=1)
    print("wrote", os.path.join(HERE, "offline_train_rng.json"))
