"""Offline trainer (mujoco_rl_ur5_b200/offline_train.py = the reference's `Offline RL/train.py` on the device).

CPU: the random-number plan (split, batch order, per-sample ColorJitter parameters) and the metrics equal what the reference's own code
produces (tests/golden/offline_train_rng.json, written by tests/golden/make_offline_train_golden.py).
GPU: two seeded epochs end to end - finite metrics, a checkpoint that loads strictly into the torch module and Adam, bit-identical runs,
and a test loss that a torch fp32 eval() forward of the saved weights reproduces on the same device-transformed states.
"""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "offline_train_rng.json")
RNG_CASE = {"n": 40, "size": 16, "seed": 30, "batch_size": 15, "epochs": 2}
METRIC_CASES = [{"seed": 1, "batches": [15, 15, 2]}, {"seed": 2, "batches": [7, 15], "all_neg": 0}, {"seed": 3, "batches": [5, 9, 1], "all_pos": 1},
                {"seed": 4, "batches": [1], "all_neg": 0}]


def synthetic_file(directory, n, size, seed=0):
    """a seeded transition file in the reference's format; the action of transition k is k"""
    from mujoco_rl_ur5_b200 import offline_data as od

    r = np.random.RandomState(seed)
    rgb = r.randint(0, 256, (n, size, size, 3)).astype(np.uint8)
    depth = (0.6 + 0.6 * r.rand(n, size, size)).astype(np.float32)
    path = os.path.join(directory, "grasping_data_1.pt")
    od.save_transitions(path, rgb, depth, np.arange(n), r.randint(0, 2, n))
    return path


def metric_batches(case):
    """(predictions [b,1] f32, targets [b,1] int64, a loss value) per batch"""
    g = torch.Generator().manual_seed(case["seed"])
    out = []
    for k, b in enumerate(case["batches"]):
        pred = torch.rand((b, 1), generator=g)
        target = torch.randint(0, 2, (b, 1), generator=g)
        if case.get("all_neg") == k:
            target.zero_()
        if case.get("all_pos") == k:
            target.fill_(1)
        out.append((pred, target, float(torch.rand(1, generator=g))))
    return out


def test_trainer_rng_plan_matches_the_reference():
    """batch indices of both splits and every sample's ColorJitter (order, brightness, contrast, saturation, hue) over 2 epochs equal
    those of the reference's Grasping_Dataset / DataLoader / MULTIDISCRETE_RESNET sequence (train.py:28-76,102,175)"""
    from mujoco_rl_ur5_b200.offline_train import rng_plan

    g = json.load(open(GOLD))["rng"]
    plan = rng_plan(RNG_CASE["n"], RNG_CASE["epochs"], RNG_CASE["batch_size"], RNG_CASE["seed"])
    assert len(plan) == len(g) == RNG_CASE["epochs"]
    for ep, gep in zip(plan, g):
        for split in ("train", "test"):
            assert len(ep[split]) == len(gep[split]), split
            for (idx, fac, order), gb in zip(ep[split], gep[split]):
                assert idx == gb["idx"]
                assert order == gb["order"]
                assert fac == gb["factors"]  # exact: the same float32 draws
    sizes = [len(b[0]) for b in plan[0]["train"]] + [len(b[0]) for b in plan[0]["test"]]
    assert sizes == [15, 15, 2, 8]


def test_metrics_match_the_reference():
    from mujoco_rl_ur5_b200.offline_train import AverageMeter, binary_accuracy

    g = json.load(open(GOLD))["metrics"]
    assert len(g) == len(METRIC_CASES)
    for case, gc in zip(METRIC_CASES, g):
        pos, neg, loss = AverageMeter(), AverageMeter(), AverageMeter()
        for (pred, target, lv), gb in zip(metric_batches(case), gc["batches"]):
            pa, npos, na, nneg = binary_accuracy(pred, target)
            assert [float(pa), float(npos), float(na), float(nneg)] == gb
            pos.update(pa, npos)
            neg.update(na, nneg)
            loss.update(lv, len(pred))
        assert (pos.avg, neg.avg, loss.avg) == (gc["pos_avg"], gc["neg_avg"], gc["loss_avg"])
    assert any(b[1] == 0 for c in g for b in c["batches"]) and any(b[3] == 0 for c in g for b in c["batches"])


# ------------------------------------------------------------------------------------------------ GPU
def _run(path, epochs=2):
    from mujoco_rl_ur5_b200.offline_train import OfflineTrainer

    tr = OfflineTrainer(path, device=0, epochs=epochs, seed=30)
    tr.run()
    return tr


@pytest.mark.gpu
def test_trainer_end_to_end(tmp_path):
    from mujoco_rl_ur5_b200.offline_data import load_transitions
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    r = np.random.RandomState(7)
    n = 60
    rgb = r.randint(0, 256, (n, 200, 200, 3)).astype(np.uint8)
    depth = (0.7 + 0.5 * r.rand(n, 200, 200)).astype(np.float32)
    actions = r.randint(0, 6 * 40000, n)
    rewards = r.randint(0, 2, n)
    from mujoco_rl_ur5_b200 import offline_data as od

    path = str(tmp_path / "data.pt")
    od.save_transitions(path, rgb, depth, actions, rewards)
    tr = _run(path)
    assert [h["epoch"] for h in tr.history] == [1, 2]
    for h in tr.history:
        for k in ("train_loss", "train_pos_acc", "train_neg_acc", "test_loss", "test_pos_acc", "test_neg_acc"):
            assert np.isfinite(h[k]), (k, h)
        assert 0 <= h["train_pos_acc"] <= 1 and 0 <= h["test_neg_acc"] <= 1
    out = str(tmp_path / "w.pt")
    tr.save(out)
    ck = torch.load(out, weights_only=False)
    net = make_torch_qnet(6)
    net.load_state_dict(ck["model_state_dict"], strict=True)
    torch.optim.Adam(net.parameters()).load_state_dict(ck["optimizer_state_dict"])
    nbt = ck["model_state_dict"]["0.RB1.bn1.num_batches_tracked"]
    assert nbt.dtype == torch.int64 and int(nbt) == 2 * 4  # 48 training transitions = 4 batches per epoch
    # same seed, same file: bit-identical checkpoint
    ck2 = _run(path).checkpoint()
    for k, v in ck["model_state_dict"].items():
        assert torch.equal(v, ck2["model_state_dict"][k]), k
    for pid, st in ck["optimizer_state_dict"]["state"].items():
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(st[k], ck2["optimizer_state_dict"]["state"][pid][k])
    # the test loss of the last epoch against torch fp32 eval() on the states the trainer used
    net = net.cuda().eval()
    _, _, acts, rews = load_transitions(path)
    F = torch.nn.functional
    tot, cnt, worst = 0.0, 0, 0.0
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False  # a true fp32 comparison target
    with torch.no_grad():
        for idx, fac, order, q_ours in tr.last_test:
            st = tr.states(idx, fac, order, tr.epoch)
            q = net(st).view(len(idx), -1).gather(1, torch.as_tensor(acts[idx.numpy()]).cuda().view(-1, 1))
            tot += float(F.binary_cross_entropy(q, torch.as_tensor(rews[idx.numpy()]).cuda().float().view(-1, 1))) * len(idx)
            cnt += len(idx)
            worst = max(worst, float((q.view(-1) - q_ours).abs().max()))
    torch.backends.cudnn.allow_tf32 = tf32
    ref = tot / cnt
    print("test loss: ours %.5f, torch fp32 eval %.5f, worst |q - q_fp32| %.4f" % (tr.history[-1]["test_loss"], ref, worst))
    assert worst <= 5e-2
    assert abs(tr.history[-1]["test_loss"] - ref) <= 5e-2 * max(1.0, ref)
