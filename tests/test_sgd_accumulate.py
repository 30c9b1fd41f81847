"""SGD and gradient accumulation on the host: the reference-format SGD checkpoint (sgd_to_torch / sgd_from_torch through a CPU
torch.optim.SGD), optimiser detection, argument checks of the learner, the trainers and the CLIs, and the online trainer's warm-up gate
and draw size with stand-ins for the environment and the learner.  tests/test_sgd_accumulate_gpu.py covers the kernels, the learner and
the trainer on the GPU."""
import types

import numpy as np
import pytest
import torch

NEW_KEYS = ("maximize", "foreach", "differentiable", "fused")


def _params(seed):
    from mujoco_rl_ur5_b200.qnet_learn import _meta_qnet

    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(p.shape, generator=g) for k, p in _meta_qnet().named_parameters()}


@pytest.mark.parametrize("with_buf", [True, False])
def test_sgd_state_round_trips_through_torch(with_buf):
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import sgd_from_torch, sgd_to_torch

    params, buf = _params(1), (_params(2) if with_buf else None)
    sd = sgd_to_torch(params, buf, 0.003, 0.85, 3e-5)
    g = sd["param_groups"][0]
    assert (g["lr"], g["momentum"], g["dampening"], g["weight_decay"], g["nesterov"]) == (0.003, 0.85, 0, 3e-5, False)
    assert len(g["params"]) == 51 and (len(sd["state"]) == 51) == with_buf
    # torch's own SGD takes it and gives it back unchanged
    opt = torch.optim.SGD(make_torch_qnet(6).parameters(), lr=0.1, momentum=0.5)
    opt.load_state_dict(sd)
    back, hyper = sgd_from_torch(opt.state_dict())
    assert hyper == dict(lr=0.003, momentum=0.85, weight_decay=3e-5)
    if with_buf:
        assert back.keys() == buf.keys() and all(torch.equal(back[k], buf[k]) for k in buf)
    else:
        assert back is None


def test_an_sgd_state_without_the_newer_torch_keys_loads():
    """the 2020-era reference wrote SGD param groups without maximize / foreach / differentiable / fused"""
    from mujoco_rl_ur5_b200.qnet_learn import optimizer_of, sgd_from_torch, sgd_to_torch

    buf = _params(3)
    sd = sgd_to_torch(_params(4), buf, 0.001, 0.9, 2e-5)
    for k in NEW_KEYS:
        sd["param_groups"][0].pop(k, None)
    assert set(sd["param_groups"][0]) == {"lr", "momentum", "dampening", "weight_decay", "nesterov", "params"}
    assert optimizer_of(sd) == "sgd"
    back, hyper = sgd_from_torch(sd)
    assert hyper == dict(lr=0.001, momentum=0.9, weight_decay=2e-5) and all(torch.equal(back[k], buf[k]) for k in buf)


@pytest.mark.parametrize("key,value", [("nesterov", True), ("dampening", 0.1), ("maximize", True)])
def test_sgd_settings_the_learner_lacks_are_refused(key, value):
    from mujoco_rl_ur5_b200.qnet_learn import sgd_from_torch, sgd_to_torch

    sd = sgd_to_torch(_params(5), None, 0.001, 0.9, 2e-5)
    sd["param_groups"][0][key] = value
    with pytest.raises(ValueError, match=key):
        sgd_from_torch(sd)


def test_partial_momentum_buffers_are_refused():
    from mujoco_rl_ur5_b200.qnet_learn import sgd_from_torch, sgd_to_torch

    sd = sgd_to_torch(_params(6), _params(7), 0.001, 0.9, 2e-5)
    del sd["state"][3]
    with pytest.raises(ValueError, match="some parameters"):
        sgd_from_torch(sd)


def test_the_optimizer_is_detected_and_a_mismatch_is_refused():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner, adam_to_torch, optimizer_of, sgd_to_torch

    p = _params(8)
    adam, sgd = adam_to_torch(p, p, p, 0, 0.001, (0.9, 0.999), 1e-8, 2e-5), sgd_to_torch(p, None, 0.001, 0.9, 2e-5)
    assert optimizer_of(adam) == "adam" and optimizer_of(sgd) == "sgd"
    for other in (torch.optim.RMSprop, torch.optim.Adagrad):  # (RMSprop has a momentum too)
        with pytest.raises(ValueError, match="neither"):
            optimizer_of(other([torch.zeros(1, requires_grad=True)]).state_dict())
    # the mismatch is found before any device is touched
    for opt, asked, held in ((sgd, "adam", "sgd"), (adam, "sgd", "adam")):
        with pytest.raises(ValueError) as e:
            QNetLearner.from_checkpoint({"model_state_dict": {}, "optimizer_state_dict": opt}, 0, optimizer=asked)
        assert repr(asked) in str(e.value) and repr(held) in str(e.value)


BAD_OPT = [dict(optimizer="rmsprop"), dict(optimizer="SGD"), dict(accumulate=0), dict(accumulate=-2), dict(accumulate=2.0), dict(accumulate=True),
           dict(momentum=-0.1), dict(momentum=float("nan")), dict(momentum=float("inf")), dict(momentum="0.9")]


@pytest.mark.parametrize("kw", BAD_OPT, ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_bad_optimizer_settings_are_refused(kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer
    from mujoco_rl_ur5_b200.offline_train import OfflineTrainer
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner, check_optimizer

    full = {**dict(optimizer="sgd", accumulate=1, momentum=0.9), **kw}
    with pytest.raises(ValueError):
        check_optimizer(full["optimizer"], full["accumulate"], full["momentum"])
    with pytest.raises(ValueError):  # before any environment or device is touched
        BatchedTrainer(4, "A", 0, **kw)
    with pytest.raises(ValueError):
        QNetLearner(None, 0, **kw)
    if "accumulate" not in kw:
        with pytest.raises(ValueError):
            OfflineTrainer(None, 0, **kw)


def test_good_optimizer_settings_pass():
    from mujoco_rl_ur5_b200.qnet_learn import check_optimizer

    assert check_optimizer("adam", 1) == ("adam", 1, 0.9)
    assert check_optimizer("sgd", 4, 0) == ("sgd", 4, 0.0) and check_optimizer("sgd", 2, 0.95) == ("sgd", 2, 0.95)


@pytest.mark.parametrize("argv", [["--accumulate", "0"], ["--accumulate", "-1"], ["--optimizer", "rmsprop"], ["--momentum", "-0.5"],
                                  ["--momentum", "nan"], ["--accumulate", "1.5"]])
def test_cli_refuses_bad_optimizer_arguments(argv, capsys):
    from mujoco_rl_ur5_b200.batched_train import main

    with pytest.raises(SystemExit) as e:
        main(["--envs", "4"] + argv)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert any(w in err for w in ("accumulate", "optimizer", "momentum")), err


@pytest.mark.parametrize("argv", [["--optimizer", "adagrad"], ["--momentum", "-1"]])
def test_offline_cli_refuses_bad_optimizer_arguments(argv, capsys):
    from mujoco_rl_ur5_b200.offline_train import main

    with pytest.raises(SystemExit) as e:
        main(["data.pt"] + argv)
    assert e.value.code == 2


@pytest.mark.parametrize("B,K", [(13, 2), (12, 5), (1, 2)])
def test_learn_step_refuses_rows_that_do_not_split(B, K):
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    stand_in = types.SimpleNamespace(accumulate=K, torch=torch)  # the check comes before any device work
    with pytest.raises(ValueError, match="micro-batches"):
        QNetLearner.learn_step(stand_in, torch.zeros(B, 4, 2, 2), torch.zeros(B, dtype=torch.int64), torch.zeros(B))


# ------------------------------------------------------------------------------------------------ the online trainer with stand-ins
class _FakeEnv:
    IMAGE_WIDTH = IMAGE_HEIGHT = 4
    TABLE_HEIGHT = 0.9
    rotations = list(range(6))
    cam = 0

    def __init__(self, n, scene, device, env_index_offset=0):
        self.n = n
        self.engine = types.SimpleNamespace(device=torch.device("cpu"))
        self.arrays = {"cam_fovy": [45.0], "cam_pos0": [0.0, 0.0, 2.0], "cam_mat0": list(np.eye(3).ravel())}
        self.current_observation = self._obs()

    def _obs(self):
        return {"rgb": torch.zeros(self.n, 4, 4, 3, dtype=torch.uint8), "depth": torch.ones(self.n, 4, 4)}

    def step(self, act):
        return self._obs(), np.zeros(self.n, dtype=np.float64), None, None


def _fake_trainer(monkeypatch, n, **kw):
    from mujoco_rl_ur5_b200 import batched_train

    made = []

    def learner(*a, **k):
        made.append(k)
        return types.SimpleNamespace(step_count=0)

    monkeypatch.setattr(batched_train, "BatchedGraspEnv", _FakeEnv)
    monkeypatch.setattr(batched_train, "QNetLearner", learner)
    tr = batched_train.BatchedTrainer(n, **kw)
    act = torch.zeros(n, 2, dtype=torch.int32)
    tr.act = lambda obs: (None, act, torch.zeros(n, dtype=torch.bool), torch.zeros(n, dtype=torch.bool))
    return tr, made


@pytest.mark.parametrize("K", [1, 2, 3])
def test_warm_up_gate_waits_for_two_full_accumulated_batches(monkeypatch, K):
    """the reference's `len(memory) < 2 * BATCH_SIZE` with BATCH_SIZE = 12 K: updating starts once the replay holds 24 K transitions"""
    tr, made = _fake_trainer(monkeypatch, 4, optimizer="sgd", accumulate=K, updates_per_step=2)
    assert made[-1]["accumulate"] == K and made[-1]["optimizer"] == "sgd" and made[-1]["momentum"] == 0.9
    seen = []
    tr.update = lambda: seen.append(len(tr.replay)) or 0.5
    recs = [tr.step() for _ in range(6 * K + 2)]
    first = next(i for i, r in enumerate(recs) if r["updates"])
    assert first == 6 * K - 1 and seen[0] == 24 * K  # after the (6 K)-th batched step of 4 envs
    assert all(r["updates"] == (2 if i >= first else 0) for i, r in enumerate(recs))


def test_one_update_draws_all_micro_batches_in_one_call(monkeypatch):
    tr, _ = _fake_trainer(monkeypatch, 4, accumulate=2, batch_size=12)
    drawn, trained = [], []

    def sample(n, *a):
        drawn.append(n)
        return torch.zeros(n, 4, 4, 4), torch.zeros(n, 1, dtype=torch.int64), torch.zeros(n, 1)

    tr.replay = types.SimpleNamespace(sample=sample)
    tr.learner.fw = None
    tr.learner.learn_step = lambda s, a, r, **k: trained.append(s.shape[0]) or 0.25
    assert tr.update() == 0.25 and drawn == [24] and trained == [24]


def test_the_trainer_leaves_the_optimizer_to_a_checkpoint(monkeypatch):
    """with `load` and no optimizer the learner takes the checkpoint's (no optimizer keyword); an explicit one is passed through"""
    from mujoco_rl_ur5_b200 import batched_train

    calls = []
    fake = types.SimpleNamespace(from_checkpoint=lambda ck, dev, **k: calls.append(k) or types.SimpleNamespace(step_count=0))
    monkeypatch.setattr(batched_train, "BatchedGraspEnv", _FakeEnv)
    monkeypatch.setattr(batched_train, "QNetLearner", fake)
    batched_train.BatchedTrainer(4, load={"step": 8}, accumulate=2)
    batched_train.BatchedTrainer(4, load={"step": 8}, optimizer="sgd")
    assert calls == [dict(process_group=None, accumulate=2), dict(process_group=None, accumulate=1, optimizer="sgd")]
