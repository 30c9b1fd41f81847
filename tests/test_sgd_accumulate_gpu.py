"""SGD and gradient accumulation on the GPU: gq_sgd and gq_grad_accumulate against torch, the learner's K = 1 Adam step unchanged kernel
for kernel, the accumulated gradient against the learner's own blocks (bit for bit) and against the reference's learn() loop in torch,
exact SGD resume from a reference-format checkpoint, and the online trainer with SGD and accumulation."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LR, MOM, WD = 1e-3, 0.9, 2e-5


def _batch(B, seed=0):
    sys.path.insert(0, HERE)
    from test_qnet_learn import _batch as batch

    s, a, r = batch(B + seed) if seed else batch(B)
    return s[:B], a[:B], r[:B]


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ kernels
@pytest.fixture(scope="module")
def learner():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    return QNetLearner(seed=0)


@pytest.mark.parametrize("momentum", [MOM, 0.0])
def test_sgd_step_matches_torch(learner, momentum):
    """three steps of gq_sgd against torch.optim.SGD(lr 1e-3, momentum, weight_decay 2e-5) in fp32 on the device: the first step sets
    the momentum buffer, momentum 0 runs without one"""
    L = learner
    n = 10007
    g = torch.Generator(device="cuda").manual_seed(4)
    p = torch.randn(n, generator=g, device="cuda")
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.SGD([ref], lr=LR, momentum=momentum, weight_decay=WD)
    buf = torch.full((n,), float("nan"), device="cuda") if momentum else None  # the first step must not read it
    for step in (1, 2, 3):
        grad = torch.randn(n, generator=g, device="cuda") * 0.01
        ref.grad = grad.clone()
        opt.step()
        L._ck(L.L.gq_sgd(L._p(p), L._p(grad), L._p(buf), n, LR, momentum, WD, int(step == 1), L._st()), "gq_sgd")
        assert (p - ref.detach()).abs().max() < 1e-6  # one fp32 unit in the last place at |p| ~ 4
        if momentum:
            assert (buf - opt.state[ref]["momentum_buffer"]).abs().max() < 1e-7
        else:
            assert "momentum_buffer" not in opt.state.get(ref, {}) or opt.state[ref]["momentum_buffer"] is None


def test_sgd_refuses_a_missing_buffer(learner):
    L = learner
    x = torch.zeros(8, device="cuda")
    assert L.L.gq_sgd(L._p(x), L._p(x), None, 8, LR, MOM, WD, 1, L._st()) != 0
    assert "gq_sgd" in L.L.gq_last_error().decode()


def test_grad_accumulate_is_torchs_grad_sum(learner):
    L = learner
    n = 10007
    g = torch.Generator(device="cuda").manual_seed(9)
    parts = [torch.randn(n, generator=g, device="cuda") for _ in range(3)]
    acc = torch.full((n,), float("nan"), device="cuda")
    for k, x in enumerate(parts):
        L._ck(L.L.gq_grad_accumulate(L._p(acc), L._p(x), n, int(k == 0), L._st()), "gq_grad_accumulate")
    assert torch.equal(acc, (parts[0] + parts[1]) + parts[2])


# ------------------------------------------------------------------------------------------------ the learner
def _state(L):
    out = {"flat": L.flat.clone(), "step": L.step_count}
    for bn in L.running_mean:
        out[bn] = (L.running_mean[bn].clone(), L.running_var[bn].clone(), L.num_batches_tracked[bn])
    for k in ("m", "v", "momentum_buf"):
        if getattr(L, k, None) is not None:
            out[k] = getattr(L, k).clone()
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], tuple):
            assert torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) and a[k][2] == b[k][2], k
        elif isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def test_one_micro_batch_with_adam_is_the_old_step_bit_for_bit():
    """learn_step with the defaults (Adam, accumulate 1) against the step body before accumulation and SGD existed, run by hand:
    forward_train, backward, gq_adam, _repack - parameters, BatchNorm buffers, moments and kernel launches per step identical"""
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    new, old = QNetLearner(seed=0), QNetLearner(seed=0)
    assert new.grad_acc is None and new.momentum_buf is None
    for step in range(3):
        s, a, r = _batch(12, seed=step)
        n0, f0 = new.launches, new.fw.launches
        loss_new, q_new = new.learn_step(s, a, r, return_pred=True)
        o0, g0 = old.launches, old.fw.launches
        q, saved = old.forward_train(s)
        loss_old, q_old = old.backward(q, saved, a, r)
        old.step_count += 1
        old._ck(old.L.gq_adam(old._p(old.flat), old._p(old.grad), old._p(old.m), old._p(old.v), old.flat.numel(), old.lr, old.betas[0], old.betas[1], old.eps,
                              old.wd, old.step_count, old._st()), "gq_adam")
        old._repack()
        assert (new.launches - n0, new.fw.launches - f0) == (old.launches - o0, old.fw.launches - g0), step
        assert loss_new == float(loss_old) and torch.equal(q_new, q_old)
        _same(_state(new), _state(old))


def _two_slices(R, s, a, r, K=2):
    """the fp32 sum of K separate forward_train + backward calls with weight 1 / K on consecutive slices, in slice order -> (gradient,
    losses, q_pred)"""
    b = s.shape[0] // K
    acc, losses, qs = None, [], []
    for k in range(K):
        rows = slice(k * b, (k + 1) * b)
        q, saved = R.forward_train(s[rows])
        loss, qsel = R.backward(q, saved, a[rows], r[rows], weight=torch.full((b,), 1.0 / K, device="cuda"))
        acc = R.grad.clone() if acc is None else acc + R.grad
        losses.append(float(loss))
        qs.append(qsel.clone())
    return acc, losses, torch.cat(qs)


@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_accumulated_gradient_is_the_sum_of_the_micro_batch_gradients(optimizer):
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    L, R = QNetLearner(seed=0, optimizer=optimizer, accumulate=2), QNetLearner(seed=0)
    s, a, r = _batch(24)
    want, losses, q_want = _two_slices(R, s, a, r)
    before = L.flat.clone()
    loss, q = L.learn_step(s, a, r, return_pred=True)
    assert torch.equal(L.grad_acc, want)
    assert torch.equal(q, q_want) and q.shape == (24,)
    assert abs(loss - sum(losses)) <= 1e-6 * abs(loss)
    assert L.step_count == 1
    for bn in L.running_mean:  # two running-statistics updates, as R's two forwards made
        assert L.num_batches_tracked[bn] == 2 and torch.equal(L.running_mean[bn], R.running_mean[bn]) and torch.equal(L.running_var[bn], R.running_var[bn])
    if optimizer == "sgd":  # then the step is torch's SGD on that gradient
        ref = before.clone().requires_grad_(True)
        opt = torch.optim.SGD([ref], lr=LR, momentum=MOM, weight_decay=WD)
        ref.grad = want.clone()
        opt.step()
        assert (L.flat - ref.detach()).abs().max() < 1e-6 and L.momentum_init


def test_prioritized_weights_are_scaled_per_micro_batch():
    """with importance weights w the micro-batch backward uses w / K: the accumulated gradient is the sum of the weighted blocks"""
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    L, R = QNetLearner(seed=0, optimizer="sgd", accumulate=2), QNetLearner(seed=0)
    s, a, r = _batch(24, seed=3)
    w = torch.linspace(0.2, 1.0, 24, device="cuda")
    acc = None
    for k in range(2):
        rows = slice(12 * k, 12 * (k + 1))
        q, saved = R.forward_train(s[rows])
        R.backward(q, saved, a[rows], r[rows], weight=w[rows] / 2)
        acc = R.grad.clone() if acc is None else acc + R.grad
    L.learn_step(s, a, r, weight=w)
    assert torch.equal(L.grad_acc, acc)


def test_accumulation_matches_the_reference_loop():
    """the reference's learn() with NUMBER_ACCUMULATIONS_BEFORE_UPDATE = 2 and SGD, in torch (fp32, train mode, on the device): two
    12-row slices, loss / 2 and backward() each, then SGD.step().  Every gradient tensor within _check_learn_step's bar (no worse than
    1.1 x torch-autocast-bf16's error + 0.01); the running statistics within test_qnet_eval's bar, num_batches_tracked + 2; the SGD
    step on the same gradient within one fp32 ulp"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    s, a, r = _batch(24, seed=5)
    torch.manual_seed(0)
    net = make_torch_qnet(6)
    L = QNetLearner(net.state_dict(), 0, lr=LR, weight_decay=WD, optimizer="sgd", accumulate=2)
    nets = {}
    for kind in ("fp32", "bf16"):
        m = make_torch_qnet(6)
        m.load_state_dict(net.state_dict())
        nets[kind] = m.cuda().train()
    for k in range(2):
        rows = slice(12 * k, 12 * (k + 1))
        st, ac, rw = s[rows].cuda(), a[rows].cuda(), r[rows].cuda()
        q_pred = nets["fp32"](st).view(12, -1).gather(1, ac)
        (F.binary_cross_entropy(q_pred, rw) / 2).backward()
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            q16 = nets["bf16"](st).float().view(12, -1).gather(1, ac)
        (F.binary_cross_entropy(q16, rw) / 2).backward()
    before = L.flat.clone()
    L.learn_step(s, a, r)
    acc = L._flat_views(L.grad_acc)
    p32, p16 = dict(nets["fp32"].named_parameters()), dict(nets["bf16"].named_parameters())
    bad = {}
    for k, p in p32.items():
        e, auto = _rel(acc[k], p.grad), _rel(p16[k].grad, p.grad)
        if not e <= 1.1 * auto + 0.01:
            bad[k] = (e, auto)
    assert not bad, bad
    ours, sd32, sd16 = L.model_state_dict(), nets["fp32"].state_dict(), nets["bf16"].state_dict()
    for k in sd32:
        if "running" in k:
            e, auto = _rel(ours[k], sd32[k].cpu()), _rel(sd16[k].cpu(), sd32[k].cpu())
            assert e <= 1.1 * auto + 0.01, (k, e, auto)
        elif "num_batches" in k:
            assert int(ours[k]) == int(sd32[k]) == 2, k
    ref = before.clone().requires_grad_(True)
    o2 = torch.optim.SGD([ref], lr=LR, momentum=MOM, weight_decay=WD)
    ref.grad = L.grad_acc.clone()
    o2.step()
    assert (L.flat - ref.detach()).abs().max() < 1e-6


def test_sgd_resume_is_exact(tmp_path):
    """2 SGD steps, checkpoint, from_checkpoint, 1 step == 3 uninterrupted steps, bit for bit; the checkpoint is torch's SGD format"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    batches = [_batch(12, seed=k) for k in range(3)]
    A = QNetLearner(seed=0, optimizer="sgd")
    for b in batches:
        A.learn_step(*b)
    B = QNetLearner(seed=0, optimizer="sgd")
    for b in batches[:2]:
        B.learn_step(*b)
    path = str(tmp_path / "sgd.pt")
    torch.save(B.checkpoint(), path)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert ck["learner_step"] == 2 and set(ck) == {"model_state_dict", "optimizer_state_dict", "learner_step"}
    net = make_torch_qnet(6)
    net.load_state_dict(ck["model_state_dict"], strict=True)
    opt = torch.optim.SGD(net.parameters(), lr=0.5)
    opt.load_state_dict(ck["optimizer_state_dict"])
    assert opt.param_groups[0]["momentum"] == MOM and len(opt.state) == 51
    C = QNetLearner.from_checkpoint(ck, 0)
    assert C.optimizer == "sgd" and C.step_count == 2 and C.momentum_init and C.m is None
    C.learn_step(*batches[2])
    _same(_state(C), _state(A))
    # a checkpoint before the first step has no momentum buffers, like torch's
    fresh = QNetLearner(seed=0, optimizer="sgd").checkpoint()
    assert fresh["optimizer_state_dict"]["state"] == {} and fresh["learner_step"] == 0
    # the reference's own SGD checkpoints have no learner_step: they resume at step 0
    ck.pop("learner_step")
    D = QNetLearner.from_checkpoint(ck, 0)
    assert D.step_count == 0 and torch.equal(D.momentum_buf, B.momentum_buf)
    buf = io.BytesIO()
    torch.save(D.checkpoint(), buf)
    assert torch.load(io.BytesIO(buf.getvalue()), weights_only=False)["learner_step"] == 0


def test_adam_checkpoints_are_unchanged():
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    L = QNetLearner(seed=0)
    L.learn_step(*_batch(12))
    ck = L.checkpoint()
    assert set(ck) == {"model_state_dict", "optimizer_state_dict"} and "betas" in ck["optimizer_state_dict"]["param_groups"][0]
    with pytest.raises(ValueError, match="'sgd'"):
        QNetLearner.from_checkpoint(ck, 0, optimizer="sgd")


# ------------------------------------------------------------------------------------------------ the online trainer
def _trainer(n, **kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    return BatchedTrainer(n, "A", 0, **kw)


@pytest.fixture(scope="module")
def sgd_run(tmp_path_factory):
    """a 16-env SGD trainer with accumulate 2, 1 episode x 5 steps, 1 update per step: (records, checkpoint path, checkpoint, the
    learner's step_count)"""
    tr = _trainer(16, seed=7, updates_per_step=1, optimizer="sgd", accumulate=2)
    try:
        tr.env.reset()
        recs = [tr.step() for _ in range(5)]
        path = str(tmp_path_factory.mktemp("sgd") / "ck.pt")
        return recs, path, tr.save(path), tr.learner.step_count
    finally:
        tr.close()


def test_sgd_trainer_starts_updating_at_48_transitions(sgd_run):
    recs, _, _, step_count = sgd_run
    assert [r["updates"] for r in recs] == [0, 0, 1, 1, 1]  # 16, 32, 48, ... transitions in the replay
    assert all(np.isfinite(r["mean_loss"]) for r in recs[2:]) and step_count == 3


def test_sgd_trainer_checkpoint_resumes(sgd_run):
    from mujoco_rl_ur5_b200.batched_train import COUNTERS

    _, path, ck, _ = sgd_run
    assert ck["learner_step"] == 3 and "momentum" in ck["optimizer_state_dict"]["param_groups"][0]
    tr = _trainer(16, seed=7, updates_per_step=1, load=path, accumulate=2)
    try:
        L = tr.learner
        assert L.optimizer == "sgd" and L.step_count == 3 and L.momentum_init and L.accumulate == 2
        assert tr.steps_done == ck["step"] == 5 * 16 and tr.eps_threshold == ck["epsilon"]
        assert {k: dict(v) for k, v in tr.counters().items()} == {k: dict(ck[k]) for k in COUNTERS}
        bv = L._flat_views(L.momentum_buf)
        for i, k in enumerate(L.names):
            assert torch.equal(bv[k].cpu(), ck["optimizer_state_dict"]["state"][i]["momentum_buffer"]), k
    finally:
        tr.close()


def test_prioritized_accumulating_update_writes_every_drawn_priority():
    tr = _trainer(32, seed=5, updates_per_step=0, accumulate=2, prioritized=dict(beta_updates=10))
    try:
        tr.env.reset()
        tr.step()
        tr.step()
        rp = tr.replay
        seen = []
        upd = rp.update_priorities

        def rec(idx, qsel, reward):
            seen.append((idx.clone(), qsel.clone(), torch.as_tensor(reward).reshape(-1).clone()))
            return upd(idx, qsel, reward)

        rp.update_priorities = rec
        loss = tr.update()
        assert np.isfinite(loss) and tr.learner.step_count == 1
        (idx, qsel, reward), = seen
        assert idx.numel() == qsel.numel() == reward.numel() == 24
        want = {}
        for j in range(24):  # in batch order: a slot drawn twice keeps the later value
            want[int(idx[j])] = (abs(float(reward[j]) - float(qsel[j])) + rp.eps) ** rp.alpha
        leaves = rp.tree[rp.cap:].cpu().numpy()
        for slot, p in want.items():
            assert abs(leaves[slot] - p) <= 1e-12 * p, slot
    finally:
        tr.close()


def test_bootstrapped_accumulation_syncs_the_target_on_the_same_updates():
    syncs = {}
    for K in (1, 2):
        tr = _trainer(64, seed=11, updates_per_step=2, gamma=0.9, target_update=3, accumulate=K, optimizer="sgd")
        try:
            got = []
            sync = tr.learner.sync_target

            def rec(*a, **k):
                got.append(tr.learner.step_count)
                return sync(*a, **k)

            tr.learner.sync_target = rec
            tr.train(1, 4)
            assert tr.learner.step_count == 8
            syncs[K] = got
        finally:
            tr.close()
    assert syncs[1] == syncs[2] == [0, 3, 6]


def test_cli_trains_with_sgd_and_accumulation(tmp_path):
    out = str(tmp_path / "w.pt")
    r = subprocess.run([sys.executable, "-m", "mujoco_rl_ur5_b200.batched_train", "--envs", "64", "--episodes", "1", "--steps-per-episode", "2",
                        "--updates-per-step", "2", "--optimizer", "sgd", "--accumulate", "2", "--out", out], cwd=ROOT, capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    recs = [json.loads(ln) for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(recs) == 2 and all(rec["updates"] == 2 for rec in recs) and all(np.isfinite(rec["mean_loss"]) for rec in recs)
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    ck = torch.load(out, map_location="cpu", weights_only=False)
    net = make_torch_qnet(6)
    net.load_state_dict(ck["model_state_dict"], strict=True)
    opt = torch.optim.SGD(net.parameters(), lr=0.5)
    opt.load_state_dict(ck["optimizer_state_dict"])
    assert len(opt.state) == 51 and ck["learner_step"] == 4


def test_the_reference_agent_resumes_the_sgd_checkpoint(sgd_run, tmp_path):
    """the reference's unchanged Grasp_Agent(load_path=..., optimizer="SGD") loads the trainer's SGD checkpoint into its torch SGD: the
    momentum buffers are the checkpoint's"""
    import shutil

    from tests.test_reference_scripts_gpu import COMPAT, _ref_dir

    ref = _ref_dir()
    if ref is None:
        pytest.skip("reference scripts not staged: run tools/stage_reference.py where the reference exists")
    _, path, ck, _ = sgd_run
    shutil.copy(path, str(tmp_path / "weights.pt"))
    code = ("import json, torch\n"
            "_load = torch.load\n"
            "torch.load = lambda f, *a, **k: _load(f, *a, **{**k, 'weights_only': False})\n"
            "import Grasping_Agent_multidiscrete as G\n"
            "a = G.Grasp_Agent(load_path='weights.pt', optimizer='SGD')\n"
            "ck = torch.load('weights.pt', map_location='cpu')\n"
            "same = all(torch.equal(a.optimizer.state[p]['momentum_buffer'].cpu(), ck['optimizer_state_dict']['state'][i]['momentum_buffer'])\n"
            "           for i, p in enumerate(a.policy_net.parameters()))\n"
            "print('LOADED ' + json.dumps([type(a.optimizer).__name__, a.steps_done, same]))\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, COMPAT, ref]))
    env.pop("GRASP_SCENE", None)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    name, steps, same = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("LOADED "))[7:])
    assert name == "SGD" and steps == ck["step"] and same


def test_offline_trainer_trains_and_resumes_with_sgd(tmp_path):
    """offline_train with optimizer="sgd": an epoch trains, the checkpoint is torch's SGD format, and loading it continues with SGD"""
    from mujoco_rl_ur5_b200.offline_train import OfflineTrainer

    r = np.random.RandomState(3)
    n = 10
    data = (r.randint(0, 256, (n, 200, 200, 3)).astype(np.uint8), r.uniform(0.9, 1.2, (n, 200, 200)).astype(np.float32),
            r.randint(0, 6 * 200 * 200, n), r.randint(0, 2, n))
    tr = OfflineTrainer(data, device=0, batch_size=4, epochs=1, optimizer="sgd")
    hist = tr.run()
    assert len(hist) == 1 and np.isfinite(hist[0]["train_loss"])
    path = str(tmp_path / "offline_sgd.pt")
    tr.save(path)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert ck["learner_step"] == tr.learner.step_count == 2 and len(ck["optimizer_state_dict"]["state"]) == 51
    again = OfflineTrainer(data, device=0, batch_size=4, epochs=1, load=path)
    assert again.learner.optimizer == "sgd" and again.learner.step_count == 2 and again.learner.momentum_init
    assert torch.equal(again.learner.momentum_buf, tr.learner.momentum_buf)
    with pytest.raises(ValueError, match="'adam'"):
        OfflineTrainer(data, device=0, batch_size=4, epochs=1, load=path, optimizer="adam")
