"""Bootstrapped Q-learning on the GPU: gq_head_max_target against the forward's own head and arg-max (bit for bit) and against the fp32
torch network, the loss kernels with fractional targets against float64 torch, the target network's syncs, the next-observation
replay, and the trainer with gamma > 0 (determinism, sharding, gamma = 0 unchanged, checkpoints)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _stepped_sd(seed=0):
    """make_torch_qnet(6) after a few training-mode forwards: non-trivial running statistics"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    torch.manual_seed(seed)
    net = make_torch_qnet(6)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for _ in range(3):
            net(torch.rand((2, 4, 200, 200), generator=g))
    return net.eval().state_dict()


def _rewards(B, seed):
    r = (torch.rand(B, generator=torch.Generator().manual_seed(seed)) < 0.5).float()
    r[0] = 1.0
    if B > 1:
        r[1] = 0.0
    return r.cuda()


def _torch_target(r, gamma, qmax):
    """the fp32 target torch computes: clamp(r + tensor(gamma, f32) * qmax, max=1), each op rounded on its own"""
    return torch.clamp(r + torch.tensor(gamma, dtype=torch.float32, device=qmax.device) * qmax, max=1.0)


def _max_target(f, x, h, w, r, gamma):
    B = x.shape[0]
    qmax = torch.full((B,), -7.0, device="cuda")
    y = torch.full((B,), -7.0, device="cuda")
    f._ck(f.L.gq_head_max_target(f._p(x), f._p(f.w_head), f._p(f.b_head), f._p(r), float(gamma), f._p(qmax), f._p(y), B, h, w, f.A, f._stream()),
          "gq_head_max_target")
    return qmax, y


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("B", [1, 12, 15])
def test_head_max_target_is_the_forwards_maximum(B):
    from mujoco_rl_ur5_b200.qnet import QNetForward

    f = QNetForward(_stepped_sd(0), 0, max_batch=64, batchnorm="running")
    state = torch.rand((B, 4, 200, 200), generator=torch.Generator().manual_seed(B)).cuda()
    x, h, w = f._trunk(state)  # the real head input of a forward
    q = f._head(x, h, w)
    _, val = f.greedy(q)
    r = _rewards(B, B)
    for gamma in (0.9, 0.0, 1.0, 0.3):
        qmax, y = _max_target(f, x, h, w, r, gamma)
        assert torch.equal(qmax, val), (gamma, (qmax - val).abs().max())
        assert torch.equal(y, _torch_target(r, gamma, qmax)), gamma
        assert torch.equal(y[r == 1], torch.ones_like(y[r == 1]))
        if gamma == 0.0:
            assert torch.equal(y, r)
        qmax2, y2 = _max_target(f, x, h, w, r, gamma)  # deterministic
        assert torch.equal(qmax, qmax2) and torch.equal(y, y2)
    # max_target: the same through the trunk, chunked like forward
    qm, ym = f.max_target(state, r, 0.9)
    assert torch.equal(qm, val) and torch.equal(ym, _torch_target(r, 0.9, val))
    f5 = QNetForward(_stepped_sd(0), 0, max_batch=5, batchnorm="running")
    qm5, ym5 = f5.max_target(state, r, 0.9)
    assert torch.equal(qm5, qm) and torch.equal(ym5, ym)


@pytest.mark.parametrize("B,H,W,A", [(3, 37, 41, 6), (2, 16, 16, 8), (1, 1, 5, 1), (4, 33, 17, 3)])
def test_head_max_target_at_other_shapes(B, H, W, A):
    """random head inputs at map sizes that are not multiples of the tile (and a single row), other A: qmax = gq_argmax's val of gq_head_up2"""
    from mujoco_rl_ur5_b200.qnet import QNetForward, make_torch_qnet

    torch.manual_seed(1)
    sd = make_torch_qnet(A).state_dict()
    f = QNetForward(sd, 0)
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    x = (torch.randn((B, H, W, 64), generator=g, device="cuda") * 2).to(torch.bfloat16)
    q = f._head(x, H, W)
    _, val = f.greedy(q)
    qmax, y = _max_target(f, x, H, W, torch.zeros(B, device="cuda"), 0.5)
    assert torch.equal(qmax, val) and torch.equal(y, _torch_target(torch.zeros(B, device="cuda"), 0.5, val))


def test_target_values_agree_with_the_fp32_torch_network():
    """the synced target network's qmax against make_torch_qnet(6).eval() in fp32 on the learner's weights and running statistics; the
    bar is the whole-map bar of tests/test_qnet_eval.py (max |err| 5e-2), which bounds the error of a maximum too"""
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    sys.path.insert(0, HERE)
    from test_qnet_learn import _batch

    L = QNetLearner(seed=0)
    for B in (3, 12):
        s, a, r = _batch(B)
        L.learn_step(s, a, r)
    tgt = L.sync_target()
    B = 12
    state = torch.rand((B, 4, 200, 200), generator=torch.Generator().manual_seed(21))
    r = _rewards(B, 3)
    qmax, y = tgt.max_target(state.cuda(), r, 0.9)
    net = make_torch_qnet(6)
    net.load_state_dict(L.model_state_dict(), strict=True)
    net = net.cuda().eval()
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref_q = net(state.cuda())
    torch.backends.cudnn.allow_tf32 = tf32
    ref = ref_q.view(B, -1).max(1)[0]
    map_err = (tgt.forward(state.cuda()) - ref_q).abs()
    assert float(map_err.mean()) <= 5e-3 and float(map_err.max()) <= 5e-2, (float(map_err.mean()), float(map_err.max()))
    assert float((qmax - ref).abs().max()) <= 5e-2, (qmax, ref)
    assert torch.equal(y, _torch_target(r, 0.9, qmax))
    assert bool(((y > 0) & (y <= 1)).all())


@pytest.mark.parametrize("weighted", [False, True])
def test_loss_head_backward_with_fractional_targets(weighted):
    """gq_loss_head_bwd(_weighted) with targets in (0, 1): loss terms and head gradients against float64 torch BCE on the kernel's q"""
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    sys.path.insert(0, HERE)
    from test_qnet_learn import _batch

    B = 12
    L = QNetLearner(seed=0)
    s, a, _ = _batch(B)
    q, saved = L.forward_train(s)
    fw = L.fw
    H = W = 100
    A = fw.A
    g = torch.Generator().manual_seed(7)
    y = (0.02 + 0.96 * torch.rand(B, generator=g)).cuda()
    wt = (0.2 + torch.rand(B, generator=g)).cuda()
    action = a.reshape(B).cuda()
    x = saved["b5"]
    lt, qsel = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    dX = torch.empty((B, H * W, 64), dtype=torch.bfloat16, device="cuda")
    dWp, dbp = torch.empty((B, A, 64), device="cuda"), torch.empty((B, A), device="cuda")
    dW, db = torch.empty((A, 64), device="cuda"), torch.empty(A, device="cuda")
    args = [L._p(q), L._p(x), L._p(fw.w_head), L._p(action), L._p(y)]
    outs = [B, A, H, W, L._p(lt), L._p(qsel), L._p(dX), L._p(dWp), L._p(dbp), L._p(dW), L._p(db), L._st()]
    if weighted:
        L._ck(L.L.gq_loss_head_bwd_weighted(*args, L._p(wt), *outs), "gq_loss_head_bwd_weighted")
    else:
        L._ck(L.L.gq_loss_head_bwd(*args, *outs), "gq_loss_head_bwd")
    torch.cuda.synchronize()
    assert torch.equal(qsel, q.view(B, -1).gather(1, action[:, None])[:, 0])
    # float64 torch on the same q: BCE and its gradient w.r.t. the pre-sigmoid value v, then v's gradient w.r.t. the head
    qd = qsel.double().requires_grad_()
    wd = wt.double() if weighted else None
    terms = F.binary_cross_entropy(qd, y.double(), weight=wd, reduction="none")
    F.binary_cross_entropy(qd, y.double(), weight=wd).backward()
    gv = (qd.grad * qd.detach() * (1 - qd.detach()))  # dL/dv
    assert float(((lt.double() - terms.detach()).abs() / terms.detach()).max()) <= 1e-5
    W64 = fw.w_head.double().requires_grad_()
    b64 = fw.b_head.double().requires_grad_()
    z = torch.einsum("bhwc,ac->bahw", x.view(B, H, W, 64).double(), W64) + b64[None, :, None, None]
    v = F.interpolate(z, scale_factor=2, mode="bilinear", align_corners=True).reshape(B, -1).gather(1, action[:, None])[:, 0]
    (v * gv).sum().backward()
    for got, ref in ((dW, W64.grad), (db, b64.grad)):
        assert float((got.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) + 1e-9, (float((got.double() - ref).abs().max()), float(ref.abs().max()))


# ------------------------------------------------------------------------------------------------ the target network
def _packed(f):
    out = {"w_first": f.w_first, "w_head": f.w_head, "b_head": f.b_head}
    for i, b in enumerate(f.blocks):
        out.update({f"{i}.{k}": v for k, v in b.items() if isinstance(v, torch.Tensor)})
    return {k: v.clone() for k, v in out.items()}


def test_sync_target_is_the_eval_forward_and_stays_put():
    from mujoco_rl_ur5_b200.qnet import QNetForward
    from mujoco_rl_ur5_b200.qnet_learn import QNetLearner

    sys.path.insert(0, HERE)
    from test_qnet_learn import _batch

    L = QNetLearner(seed=0)
    s, a, r = _batch(12)
    L.learn_step(s, a, r)
    assert L.target is None
    tgt = L.sync_target()
    assert L.target is tgt and L.target_step == 1 and tgt.batchnorm == "running"
    want = _packed(QNetForward(L.model_state_dict(), 0, batchnorm="running"))
    got = _packed(tgt)
    assert want.keys() == got.keys() and len(got) == 3 + 6 * 4
    for k in want:
        assert torch.equal(got[k], want[k]), k
    q0 = tgt.forward(s[:2].cuda())
    for _ in range(2):
        L.learn_step(s, a, r)
    for k, v in _packed(tgt).items():
        assert torch.equal(v, got[k]), k  # the learner's steps leave the target alone
    assert torch.equal(tgt.forward(s[:2].cuda()), q0)
    assert not torch.equal(_packed(L.eval_forward())["w_head"], got["w_head"])


def _trainer(n, **kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    return BatchedTrainer(n, "A", 0, **kw)


def _record_syncs(tr):
    syncs = []
    sync = tr.learner.sync_target

    def rec(*a, **k):
        syncs.append(tr.learner.step_count)
        return sync(*a, **k)

    tr.learner.sync_target = rec
    return syncs


@pytest.fixture(scope="module")
def bootstrap_runs(tmp_path_factory):
    """two seeded gamma = 0.9 trainers, 64 envs, 2 episodes x 3 steps, 2 updates per step, target_update 5: (checkpoint paths, syncs)"""
    paths, syncs = [], []
    for run in range(2):
        tr = _trainer(64, seed=11, updates_per_step=2, gamma=0.9, target_update=5)
        try:
            assert tr.replay.next_obs and tr.replay.next_rgb is not None
            syncs.append(_record_syncs(tr))
            tr.train(2, 3)
            assert tr.learner.step_count == 12
            p = str(tmp_path_factory.mktemp(f"run{run}") / "ck.pt")
            tr.save(p)
            paths.append(p)
        finally:
            tr.close()
    return paths, syncs


def test_bootstrapped_training_is_deterministic_and_syncs_on_schedule(bootstrap_runs):
    paths, syncs = bootstrap_runs
    assert syncs[0] == syncs[1] == [0, 5, 10]
    assert open(paths[0], "rb").read() == open(paths[1], "rb").read()
    ck = torch.load(paths[0], map_location="cpu", weights_only=False)
    from tests.test_batched_train import REFERENCE_KEYS

    assert set(ck) == REFERENCE_KEYS  # the target network is not saved


def test_resumed_trainer_syncs_first_then_on_schedule(bootstrap_runs):
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    path = bootstrap_runs[0][0]
    make_torch_qnet(6).load_state_dict(torch.load(path, map_location="cpu", weights_only=False)["model_state_dict"], strict=True)
    tr = _trainer(64, seed=11, updates_per_step=2, gamma=0.9, target_update=5, load=path)
    try:
        assert tr.learner.step_count == 12 and tr.learner.target is None
        syncs = _record_syncs(tr)
        tr.env.reset()
        for _ in range(2):
            tr.step()
        assert syncs == [12, 15] and tr.learner.step_count == 16
    finally:
        tr.close()


def test_the_reference_agent_resumes_from_a_bootstrapped_checkpoint(bootstrap_runs, tmp_path):
    import shutil

    from tests.test_reference_scripts_gpu import COMPAT, _ref_dir

    ref = _ref_dir()
    if ref is None:
        pytest.skip("reference scripts not staged: run tools/stage_reference.py where the reference exists")
    path = bootstrap_runs[0][0]
    ck = torch.load(path, map_location="cpu", weights_only=False)
    shutil.copy(path, str(tmp_path / "weights.pt"))
    code = ("import json, torch\n"
            "_load = torch.load\n"
            "torch.load = lambda f, *a, **k: _load(f, *a, **{**k, 'weights_only': False})\n"
            "import Grasping_Agent_multidiscrete as G\n"
            "a = G.Grasp_Agent(load_path='weights.pt')\n"
            "st = a.optimizer.state[next(iter(a.policy_net.parameters()))]\n"
            "print('LOADED ' + json.dumps([a.steps_done, float(st['step'])]))\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, COMPAT, ref]))
    env.pop("GRASP_SCENE", None)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    steps, adam_step = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("LOADED "))[7:])
    assert steps == ck["step"] and adam_step == 12


# ------------------------------------------------------------------------------------------------ replay and trainer
@pytest.mark.parametrize("prioritized", [None, dict(beta_updates=10)])
def test_next_states_are_the_acting_states_of_the_next_step(prioritized):
    """transition (t, e): its regenerated next state = the state env e acts on at step t + 1, or at an episode's end the keyed transform
    of the observation before the reset (with the next step's key); drawn batches carry the next states of their slots"""
    N = 64
    tr = _trainer(N, seed=4, updates_per_step=0, gamma=0.5, target_update=3, prioritized=prioritized)
    acting, pre_reset = [], []
    act, reset = tr.act, tr.env.reset

    def act_rec(obs):
        out = act(obs)
        acting.append(out[0].clone())
        return out

    def reset_rec():
        if tr.env.current_observation is not None:
            pre_reset.append({k: v.clone() for k, v in tr.env.current_observation.items()})
        return reset()

    tr.act, tr.env.reset = act_rec, reset_rec
    try:
        tr.train(2, 2)
        rp, fw = tr.replay, tr.learner.fw
        keyed = lambda o, key: fw.obs_to_state_keyed(o["rgb"], o["depth"], tr.genv, torch.full((N,), key), tr.seed, depth_threshold=tr.depth_threshold,
                                                     noise_std=tr.noise_std)
        nxt = lambda t: rp._states(torch.arange(t * N, (t + 1) * N, device="cuda"), fw, tr.seed, tr.depth_threshold, tr.noise_std, nxt=True)
        assert torch.equal(nxt(0), acting[1]) and torch.equal(nxt(2), acting[3])
        assert len(pre_reset) == 1
        at_end = keyed(pre_reset[0], 2 * N)
        assert torch.equal(nxt(1), at_end) and not torch.equal(at_end, acting[2])  # not the observation after the reset
        last = nxt(3)
        assert torch.equal(last, keyed(tr.env.current_observation, 4 * N))
        for t in range(4):  # and the stored states are the acting states
            assert torch.equal(rp._states(torch.arange(t * N, (t + 1) * N, device="cuda"), fw, tr.seed, tr.depth_threshold, tr.noise_std), acting[t])
        if prioritized is None:
            st = rp.rng.getstate()
            idx = rp.sample_indices(12)
            rp.rng.setstate(st)
            s, _, _, s2 = rp.sample(12, fw, tr.seed, tr.depth_threshold, tr.noise_std)
        else:
            s, _, _, s2, idx, _ = rp.sample(12, fw, tr.seed, 0.4, 0, 0, tr.depth_threshold, tr.noise_std)
            idx = idx.tolist()
        for row, slot in enumerate(idx):
            t, e = divmod(slot, N)
            assert torch.equal(s[row], acting[t][e])
            assert torch.equal(s2[row], acting[t + 1][e] if t in (0, 2) else (at_end[e] if t == 1 else last[e])), (row, slot)
    finally:
        tr.close()


def test_sharded_bootstrapping_trainers_act_like_one():
    one = _trainer(256, seed=3, updates_per_step=0, gamma=0.9, target_update=4)
    two = [_trainer(128, seed=3, updates_per_step=0, env_index_offset=o, n_total=256, gamma=0.9, target_update=4) for o in (0, 128)]
    try:
        for tr in [one] + two:
            tr.env.reset()
        for t in range(3):
            one.step()
            for tr in two:
                tr.step()
            for k in ("actions", "is_random", "reward"):
                assert np.array_equal(np.asarray(one.last_step[k]), np.concatenate([np.asarray(tr.last_step[k]) for tr in two])), (t, k)
        for s in range(3):
            for h, tr in enumerate(two):
                rows = torch.arange(s * 128, (s + 1) * 128, device="cuda")
                want = one.replay._states(rows + s * 128 + h * 128, one.learner.fw, 3, one.depth_threshold, one.noise_std, nxt=True)
                got = tr.replay._states(rows, tr.learner.fw, 3, tr.depth_threshold, tr.noise_std, nxt=True)
                assert torch.equal(want, got), (s, h)
        assert torch.equal(one.replay.next_steps[:256], torch.full((256,), 256, dtype=torch.int32, device="cuda"))
    finally:
        for tr in [one] + two:
            tr.close()


def test_gamma_zero_is_the_default_trainer(tmp_path):
    recs, paths = [], []
    for run, kw in enumerate(({}, dict(gamma=0.0))):
        tr = _trainer(64, seed=2, updates_per_step=1, **kw)
        try:
            assert tr.gamma == 0.0 and not tr.replay.next_obs
            assert tr.replay.next_rgb is None and tr.replay.next_depth is None and tr.replay.next_steps is None
            tr.env.reset()
            recs.append([tr.step() for _ in range(3)])
            assert tr.learner.target is None
            os.makedirs(str(tmp_path / f"run{run}"))
            p = str(tmp_path / f"run{run}" / "ck.pt")
            tr.save(p)
            paths.append(p)
        finally:
            tr.close()
    assert recs[0] == recs[1] and recs[0][-1]["updates"] == 1
    assert open(paths[0], "rb").read() == open(paths[1], "rb").read()


def test_cli_trains_with_gamma(tmp_path):
    out = str(tmp_path / "w.pt")
    r = subprocess.run([sys.executable, "-m", "mujoco_rl_ur5_b200.batched_train", "--envs", "64", "--episodes", "1", "--steps-per-episode", "2",
                        "--updates-per-step", "3", "--gamma", "0.9", "--target-update", "2", "--prioritized", "--out", out], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    recs = [json.loads(ln) for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(recs) == 2 and all(rec["updates"] == 3 for rec in recs) and all(np.isfinite(rec["mean_loss"]) for rec in recs)
    assert torch.load(out, map_location="cpu", weights_only=False)["optimizer_state_dict"]["state"][0]["step"] == 6
