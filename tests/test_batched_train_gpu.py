"""The online trainer on the GPU: gq_sample_actions and gq_obs_to_state_keyed against the numpy mirror of tests/test_batched_train.py
and against the existing kernels they must agree with (ge_pixel_2_world, gq_obs_to_state_train), the observation replay, sharding
invariance, determinism, checkpoints and the CLI."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_batched_train import keyed_jitter, sample_actions_mirror

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def qf():
    from mujoco_rl_ur5_b200.qnet import QNetForward, make_torch_qnet

    torch.manual_seed(0)
    return QNetForward(make_torch_qnet(6).state_dict(), 0, max_batch=8)


def _camera(A, cam):
    return (float(np.asarray(A["cam_fovy"]).ravel()[cam]), np.asarray(A["cam_pos0"], dtype=np.float64).reshape(-1, 3)[cam],
            np.asarray(A["cam_mat0"], dtype=np.float64).reshape(-1, 9)[cam])


def _check_engine_z(eng, cam, depth, cand, acc, z_min):
    """every candidate's accept decision of the mirror = the engine's pixel_2_world z test"""
    B, H, W = depth.shape
    for k in range(cand.shape[1]):
        a1 = torch.from_numpy(cand[:, k] % (H * W))
        x, y = (a1 % W).to(torch.int32), (a1 // W).to(torch.int32)
        d = depth[torch.arange(B), y.long(), x.long()].contiguous()
        z = eng.pixel_2_world(x.cuda(), y.cuda(), d.cuda(), cam, W, H)[:, 2].cpu().numpy()
        assert np.array_equal(z >= z_min, acc[:, k]), k


def test_sample_actions_equal_the_mirror_and_the_engine_z_test(qf, scene_a):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    blob, A, _ = scene_a
    B, H, W, R = 4096, 200, 200, 6
    cam = int(np.asarray(A["cam_top_down"]).ravel()[0])
    camera = _camera(A, cam)
    g = torch.Generator().manual_seed(3)
    depth = (1.0 + 0.2 * torch.rand((B, H, W), generator=g)).to(torch.float32)  # z = 2 - depth: about half the pixels on the table
    depth[:, :100] = 1.12 + 0.001 * torch.rand((B, 100, W), generator=g)            # top half just below the table height
    depth[77] = 1.5                                                                  # an image without a table pixel
    # few table pixels (5 %): most envs accept in a later round of 32 candidates than the first
    sparse = torch.where(torch.rand((B, H, W), generator=g) < 0.05, torch.tensor(1.05), 1.12 + 0.001 * torch.rand((B, H, W), generator=g)).to(torch.float32)
    greedy = torch.randint(0, H * W * R, (B,), generator=g, dtype=torch.int32)
    env = 1000 + 3 * np.arange(B, dtype=np.int64) + (2 ** 33) * (np.arange(B) % 2)
    seed, step, z_min = 77, 12345, 0.91 - 0.01
    eng = BatchedEngine(blob, B, 0)
    try:
        for name, dep in (("dense", depth), ("sparse", sparse)):
            dd = dep.cuda()
            for max_draws in (256, 1):
                for eps in (0.0, 0.3, 1.0):
                    act, rnd, exh = qf.sample_actions(dd, greedy.cuda(), torch.full((B,), eps, dtype=torch.float64), torch.from_numpy(env), step, seed,
                                                      camera, z_min, R, max_draws)
                    w_act, w_rnd, w_exh, cand, acc = sample_actions_mirror(dep.numpy(), greedy.numpy(), eps, env, step, seed, camera, z_min, R, max_draws)
                    where = (name, max_draws, eps)
                    assert np.array_equal(rnd.cpu().numpy(), w_rnd) and np.array_equal(exh.cpu().numpy(), w_exh), where
                    assert np.array_equal(act.cpu().numpy(), w_act), (where, np.argwhere(act.cpu().numpy() != w_act)[:5])
                    if eps == 0.0:
                        assert not w_rnd.any()
                    if eps == 0.3:
                        assert 0.25 < w_rnd.mean() < 0.35
                    if eps == 1.0 and max_draws == 256:
                        assert w_rnd.all()
                        first = np.where(acc.any(1), acc.argmax(1), -1)
                        if name == "dense":
                            assert w_exh[77] and w_exh.sum() == 1
                        else:  # accepted in rounds 2 .. 8 of the warp's 32-candidate rounds
                            assert (first >= 32).sum() > 300 and (first >= 64).sum() > 100 and (first >= 128).sum() > 5, np.bincount(first // 32 + 1)
                        _check_engine_z(eng, cam, dep, cand, acc, z_min)
    finally:
        eng.close()


def test_keyed_transform_equals_the_explicit_training_transform(qf):
    S, B = 9, 12
    g = torch.Generator().manual_seed(1)
    rgb = torch.randint(0, 256, (S, 200, 200, 3), generator=g, dtype=torch.uint8).cuda()
    depth = (0.9 + 0.3 * torch.rand((S, 200, 200), generator=g)).cuda()
    slot = torch.tensor([4, 0, 8, 8, 1, 2, 3, 5, 6, 7, 4, 0])
    env = torch.tensor([3, 9, 4096, 17, 2 ** 33 + 5, 0, 11, 12, 13, 14, 15, 16])
    steps = torch.tensor([5] * 6 + [2 ** 32 - 1] * 6)
    state, fac, order = qf.obs_to_state_keyed(rgb, depth, env, steps, 77, slot=slot, return_draws=True)
    w_fac, w_ord = keyed_jitter(77, env.numpy(), steps.numpy())
    assert np.array_equal(fac.cpu().numpy(), w_fac) and np.array_equal(order.cpu().numpy(), w_ord)
    for rows, st in ((slice(0, 6), 5), (slice(6, 12), 2 ** 32 - 1)):
        s = slot[rows].cuda()
        want = qf.obs_to_state_train({"rgb": rgb[s].contiguous(), "depth": depth[s].contiguous()}, 1.1, 0.001, seed=77, step=st, env_index=env[rows],
                                     jitter=fac[rows].contiguous(), order=order[rows].contiguous())
        assert torch.equal(state[rows], want)


def test_replay_regenerates_the_acting_states(qf):
    from mujoco_rl_ur5_b200.replay_buffer import ObservationReplay

    N, size, seed = 4096, 10000, 5
    g = torch.Generator().manual_seed(2)
    rp = ObservationReplay(size, (200, 200), device="cuda", rng=__import__("random").Random(1))
    env = 4096 + torch.arange(N)
    acting = []
    for t in range(3):
        rgb = torch.randint(0, 256, (N, 200, 200, 3), generator=g, dtype=torch.uint8).cuda()
        depth = (0.9 + 0.3 * torch.rand((N, 200, 200), generator=g)).cuda()
        key = torch.full((N,), 1000 + t * N)
        acting.append([qf.obs_to_state_keyed(rgb[i:i + 512], depth[i:i + 512], env[i:i + 512], key[i:i + 512], seed).cpu() for i in range(0, N, 512)])
        rp.push_batch(rgb, depth, torch.arange(N), torch.zeros(N), env, key)
    assert len(rp) == size and rp.position == (3 * N) % size
    # transition j (0 .. 3N-1) survives iff j >= 3N - size; it lives in slot j % size
    for j0 in range(3 * N - size, 3 * N, 512):
        js = torch.arange(j0, min(j0 + 512, 3 * N))
        slots = js % size
        got = qf.obs_to_state_keyed(rp.rgb, rp.depth, rp.envs[slots.cuda()], rp.steps[slots.cuda()], seed, slot=slots).cpu()
        for r, j in enumerate(js.tolist()):
            t, i = divmod(j, N)
            assert torch.equal(got[r], acting[t][i // 512][i % 512]), j
    state = rp.rng.getstate()
    idx = rp.sample_indices(12)
    rp.rng.setstate(state)
    states, actions, _ = rp.sample(12, qf, seed)  # the same draws, through sample()
    assert torch.equal(actions[:, 0].cpu(), rp.actions[idx].cpu())
    for r, s in enumerate(idx):
        j = max(j for j in range(3 * N - size, 3 * N) if j % size == s)
        t, i = divmod(j, N)
        assert torch.equal(states[r].cpu(), acting[t][i // 512][i % 512])


def _trainer(n, **kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    return BatchedTrainer(n, "A", 0, **kw)


def test_sharded_trainers_act_like_one(qf):
    one = _trainer(256, seed=3, updates_per_step=0)
    two = [_trainer(128, seed=3, updates_per_step=0, env_index_offset=o, n_total=256) for o in (0, 128)]
    try:
        for tr in [one] + two:
            tr.env.reset()
        for t in range(3):
            one.step()
            for tr in two:
                tr.step()
            for k in ("actions", "is_random", "reward"):
                a = one.last_step[k]
                b = np.concatenate([np.asarray(tr.last_step[k]) for tr in two])
                assert np.array_equal(np.asarray(a), b), (t, k)
        assert one.steps_done == two[0].steps_done == two[1].steps_done == 3 * 256
        assert 0 < np.asarray(one.last_step["is_random"]).sum()
        for s in range(3):
            for h, tr in enumerate(two):
                rows = torch.arange(s * 128, (s + 1) * 128)
                want = qf.obs_to_state_keyed(one.replay.rgb, one.replay.depth, one.replay.envs[(rows + s * 128 + h * 128).cuda()],
                                             one.replay.steps[(rows + s * 128 + h * 128).cuda()], 3, slot=rows + s * 128 + h * 128, depth_threshold=one.depth_threshold)
                got = qf.obs_to_state_keyed(tr.replay.rgb, tr.replay.depth, tr.replay.envs[rows.cuda()], tr.replay.steps[rows.cuda()], 3, slot=rows,
                                            depth_threshold=tr.depth_threshold)
                assert torch.equal(want, got), (s, h)
    finally:
        for tr in [one] + two:
            tr.close()


def test_training_is_deterministic_and_acts_on_the_learners_weights(tmp_path):
    from mujoco_rl_ur5_b200.qnet import QNetForward

    paths = []
    for run in range(2):
        tr = _trainer(64, seed=11, updates_per_step=2)
        try:
            tr.train(2, 3)
            assert tr.learner.step_count == 2 * 6
            os.makedirs(str(tmp_path / f"run{run}"))
            p = str(tmp_path / f"run{run}" / "ck.pt")  # same file name: torch.save writes it into the archive
            tr.save(p)
            paths.append(p)
            if run == 0:  # the acting path uses the learner's current weights
                obs = tr.env.current_observation
                states = tr.acting_states(obs, 42)
                fresh = QNetForward(tr.learner.model_state_dict(), 0, max_batch=64)
                q = fresh.forward(states)
                assert torch.equal(tr.learner.fw.forward(states), q)
                act, _ = fresh.greedy(q)
                want = (act[:, 1] * 200 * 200 + act[:, 0]).to(torch.int32)
                assert torch.equal(tr.greedy_indices(states), want)
        finally:
            tr.close()
    a, b = (torch.load(p, map_location="cpu", weights_only=False) for p in paths)
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], dict) and k.endswith("state_dict") and k.startswith("model"):
            assert all(torch.equal(a[k][n], b[k][n]) for n in a[k]), k
        elif k == "optimizer_state_dict":
            for pid, st in a[k]["state"].items():
                assert all(torch.equal(st[n], b[k]["state"][pid][n]) for n in st)
        else:
            assert a[k] == b[k], k
    assert open(paths[0], "rb").read() == open(paths[1], "rb").read()


@pytest.fixture(scope="module")
def trained_checkpoint(tmp_path_factory):
    """a 64-env trainer after 1 episode x 3 steps, 1 update per step: (path of its checkpoint, the dict it saved)"""
    tr = _trainer(64, seed=2, updates_per_step=1)
    try:
        from mujoco_rl_ur5_b200.batched_train import EPS_START

        assert tr.eps_threshold == EPS_START and tr.checkpoint()["epsilon"] == EPS_START  # a fresh agent starts at EPS_START (:182)
        tr.train(1, 3)
        path = str(tmp_path_factory.mktemp("ck") / "weights.pt")
        return path, tr.save(path)
    finally:
        tr.close()


def test_checkpoint_loads_into_torch_and_resumes(trained_checkpoint):
    from mujoco_rl_ur5_b200.batched_train import COUNTERS, epsilon
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet

    path, ck = trained_checkpoint
    assert ck["step"] == 3 * 64 and ck["epsilon"] == epsilon(3 * 64 - 1)
    loaded = torch.load(path, map_location="cpu", weights_only=False)
    make_torch_qnet(6).load_state_dict(loaded["model_state_dict"], strict=True)
    tr2 = _trainer(64, seed=2, updates_per_step=0, load=path)
    try:
        assert tr2.steps_done == 3 * 64 and tr2.eps_threshold == ck["epsilon"] and tr2.learner.step_count == 3
        assert tr2.epsilons()[0] == epsilon(3 * 64)       # the first resumed transition continues the schedule
        assert {k: dict(v) for k, v in tr2.counters().items()} == {k: dict(ck[k]) for k in COUNTERS}
        tr2.env.reset()
        tr2.step()
        ck2 = tr2.checkpoint()
        assert ck2["step"] == 4 * 64
        n_greedy = tr2.last_step["is_random"].size - int(np.asarray(tr2.last_step["is_random"]).sum())
        assert sum(ck2["greedy_rotations"].values()) == sum(ck["greedy_rotations"].values()) + n_greedy
    finally:
        tr2.close()


def test_the_reference_agent_resumes_from_the_checkpoint(trained_checkpoint, tmp_path):
    """the reference's unchanged Grasp_Agent(load_path=...) (Grasping_Agent_multidiscrete.py:111-179) on the GPU facade.  Its
    torch.load(load_path) predates torch's weights_only=True default (torch >= 2.6), which refuses the checkpoint's defaultdict
    counters - the reference's own checkpoints hold them too - so the child loads with weights_only=False."""
    import shutil

    from tests.test_reference_scripts_gpu import COMPAT, _ref_dir

    ref = _ref_dir()
    if ref is None:
        pytest.skip("reference scripts not staged: run tools/stage_reference.py where the reference exists")
    path, ck = trained_checkpoint
    shutil.copy(path, str(tmp_path / "weights.pt"))
    code = ("import json, torch\n"
            "_load = torch.load\n"
            "torch.load = lambda f, *a, **k: _load(f, *a, **{**k, 'weights_only': False})\n"
            "import Grasping_Agent_multidiscrete as G\n"
            "a = G.Grasp_Agent(load_path='weights.pt')\n"
            "st = a.optimizer.state[next(iter(a.policy_net.parameters()))]\n"
            "w = a.policy_net.state_dict()['0.C1.weight'].double().sum().item()\n"
            "print('LOADED ' + json.dumps([a.steps_done, a.eps_threshold, dict(a.greedy_rotations), float(st['step']), w]))\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, COMPAT, ref]))
    env.pop("GRASP_SCENE", None)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    steps, eps, greedy, adam_step, w = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("LOADED "))[7:])
    assert steps == ck["step"] and eps == ck["epsilon"] and greedy == dict(ck["greedy_rotations"]) and adam_step == 3
    assert w == ck["model_state_dict"]["0.C1.weight"].double().sum().item()


def test_cli_trains_and_writes_a_checkpoint(tmp_path):
    out = str(tmp_path / "w.pt")
    r = subprocess.run([sys.executable, "-m", "mujoco_rl_ur5_b200.batched_train", "--envs", "256", "--episodes", "1", "--steps-per-episode", "3",
                        "--updates-per-step", "4", "--out", out], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    recs = [json.loads(ln) for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(recs) == 3 and all(rec["updates"] == 4 for rec in recs)
    assert all(np.isfinite(rec["mean_loss"]) for rec in recs)
    assert os.path.exists(out)
