"""Standardised observations on the GPU: gq_obs_to_state_standard against the reference's own transform_observation(normalize=False)
(bit for bit, tests/golden/standardize.npz) and the noise mirror, gq_obs_channel_stats against the reference's normalize.py and numpy,
the normalize CLI, and the online trainer and greedy agent on standardised states."""
import ctypes as C
import subprocess
import sys
from decimal import Decimal, getcontext

import numpy as np
import pytest
import torch

from tests.test_obs_transform import philox_normal
from tests.test_standardize import STATE_CASES, _golden, _typed, normalize_observations, synthetic_obs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qf():
    from mujoco_rl_ur5_b200.qnet import QNetForward, make_torch_qnet

    torch.manual_seed(0)
    return QNetForward(make_torch_qnet(6).state_dict(), 0, max_batch=8)


@pytest.fixture(scope="module")
def shipped():
    meta, _ = _golden()
    return _typed(meta["shipped"])


def _dev(rgb, depth):
    return {"rgb": torch.from_numpy(np.ascontiguousarray(rgb)).cuda(), "depth": torch.from_numpy(np.ascontiguousarray(depth)).cuda()}


def _bits(x):
    return x.detach().cpu().contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------ the transform
def test_noise_free_state_equals_the_reference_bit_for_bit(qf):
    meta, z = _golden()
    used = _typed(meta["used"])
    for seed, H, W in STATE_CASES:
        rgb, depth = synthetic_obs(seed, H, W)
        s, nhwc = qf.obs_to_state_standard(_dev(rgb[None], depth[None]), used, noise_std=0.0, nhwc_bf16=True)
        ref = torch.from_numpy(z[f"state_{seed}"])
        assert torch.equal(_bits(s), ref.view(torch.int32)), (seed, H, W)
        assert torch.equal(nhwc.cpu().view(torch.int16), s.permute(0, 2, 3, 1).to(torch.bfloat16).cpu().view(torch.int16)), (seed, H, W)


def test_noise_rows_slots_and_per_row_steps(qf, shipped):
    B, H, W, seed, step = 8, 200, 200, 77, 12
    g = torch.Generator().manual_seed(5)
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).cuda()
    depth = (0.9 + 0.4 * torch.rand((B, H, W), generator=g)).cuda()
    obs = {"rgb": rgb, "depth": depth}
    env = torch.tensor([3, 1000, 5, 2 ** 33 + 7, 0, 64, 4095, 9])
    clean = qf.obs_to_state_standard(obs, shipped, noise_std=0.0)
    noisy, nhwc = qf.obs_to_state_standard(obs, shipped, noise_std=0.001, seed=seed, step=step, env_index=env, nhwc_bf16=True)
    assert torch.equal(nhwc.cpu().view(torch.int16), noisy.permute(0, 2, 3, 1).to(torch.bfloat16).cpu().view(torch.int16))
    assert torch.equal(_bits(noisy[:, :3]), _bits(clean[:, :3]))  # no noise, no jitter on the colour channels
    diff = (noisy[:, 3] - clean[:, 3]).cpu().numpy().astype(np.float64)
    for b in range(B):
        want = 0.001 * philox_normal(seed, int(env[b]), step, np.arange(H * W)).reshape(H, W)
        assert np.abs(diff[b] - want).max() < 1e-6, b
    for b in range(B):  # a row alone under its global env id is the same row of the batch
        one = qf.obs_to_state_standard({"rgb": rgb[b:b + 1], "depth": depth[b:b + 1]}, shipped, seed=seed, step=step, env_index=env[b:b + 1])
        assert torch.equal(_bits(one[0]), _bits(noisy[b])), b
    sl = torch.tensor([6, 1, 1, 3])
    via_slot = qf.obs_to_state_standard(obs, shipped, seed=seed, step=torch.full((4,), step), env_index=env[sl], slot=sl)
    assert torch.equal(_bits(via_slot), _bits(noisy[sl.cuda()]))
    per_row = qf.obs_to_state_standard(obs, shipped, seed=seed, step=torch.tensor([step, step + 1] * 4), env_index=env)
    assert torch.equal(_bits(per_row[0::2]), _bits(noisy[0::2])) and not torch.equal(per_row[1::2], noisy[1::2])


def test_bad_arguments_write_nothing(qf, shipped):
    L = qf.L
    H = W = 16
    rgb = torch.zeros((2, H, W, 3), dtype=torch.uint8, device="cuda")
    depth = torch.ones((2, H, W), dtype=torch.float32, device="cuda")
    out = torch.full((2, 4, H, W), 7.0, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for bad_std, B in ((0.0, 2), (-1.0, 2), (1.0, 0)):
        ms = np.array([1, 2, 3, 1.5, 1, 1, bad_std, 0.5], dtype=np.float32)
        r = L.gq_obs_to_state_standard(C.c_void_p(rgb.data_ptr()), C.c_void_p(depth.data_ptr()), None, None, None, 0, ms.ctypes.data_as(C.c_void_p), 1.1, 0.001,
                                       0, C.c_void_p(out.data_ptr()), None, B, H * W, stream)
        assert r == -1, (bad_std, B)
        assert b"gq_obs_to_state_standard" in L.gq_last_error()
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    with pytest.raises(ValueError, match="> 0"):
        qf.obs_to_state_standard({"rgb": rgb, "depth": depth}, [1, 2, 3, 1.5, 1, 0, 1, 0.5])


# ------------------------------------------------------------------------------------------------ the statistics
def _exact_std(count):
    """population std of a u8 channel from its histogram, as an exact rational -> Decimal (60 digits)"""
    k = np.arange(256, dtype=object)
    n, s, q = int(count.sum()), int((k * count.astype(object)).sum()), int((k * k * count.astype(object)).sum())
    getcontext().prec = 60
    return (Decimal(n * q - s * s) / Decimal(n * n)).sqrt()


def _check_stats(got, rgb, depth, f32_ref=None):
    """got: channel_statistics of (rgb [n,H,W,3] u8, depth [n,H,W] f32) on the host; f32_ref: numpy's float32 depth values when known"""
    assert [type(v).__name__ for v in got] == ["float64"] * 3 + ["float32"] + ["float64"] * 3 + ["float32"]
    for c in range(3):
        ch = np.ascontiguousarray(rgb[..., c]).reshape(-1)
        assert got[c] == np.mean(ch), c                                                   # bit for bit
        exact = _exact_std(np.bincount(ch, minlength=256))
        assert abs(Decimal(float(got[4 + c])) - exact) <= 2 * Decimal(float(np.spacing(np.float64(float(exact))))), c
        assert abs(float(got[4 + c]) / np.std(ch) - 1) < 1e-12, c
    d = depth.reshape(-1)
    np32 = (np.mean(d), np.std(d)) if f32_ref is None else f32_ref
    d64 = d.astype(np.float64)
    np64 = (np.mean(d64), np.std(d64))
    for k, (mine, v32, v64) in enumerate(zip((got[3], got[7]), np32, np64)):
        assert abs(float(mine) / float(v32) - 1) < 1e-6, k
        assert abs(int(np.float32(mine).view(np.int32)) - int(np.float32(v64).view(np.int32))) <= 1, k


def test_channel_statistics_match_the_reference_normalize_py():
    from mujoco_rl_ur5_b200.obs_stats import channel_statistics

    meta, _ = _golden()
    nm = meta["normalize"]
    ref = _typed(nm)
    rgb, depth = normalize_observations(nm["seed"], nm["n"], nm["H"], nm["W"])
    got = channel_statistics(*_dev(rgb, depth).values())
    assert [float(v).hex() for v in got[:3]] == nm["values"][:3]                           # the means bit for bit
    for c in range(3):
        assert abs(float(got[4 + c]) / float(ref[4 + c]) - 1) < 1e-12
    _check_stats(got, rgb, depth, f32_ref=(ref[3], ref[7]))


def test_channel_statistics_of_4096_rendered_observations_are_numpys_and_deterministic():
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv
    from mujoco_rl_ur5_b200.obs_stats import channel_statistics

    env = BatchedGraspEnv(4096, "A", 0)
    try:
        obs = env.reset()
        a = channel_statistics(obs["rgb"], obs["depth"])
        b = channel_statistics(obs["rgb"], obs["depth"])
        assert [float(v).hex() for v in a] == [float(v).hex() for v in b]
        _check_stats(a, obs["rgb"].cpu().numpy(), obs["depth"].cpu().numpy())
    finally:
        env.close()


def test_normalize_cli_scene_a(tmp_path, shipped):
    from mujoco_rl_ur5_b200.obs_stats import load_mean_and_std

    out = tmp_path / "mean_and_std"
    r = subprocess.run([sys.executable, "-m", "mujoco_rl_ur5_b200.normalize", "--scene", "A", "--envs", "100", "--out", str(out)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "Calculated mean value of" in r.stdout and f"Wrote values to file {out}" in r.stdout
    v = load_mean_and_std(str(out))
    assert abs(float(v[3]) - float(shipped[3])) < 2e-3 and abs(float(v[7]) - float(shipped[7])) < 2e-3, v
    assert all(abs(float(v[c]) / float(shipped[c]) - 1) < 0.15 for c in range(3)), v


# ------------------------------------------------------------------------------------------------ trainer and agent
def _trainer(n, **kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    return BatchedTrainer(n, "A", 0, **kw)


def _record_acting(tr):
    """wraps tr.acting_states: -> list of (obs clone, step key, states clone) per batched step"""
    rec = []
    inner = tr.acting_states

    def wrapped(obs, step):
        s = inner(obs, step)
        rec.append(({k: v.clone() for k, v in obs.items()}, step, s.clone()))
        return s

    tr.acting_states = wrapped
    return rec


def test_trainer_acts_and_replays_on_standardised_states(qf, shipped):
    tr = _trainer(16, seed=4, updates_per_step=0, standardize=shipped, gamma=0.5, target_update=2)
    try:
        rec = _record_acting(tr)
        tr.env.reset()
        for _ in range(3):
            tr.step()
        for t, (obs, key, states) in enumerate(rec):
            want = qf.obs_to_state_standard(obs, shipped, tr.depth_threshold, 0.001, 4, key, tr.genv)
            assert torch.equal(_bits(states), _bits(want)), t
            mm = qf.obs_to_state_keyed(obs["rgb"], obs["depth"], tr.genv, torch.full((16,), key), 4, depth_threshold=tr.depth_threshold)
            assert not torch.equal(states, mm)
        state = tr.replay.rng.getstate()
        idx = tr.replay.sample_indices(24)
        tr.replay.rng.setstate(state)
        s, a, r, s2 = tr.replay.sample(24, tr.learner.fw, tr.seed, tr.depth_threshold, tr.noise_std)
        for row, slot in enumerate(idx):
            t, e = divmod(slot, 16)
            assert torch.equal(_bits(s[row]), _bits(rec[t][2][e])), slot
            if t + 1 < len(rec):  # the next state is the state the env acted on at the next step
                assert torch.equal(_bits(s2[row]), _bits(rec[t + 1][2][e])), slot
    finally:
        tr.close()


def test_sharded_standardised_trainers_act_like_one(shipped):
    one = _trainer(256, seed=3, updates_per_step=0, standardize=shipped)
    two = [_trainer(128, seed=3, updates_per_step=0, env_index_offset=o, n_total=256, standardize=shipped) for o in (0, 128)]
    try:
        for tr in [one] + two:
            tr.env.reset()
        for t in range(3):
            one.step()
            for tr in two:
                tr.step()
            for k in ("actions", "is_random", "reward"):
                assert np.array_equal(np.asarray(one.last_step[k]), np.concatenate([np.asarray(tr.last_step[k]) for tr in two])), (t, k)
        fw = one.learner.fw
        for h, tr in enumerate(two):
            rows = torch.arange(2 * 128, 3 * 128)
            want = one.replay._states((rows + 2 * 128 + h * 128).cuda(), fw, 3, one.depth_threshold, one.noise_std)
            got = tr.replay._states(rows.cuda(), fw, 3, tr.depth_threshold, tr.noise_std)
            assert torch.equal(_bits(want), _bits(got)), h
    finally:
        for tr in [one] + two:
            tr.close()


def test_checkpoint_keeps_the_statistics_and_resumes(tmp_path, shipped):
    path = tmp_path / "ck.pt"
    tr = _trainer(16, seed=2, updates_per_step=1, batch_size=4, standardize=shipped)
    try:
        tr.env.reset()
        for _ in range(2):
            rec = tr.step()
        assert rec["updates"] == 1
        tr.save(str(path))
    finally:
        tr.close()
    ck = torch.load(str(path), map_location="cpu", weights_only=False)
    assert ck["mean_and_std"] == [float(v) for v in shipped] and all(type(v) is float for v in ck["mean_and_std"])
    other = [float(v) for v in shipped]
    other[4] += 1.0
    with pytest.raises(ValueError, match="mean_and_std"):
        _trainer(16, load=str(path), standardize=other)
    tr2 = _trainer(16, seed=2, updates_per_step=1, batch_size=4, load=str(path))
    try:
        assert [float(v) for v in tr2.standardize] == ck["mean_and_std"] and tr2.replay.standardize is not None
        rec = _record_acting(tr2)
        tr2.env.reset()
        tr2.step()
        obs, key, states = rec[0]
        assert key == 2 * 16
        want = tr2.learner.fw.obs_to_state_standard(obs, shipped, tr2.depth_threshold, 0.001, 2, key, tr2.genv)
        assert torch.equal(_bits(states), _bits(want))
        assert tr2.checkpoint()["mean_and_std"] == ck["mean_and_std"]
    finally:
        tr2.close()


def test_greedy_agent_acts_on_standardised_states(shipped):
    from mujoco_rl_ur5_b200.batched_agent import BatchedGreedyAgent
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv

    env = BatchedGraspEnv(8, "A", 0, env_index_offset=40)
    try:
        obs = env.reset()
        ag = BatchedGreedyAgent(env, seed=1, standardize=shipped)
        genv = 40 + torch.arange(8)
        for k in range(2):
            want = ag.qnet.obs_to_state_standard(obs, shipped, ag.depth_threshold, 0.001, 1, k, genv)
            assert torch.equal(_bits(ag.states(obs)), _bits(want)), k
        act, val = ag.greedy(obs)
        assert act.shape == (8, 2) and act.dtype == torch.int32 and bool(torch.isfinite(val).all())
        assert BatchedGreedyAgent(env, seed=1).standardize is None
    finally:
        env.close()
