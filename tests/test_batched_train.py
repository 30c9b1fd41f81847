"""The online trainer's host side (mujoco_rl_ur5_b200/batched_train.py, ObservationReplay) and a numpy mirror of the keyed draws of
csrc/qnet.cu (the table above keyed_words): counter (c0, env_lo, env_hi, step), key (seed_lo, seed_hi) of Philox4x32-10; the depth
noise uses c0 = pixel, the draws c0 = 0x80000000 + j.  tests/test_batched_train_gpu.py compares the kernels with this mirror."""
import itertools
import json
import math
import random
import types

import numpy as np
import torch

from mujoco_rl_ur5_b200.replay_buffer import DeviceReplayBuffer, ObservationReplay
from tests.test_obs_transform import philox_normal
from tests.test_replay_buffer import GOLD, REPLAY_CASES, _drive

KEYED_C0 = 0x80000000
PERMS = list(itertools.permutations(range(4)))  # lexicographic
REFERENCE_KEYS = {"step", "model_state_dict", "optimizer_state_dict", "epsilon", "greedy_rotations", "greedy_rotations_successes",
                  "random_rotations_successes"}


# ------------------------------------------------------------------------------------------------ numpy mirror
def philox_words(seed, c0, env, step):
    """Philox4x32-10 words [4, n] for counters (c0, env_lo, env_hi, step) (arrays broadcast to one length) under key (seed_lo, seed_hi)"""
    c0, env, step = np.broadcast_arrays(np.asarray(c0, dtype=np.uint64), np.asarray(env, dtype=np.uint64), np.asarray(step, dtype=np.uint64))
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
    x0 = (c0 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    x1 = (env & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    x2 = (env >> np.uint64(32)).astype(np.uint32)
    x3 = (step & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    k0, k1 = np.uint32(seed & 0xFFFFFFFF), np.uint32((seed >> 32) & 0xFFFFFFFF)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * x0.astype(np.uint64)
            p1 = M1 * x2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
            x0, x1, x2, x3 = hi1 ^ x1 ^ k0, lo1, hi0 ^ x3 ^ k1, lo0
            k0, k1 = np.uint32(k0 + W0), np.uint32(k1 + W1)
    return np.stack([x0, x1, x2, x3])


def uniform(w):
    return (((w >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def keyed_jitter(seed, env, step):
    """-> (factors [n,4] f32: brightness, contrast, saturation, hue; order [n,4] int32) of the keyed draws j = 0, 1"""
    w = philox_words(seed, KEYED_C0 + 0, env, step)
    v = philox_words(seed, KEYED_C0 + 1, env, step)
    h = np.float32(0.5)
    fac = np.stack([h + uniform(w[1]), h + uniform(w[2]), h + uniform(w[3]), uniform(v[0]) - h], axis=1).astype(np.float32)
    perm = ((v[1].astype(np.uint64) * np.uint64(24)) >> np.uint64(32)).astype(np.int64)
    return fac, np.array([PERMS[p] for p in perm], dtype=np.int32).reshape(-1, 4)


def keyed_epsilon_uniform(seed, env, step):
    return uniform(philox_words(seed, KEYED_C0, env, step)[0])


def keyed_candidates(seed, env, step, k, n_actions):
    """flat candidate actions [n, len(k)] of draws j = 2 + k"""
    env = np.asarray(env, dtype=np.uint64)[:, None]
    w = philox_words(seed, KEYED_C0 + 2 + np.asarray(k, dtype=np.uint64)[None, :], env, step)[0]
    return ((w.astype(np.uint64) * np.uint64(n_actions)) >> np.uint64(32)).astype(np.int64)


def world_z(camera, W, H, px, py, depth):
    """z of pixel_2_world (MujocoController.py:783-806) in float64, the engine's expression order"""
    fovy, pos, mat = camera
    f = 0.5 * H / math.tan(fovy * 3.14159265358979323846 / 360.0)
    d = -depth.astype(np.float64)
    t = [(px * d - 0.5 * W * d) / f + pos[0], (py * d - 0.5 * H * d) / f + pos[1], d + pos[2]]
    return mat[2] * t[0] + mat[5] * t[1] + mat[8] * t[2]


def sample_actions_mirror(depth, greedy_idx, eps, env, step, seed, camera, z_min, R, max_draws):
    """sequential epsilon_greedy per env -> (action [B,2], is_random [B], exhausted [B], candidates [B,max_draws], accepted [B,max_draws])"""
    B, H, W = depth.shape
    HW = H * W
    u = keyed_epsilon_uniform(seed, env, step)
    rnd = ~(u.astype(np.float64) > eps)
    cand = keyed_candidates(seed, env, step, np.arange(max_draws), HW * R)
    a1 = cand % HW
    x, y = a1 % W, a1 // W
    acc = world_z(camera, W, H, x, y, depth[np.arange(B)[:, None], y, x]) >= z_min
    first = np.where(acc.any(1), acc.argmax(1), max_draws - 1)
    flat = np.where(rnd, cand[np.arange(B), first], greedy_idx)
    exhausted = rnd & ~acc.any(1)
    return np.stack([flat % HW, flat // HW], 1), rnd, exhausted, cand, acc


# ------------------------------------------------------------------------------------------------ tests
def test_mirror_words_reproduce_the_depth_noise_generator():
    pix = np.arange(5000)
    for seed, env, step in ((77, 4096, 12), (2 ** 40 + 3, 2 ** 33 + 5, 2 ** 32 - 1), (0, 0, 0)):
        w = philox_words(seed, pix, env, step)
        u1, u2 = uniform(w[0]), uniform(w[1])
        z = np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(2.0 * np.pi * u2.astype(np.float64))
        assert np.array_equal(z, philox_normal(seed, env, step, pix))


def test_keyed_orders_are_uniform_and_factors_in_range():
    n = 96000
    env = np.arange(n) % 4096 + 1000
    step = np.arange(n) // 4096
    fac, order = keyed_jitter(12345, env, step)
    counts = {}
    for o in map(tuple, order):
        counts[o] = counts.get(o, 0) + 1
    assert set(counts) == set(PERMS)
    mu, sd = n / 24, math.sqrt(n * (1 / 24) * (23 / 24))
    assert all(abs(c - mu) < 5 * sd for c in counts.values()), counts
    assert (fac[:, :3] > 0.5).all() and (fac[:, :3] < 1.5).all() and (fac[:, 3] > -0.5).all() and (fac[:, 3] < 0.5).all()
    for k in range(4):  # each factor spreads over its whole range
        lo, hi = (-0.5, 0.5) if k == 3 else (0.5, 1.5)
        assert np.histogram(fac[:, k], bins=10, range=(lo, hi))[0].min() > 0.09 * n
    # the streams of j = 0 (epsilon, factors), j = 1 and the candidates are not the same numbers
    u = keyed_epsilon_uniform(12345, env[:1000], step[:1000])
    assert abs(np.corrcoef(u, fac[:1000, 0])[0, 1]) < 0.1 and abs(u.mean() - 0.5) < 0.03


def test_sequential_mirror_takes_the_first_accepted_candidate():
    rng = np.random.RandomState(0)
    depth = (1.0 + 0.2 * rng.rand(5, 20, 20)).astype(np.float32)
    depth[4] = 1.5  # no pixel on the table
    camera = (45.0, np.array([0.0, -0.6, 2.0]), np.eye(3).ravel())
    env = np.arange(5) + 7
    act, rnd, exh, cand, acc = sample_actions_mirror(depth, np.arange(5), np.ones(5), env, 3, 9, camera, 0.90, 6, 64)
    assert rnd.all() and exh.tolist() == [False] * 4 + [True]
    for b in range(5):
        k = next((k for k in range(64) if acc[b, k]), 63)
        assert act[b].tolist() == [cand[b, k] % 400, cand[b, k] // 400]
    act0, rnd0, _, _, _ = sample_actions_mirror(depth, np.arange(5), np.zeros(5), env, 3, 9, camera, 0.90, 6, 64)
    assert not rnd0.any() and act0[:, 0].tolist() == list(range(5))


def test_epsilon_follows_the_reference_schedule():
    from mujoco_rl_ur5_b200.batched_train import EPS_DECAY, EPS_END, EPS_START, BatchedTrainer, epsilon

    for n in (0, 1, 12, 4095, 8000, 123457, 10 ** 7):
        assert epsilon(n) == EPS_END + (EPS_START - EPS_END) * math.exp(-1.0 * n / EPS_DECAY)
    assert epsilon(0) == 1.0
    # transition n = steps_done + t * N_total + g: env g of this rank, steps_done already advanced by t * N_total
    tr = types.SimpleNamespace(steps_done=3 * 256 + 40, env_offset=128, n_envs=128, eps_start=EPS_START, eps_end=EPS_END, eps_decay=EPS_DECAY)
    eps = BatchedTrainer.epsilons(tr)
    assert eps == [epsilon(3 * 256 + 40 + 128 + i) for i in range(128)]


def _obs_rows(n, k0):
    return (torch.full((n, 2, 2, 3), 0, dtype=torch.uint8), torch.arange(k0, k0 + n, dtype=torch.float32)[:, None, None].expand(n, 2, 2).contiguous())


def test_observation_replay_samples_like_the_device_replay_buffer():
    a = DeviceReplayBuffer(8, state_shape=(1,), device="cpu", rng=random.Random(20))
    b = ObservationReplay(8, (2, 2), device="cpu", rng=random.Random(20))
    k = 0
    for n in (3, 4, 5, 11, 2, 8, 17):  # wrap-around and pushes larger than the ring
        a.push_batch(torch.arange(k, k + n, dtype=torch.float32)[:, None], torch.arange(k, k + n), torch.ones(n))
        rgb, depth = _obs_rows(n, k)
        b.push_batch(rgb, depth, torch.arange(k, k + n), torch.ones(n), 1000 + torch.arange(k, k + n), torch.full((n,), 7))
        k += n
        assert (a.position, len(a)) == (b.position, len(b))
        assert torch.equal(a.actions, b.actions) and torch.equal(a.states[:, 0], b.depth[:, 0, 0])
        assert torch.equal(b.envs[:len(b)], 1000 + b.actions[:len(b)])
        ia, ib = a.sample_indices(4), b.sample_indices(4)
        assert ia == ib


def test_observation_replay_reproduces_the_reference_class():
    """the replay_buffer cases of tests/golden/reference_io.json, written by the reference's Modules.ReplayBuffer"""
    g = json.load(open(GOLD))["replay_buffer"]
    assert [(c["size"], c["B"], c["pushes"]) for c in g] == list(REPLAY_CASES)
    for c in g:
        b = ObservationReplay(c["size"], (2, 2), device="cpu")  # rng=None: the global `random` module, re-seeded with 20

        def push(k):
            rgb, depth = _obs_rows(1, k)
            b.push_batch(rgb, depth, torch.tensor([k * 3]), torch.tensor([k % 2]), torch.tensor([k]), torch.tensor([0]))

        got = _drive(push, lambda B_: [int(v) for v in b.actions[b.sample_indices(B_)] // 3], lambda: len(b), c["pushes"], c["size"], c["B"])
        assert got == c["samples"]


def test_checkpoint_has_the_reference_keys_and_a_torch_adam_state():
    from collections import defaultdict

    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer
    from mujoco_rl_ur5_b200.qnet import make_torch_qnet
    from mujoco_rl_ur5_b200.qnet_learn import adam_to_torch

    torch.manual_seed(0)
    net = make_torch_qnet(6)
    params = dict(net.named_parameters())
    m = {k: torch.full_like(p, 0.01) for k, p in params.items()}
    v = {k: torch.full_like(p, 0.02) for k, p in params.items()}
    learner = types.SimpleNamespace(checkpoint=lambda: {"model_state_dict": net.state_dict(),
                                                        "optimizer_state_dict": adam_to_torch(params, m, v, 5, 1e-3, (0.9, 0.999), 1e-8, 2e-5)})
    tr = types.SimpleNamespace(learner=learner, steps_done=777, eps_threshold=0.5,
                               counters=lambda: {k: defaultdict(int, {"2": 3}) for k in ("greedy_rotations", "greedy_rotations_successes",
                                                                                          "random_rotations_successes")})
    ck = BatchedTrainer.checkpoint(tr)
    assert set(ck) == REFERENCE_KEYS and ck["step"] == 777 and ck["epsilon"] == 0.5 and ck["greedy_rotations"]["2"] == 3
    net2 = make_torch_qnet(6)
    net2.load_state_dict(ck["model_state_dict"], strict=True)
    opt = torch.optim.Adam(net2.parameters(), lr=0.5, weight_decay=0.00002)
    opt.load_state_dict(ck["optimizer_state_dict"])
    assert opt.param_groups[0]["lr"] == 1e-3
    st = opt.state[next(iter(net2.parameters()))]
    assert float(st["step"]) == 5 and torch.all(st["exp_avg"] == 0.01)
