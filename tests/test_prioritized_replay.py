"""Prioritized experience replay (csrc/qnet_replay.cuh, replay_buffer.PrioritizedObservationReplay, BatchedTrainer(prioritized=...)):
a numpy mirror of the sum-tree, the stratified descent, the keyed draws and the importance weights, checked here on hand-built trees;
tests/test_prioritized_replay_gpu.py compares the kernels with it."""
import types

import numpy as np
import pytest

from tests.test_batched_train import philox_words

PER_C0 = 0xC0000000


# ------------------------------------------------------------------------------------------------ numpy mirror
def capacity(size):
    """the smallest power of two >= size"""
    return 1 << max(0, (int(size) - 1).bit_length())


class TreeMirror:
    """the device sum-tree in float64: leaf cap + i = priority of slot i, node k = tree[2k] + tree[2k+1], root tree[1]"""

    def __init__(self, size):
        self.cap = capacity(size)
        self.tree = np.zeros(2 * self.cap)
        self.pmax = 1.0

    def _fix(self, nodes):
        nodes = np.unique(np.asarray(nodes, dtype=np.int64))
        while nodes.size and nodes[0] >= 1:
            nodes = np.unique(nodes >> 1)
            nodes = nodes[nodes >= 1]
            self.tree[nodes] = self.tree[2 * nodes] + self.tree[2 * nodes + 1]

    def push(self, slots):
        leaves = self.cap + np.asarray(slots, dtype=np.int64)
        self.tree[leaves] = self.pmax
        self._fix(leaves)

    def update(self, idx, qsel, reward, alpha, eps):
        p = (np.abs(np.asarray(reward, np.float32).astype(np.float64) - np.asarray(qsel, np.float32).astype(np.float64)) + eps) ** alpha
        leaves = self.cap + np.asarray(idx, dtype=np.int64)
        for leaf, v in zip(leaves, p):  # batch order: the later entry of a duplicate wins
            self.tree[leaf] = v
        self._fix(leaves)
        self.pmax = max(self.pmax, float(p.max()))
        return p

    def leaves(self):
        return self.tree[self.cap:]


def stratum_uniforms(seed, B, update, rank):
    """U_j = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 of the keyed draws (0xC0000000 + j, update_lo, update_hi, rank) under seed"""
    w = philox_words(seed, PER_C0 + np.arange(B, dtype=np.uint64), np.uint64(update), np.uint64(rank))
    # philox_words packs its second and third counter words from a 64-bit `env`: here (update_lo, update_hi); the fourth is `step` = rank
    m = ((w[0] >> np.uint32(5)).astype(np.uint64) << np.uint64(26)) + (w[1] >> np.uint32(6)).astype(np.uint64)
    return m.astype(np.float64) * 2.0 ** -53


def descend(tree, cap, u):
    """the kernel's walk from the root: right iff u >= left and the right sum > 0 (u -= left) -> slot"""
    node = 1
    while node < cap:
        left, right = tree[2 * node], tree[2 * node + 1]
        if u >= left and right > 0.0:
            u -= left
            node = 2 * node + 1
        else:
            node = 2 * node
    return node - cap


def sample_mirror(tree, cap, length, B, beta, seed, update, rank):
    """-> (idx [B] int64, weights [B] float64 before the f32 store) of gq_per_sample"""
    total = tree[1]
    U = stratum_uniforms(seed, B, update, rank)
    idx = np.array([descend(tree, cap, (np.float64(j) + U[j]) * (total / B)) for j in range(B)], dtype=np.int64)
    w = (np.float64(length) * tree[cap + idx] / total) ** (-beta)
    return idx, w / w.max()


def build_tree(leaves):
    """a tree whose leaves are `leaves` (padded with zeros to a power of two)"""
    m = TreeMirror(len(leaves))
    m.tree[m.cap:m.cap + len(leaves)] = leaves
    m._fix(m.cap + np.arange(len(leaves)))
    return m


# ------------------------------------------------------------------------------------------------ tests
def test_capacity_is_the_next_power_of_two():
    assert [capacity(n) for n in (1, 2, 3, 2000, 2048, 16385, 1048576)] == [1, 2, 4, 2048, 2048, 32768, 1048576]


def test_mirror_tree_nodes_are_sums_of_their_children():
    m = TreeMirror(13)
    m.push(np.arange(13))
    m.update([3, 7, 3], [0.25, 0.5, 0.75], [1.0, 0.0, 0.0], 0.6, 1e-6)
    k = np.arange(1, m.cap)
    assert np.array_equal(m.tree[k], m.tree[2 * k] + m.tree[2 * k + 1])
    assert m.leaves()[3] == (0.75 + 1e-6) ** 0.6 and m.leaves()[13:].tolist() == [0.0] * 3  # later duplicate wins; unfilled leaves 0
    assert m.pmax == 1.0  # every priority here is below the initial pmax


def test_descent_follows_the_proportional_rule():
    m = build_tree([1.0, 2.0, 0.0, 3.0, 4.0])  # cap 8: slots 5..7 empty
    total = m.tree[1]
    assert total == 10.0
    cuts = np.cumsum([1.0, 2.0, 0.0, 3.0, 4.0])
    for u in np.linspace(0.0, 9.999, 997):
        want = int(np.searchsorted(cuts, u, side="right"))
        assert descend(m.tree, m.cap, u) == want, u


def test_descent_never_ends_on_an_empty_leaf():
    # an empty right subtree at every level: all mass in slot 0 of a 16-slot tree
    m = build_tree([2.5] + [0.0] * 15)
    for u in (0.0, 1.0, 2.5, 2.5 * (1 + 2 ** -52), 3.0, 1e300):  # u at and past the total (rounding of (j + U) total / B)
        assert descend(m.tree, m.cap, u) == 0
    # u rounded up to exactly the total lands on the last non-empty slot, not on the empty ones after it
    m = build_tree([0.1, 0.2, 0.3, 0.0, 0.0])
    assert descend(m.tree, m.cap, m.tree[1]) == 2 and descend(m.tree, m.cap, np.nextafter(m.tree[1], np.inf)) == 2
    # an empty left subtree: every u goes right
    m = build_tree([0.0, 0.0, 0.0, 0.0, 1.0, 1.0])
    assert {descend(m.tree, m.cap, u) for u in np.linspace(0, 2, 41)} == {4, 5}


def test_sampling_a_partly_filled_non_power_of_two_replay():
    size, length = 2000, 1234  # cap 2048; slots >= length never filled
    m = TreeMirror(size)
    m.push(np.arange(length))
    rng = np.random.RandomState(0)
    idx = rng.randint(0, length, 400)
    m.update(idx, rng.rand(400).astype(np.float32), (rng.rand(400) < 0.2).astype(np.float32), 0.6, 1e-6)
    for B, update, rank in ((1, 0, 0), (12, 7, 0), (12, 7, 1), (64, 2 ** 40 + 3, 5)):
        got, w = sample_mirror(m.tree, m.cap, length, B, 0.4, 1234, update, rank)
        assert (got < length).all() and (m.leaves()[got] > 0).all()
        if B > 1:  # stratified: stratum j draws from [j, j + 1) total / B, so the slots come out in order
            assert (np.diff(got) >= 0).all()
    a, _ = sample_mirror(m.tree, m.cap, length, 12, 0.4, 1234, 7, 0)
    b, _ = sample_mirror(m.tree, m.cap, length, 12, 0.4, 1234, 7, 1)
    assert not np.array_equal(a, b)  # the rank is part of the key


def test_stratum_uniforms_are_53_bit_and_uniform():
    U = np.concatenate([stratum_uniforms(9, 1000, u, 0) for u in range(50)])
    assert ((U >= 0) & (U < 1)).all()
    assert np.all(np.floor(U * 2.0 ** 53) == U * 2.0 ** 53)
    assert abs(U.mean() - 0.5) < 0.01 and np.histogram(U, bins=10, range=(0, 1))[0].min() > 0.09 * U.size
    assert len(np.unique(U)) == U.size


def test_importance_weights():
    m = build_tree([1.0, 4.0, 0.5, 2.5])
    total, N = m.tree[1], 4
    for beta in (0.0, 0.4, 1.0):
        idx, w = sample_mirror(m.tree, m.cap, N, 4, beta, 3, 0, 0)
        raw = (N * m.leaves()[idx] / total) ** (-beta)
        assert np.allclose(w, raw / raw.max(), rtol=0, atol=0)
        assert w.max() == 1.0 and (w > 0).all()
        # beta = 1 exactly undoes the sampling bias: w is proportional to 1 / p
        if beta == 1.0:
            assert np.allclose(w * m.leaves()[idx], (w * m.leaves()[idx])[0], rtol=1e-15)
        if beta == 0.0:
            assert (w == 1.0).all()


def test_beta_schedule():
    from mujoco_rl_ur5_b200.batched_train import per_beta

    assert per_beta(0, 0.4, 100) == 0.4
    assert per_beta(50, 0.4, 100) == pytest.approx(0.7, abs=1e-15)
    assert per_beta(100, 0.4, 100) == 1.0 and per_beta(10 ** 6, 0.4, 100) == 1.0
    assert per_beta(0, 0.4, 0) == 1.0
    b = [per_beta(u, 0.4, 12) for u in range(13)]
    assert np.allclose(np.diff(b), 0.6 / 12, rtol=0, atol=1e-15)


def test_trainer_builds_its_replay_from_the_prioritized_option(monkeypatch):
    """without `prioritized` the trainer keeps the uniform ObservationReplay; with it, the prioritized one with the given alpha / eps"""
    from mujoco_rl_ur5_b200 import batched_train
    from mujoco_rl_ur5_b200.replay_buffer import ObservationReplay

    made = []

    class FakeEnv:
        IMAGE_WIDTH = IMAGE_HEIGHT = 4
        TABLE_HEIGHT = 0.9
        rotations = list(range(6))
        cam = 0

        def __init__(self, n, scene, device, env_index_offset=0):
            import torch

            self.engine = types.SimpleNamespace(device=torch.device("cpu"))
            self.arrays = {"cam_fovy": [45.0], "cam_pos0": [0.0, 0.0, 2.0], "cam_mat0": list(np.eye(3).ravel())}

    class FakePER:
        def __init__(self, size, hw, device, alpha, eps):
            made.append(dict(size=size, hw=hw, alpha=alpha, eps=eps))

    monkeypatch.setattr(batched_train, "BatchedGraspEnv", FakeEnv)
    monkeypatch.setattr(batched_train, "QNetLearner", lambda *a, **k: types.SimpleNamespace(step_count=0))
    monkeypatch.setattr(batched_train, "PrioritizedObservationReplay", FakePER)
    tr = batched_train.BatchedTrainer(8)
    assert type(tr.replay) is ObservationReplay and tr.per is None
    tr = batched_train.BatchedTrainer(8, prioritized=dict(alpha=0.7, beta_updates=30))
    assert isinstance(tr.replay, FakePER) and made == [dict(size=2000, hw=(4, 4), alpha=0.7, eps=1e-6)]
    assert tr.per == dict(alpha=0.7, beta0=0.4, beta_updates=30, eps=1e-6)
    with pytest.raises(ValueError):
        batched_train.BatchedTrainer(8, prioritized=dict(alpha=0.6))  # beta_updates is required
    with pytest.raises(ValueError):
        batched_train.BatchedTrainer(8, prioritized=dict(beta_updates=3, gamma=0.9))


def test_prioritized_replay_refuses_a_cpu_device():
    from mujoco_rl_ur5_b200.replay_buffer import PrioritizedObservationReplay

    with pytest.raises(RuntimeError):
        PrioritizedObservationReplay(16, (2, 2), device="cpu")
