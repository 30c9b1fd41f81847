"""DeviceReplayBuffer (SURVEY 8f.2) against the reference's `Modules.ReplayBuffer` (Modules.py:28-55): same ring behaviour and the
same sampled transitions from the same `random` stream."""
import json
import os
import random

import numpy as np
import torch

from mujoco_rl_ur5_b200.replay_buffer import DeviceReplayBuffer

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_io.json")
REPLAY_CASES = ((20, 5, 57), (2000, 12, 300), (30, 12, 100))  # (size, batch, pushes)


def _drive(buf_push, buf_sample, buf_len, n_push=57, size=20, B=5):
    """the agent's pattern: one push per step, a sample as soon as 2 B transitions are stored (Grasping_Agent_multidiscrete.py:396-401)"""
    out = []
    for k in range(n_push):
        buf_push(k)
        if buf_len() >= 2 * B:
            out.append(buf_sample(B))
    return out


def _ours(size=20, B=5, n_push=57, rng=None):
    b = DeviceReplayBuffer(size, state_shape=(1, 2, 2), device="cpu", rng=rng)
    return _drive(lambda k: b.push(torch.full((1, 1, 2, 2), float(k)), torch.tensor([[k * 3]]), torch.tensor([[k % 2]])),
                  lambda B_: [int(v) for v in b.sample(B_)[0][:, 0, 0, 0]], lambda: len(b), n_push, size, B)


def test_ring_and_sampling_golden():
    # = the reference class driven the same way (tests/golden/reference_io.json, first case)
    got = _ours()
    assert got[0] == [2, 4, 1, 6, 9] and got[-1] == [47, 46, 49, 54, 56]  # = Modules.ReplayBuffer(20, simple=True) driven the same way
    again = _ours()
    assert got == again  # seed 20 at construction -> reproducible
    flat = [v for s in got for v in s]
    assert all(s[-1] == 9 + i for i, s in enumerate(got))             # the newest transition is always the last element
    assert all(len(set(s[:-1])) == 4 for s in got)                     # B - 1 distinct random picks
    assert min(got[-1]) >= 57 - 20                                     # after wrap-around only the last `size` pushes survive
    assert max(flat) == 56


def test_push_batch_equals_consecutive_pushes():
    a = DeviceReplayBuffer(8, state_shape=(1,), device="cpu", rng=random.Random(20))
    b = DeviceReplayBuffer(8, state_shape=(1,), device="cpu", rng=random.Random(20))
    k = 0
    for n in (3, 4, 5, 11, 2):
        s = torch.arange(k, k + n, dtype=torch.float32)[:, None]
        a.push_batch(s, torch.arange(k, k + n), torch.ones(n))
        for i in range(n):
            b.push(s[i], k + i, 1.0)
        k += n
        assert a.position == b.position and len(a) == len(b)
        assert torch.equal(a.states, b.states) and torch.equal(a.actions, b.actions)
        assert a.sample_indices(4) == b.sample_indices(4)


def test_same_samples_as_the_reference_class():
    """the reference's Modules.ReplayBuffer(size, simple=True), run unmodified and driven the same way, sampled these transitions
    (tests/golden/reference_io.json, written by tests/golden/make_reference_io_golden.py); ours draws the same from the same stream"""
    g = json.load(open(GOLD))["replay_buffer"]
    assert [(c["size"], c["B"], c["pushes"]) for c in g] == list(REPLAY_CASES)
    for c in g:
        assert _ours(c["size"], c["B"], c["pushes"]) == c["samples"]  # rng=None: the global `random` module, re-seeded with 20


def test_a_callers_generator_is_not_reseeded():
    """ADVICE r01: the constructor used to call rng.seed(20) on a generator passed in, and on the global module whatever `seed`"""
    r = random.Random(12345)
    expect = random.Random(12345).random()
    DeviceReplayBuffer(4, state_shape=(1,), device="cpu", rng=r)
    assert r.random() == expect
    random.seed(777)
    expect = random.Random(777).random()
    DeviceReplayBuffer(4, state_shape=(1,), device="cpu", seed=None)
    assert random.random() == expect
