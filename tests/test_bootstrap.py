"""Bootstrapped Q-learning on the host: the trainer's and the CLI's checks of gamma / target_update, and the next-observation
bookkeeping of ObservationReplay(next_obs=True) on a CPU device.  tests/test_bootstrap_gpu.py covers the kernel, the target network and
the trainer on the GPU."""
import random
import types

import pytest
import torch

from mujoco_rl_ur5_b200.replay_buffer import ObservationReplay

BAD = [dict(gamma=1.5, target_update=10), dict(gamma=-0.1, target_update=10), dict(gamma=float("nan"), target_update=10), dict(gamma="0.9", target_update=10),
       dict(gamma=True, target_update=10), dict(gamma=0.9, target_update=None), dict(gamma=0.9, target_update=0), dict(gamma=0.9, target_update=-3),
       dict(gamma=0.9, target_update=2.5), dict(gamma=0.9, target_update=True), dict(gamma=1.0, target_update="5"), dict(gamma=0.0, target_update=5)]


@pytest.mark.parametrize("kw", BAD, ids=lambda kw: f"{kw['gamma']}-{kw['target_update']}")
def test_trainer_refuses_bad_gamma_and_target_update(kw):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer, check_bootstrap

    with pytest.raises(ValueError):
        check_bootstrap(**kw)
    with pytest.raises(ValueError):  # before any environment or device is touched
        BatchedTrainer(4, "A", 0, **kw)


def test_trainer_accepts_gamma_in_the_unit_interval():
    from mujoco_rl_ur5_b200.batched_train import check_bootstrap

    assert check_bootstrap(0.0, None) == (0.0, None) and check_bootstrap(0, None) == (0.0, None)
    assert check_bootstrap(0.9, 100) == (0.9, 100) and check_bootstrap(1, 1) == (1.0, 1) and check_bootstrap(1e-9, 7) == (1e-9, 7)


@pytest.mark.parametrize("argv", [["--gamma", "0.9"], ["--gamma", "1.5", "--target-update", "10"], ["--gamma", "-1", "--target-update", "10"],
                                  ["--gamma", "0.9", "--target-update", "0"], ["--target-update", "10"], ["--gamma", "nan", "--target-update", "10"]])
def test_cli_refuses_bad_gamma_and_target_update(argv, capsys):
    from mujoco_rl_ur5_b200.batched_train import main

    with pytest.raises(SystemExit) as e:
        main(["--envs", "4"] + argv)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert "gamma" in err or "target_update" in err, err


def _obs(n, k0, offset=0):
    """n observations whose depth pixels hold k0 + i + offset and whose rgb holds it mod 256"""
    k = torch.arange(k0, k0 + n) + offset
    rgb = (k % 256).to(torch.uint8)[:, None, None, None].expand(n, 2, 2, 3).contiguous()
    depth = k.to(torch.float32)[:, None, None].expand(n, 2, 2).contiguous()
    return rgb, depth


class _KeyedStub:
    """stands in for QNetForward.obs_to_state_keyed on the CPU: row b = (depth, red channel, env, step key) of slot b"""

    def obs_to_state_keyed(self, rgb, depth, env_index, step, seed, slot=None, depth_threshold=1.1, noise_std=0.001):
        return torch.stack([depth[slot][:, 0, 0].double(), rgb[slot][:, 0, 0, 0].double(), env_index.double(), step.double()], dim=1)


def test_next_observations_stay_paired_across_wrap_around_and_oversized_pushes():
    size, N_NEXT = 8, 1000
    rp = ObservationReplay(size, (2, 2), device="cpu", rng=random.Random(20), next_obs=True)
    plain = ObservationReplay(size, (2, 2), device="cpu", rng=random.Random(20))
    assert plain.next_rgb is None and plain.next_depth is None and plain.next_steps is None
    k = 0
    for n in (3, 4, 5, 11, 2, 8, 17, 1):  # wrap-around and pushes larger than the ring
        rgb, depth = _obs(n, k)
        nrgb, ndepth = _obs(n, k, N_NEXT)
        key = torch.full((n,), 2 ** 32 - 2 + k)  # keys wrap at 2^32 too
        rp.push_batch(rgb, depth, torch.arange(k, k + n), torch.ones(n), 5000 + torch.arange(k, k + n), key, nrgb, ndepth, key + 7)
        plain.push_batch(rgb, depth, torch.arange(k, k + n), torch.ones(n), 5000 + torch.arange(k, k + n), key)
        k += n
        assert (rp.position, len(rp)) == (plain.position, len(plain))
        for name in ("rgb", "depth", "actions", "rewards", "envs", "steps"):
            assert torch.equal(getattr(rp, name), getattr(plain, name)), name
        filled = torch.arange(len(rp))
        j = rp.actions[filled]  # transition number of each filled slot
        assert torch.equal(rp.next_depth[filled, 0, 0], j.to(torch.float32) + N_NEXT)
        assert torch.equal(rp.next_rgb[filled], ((j + N_NEXT) % 256).to(torch.uint8)[:, None, None, None].expand(-1, 2, 2, 3))
        # the next key (pushed as key + 7) is stored as uint32 bits like the key
        assert torch.equal(rp.next_steps[filled], (rp.steps[filled].to(torch.int64) + 7).bitwise_and(0xFFFFFFFF).to(torch.int32))
    # sampling: the same draws as without next observations, and the next states of the drawn slots
    st = rp.rng.getstate()
    idx = rp.sample_indices(5)
    rp.rng.setstate(st)
    s, a, r, s2 = rp.sample(5, _KeyedStub(), 3)
    assert torch.equal(a[:, 0], rp.actions[idx])
    assert torch.equal(s2[:, 0], s[:, 0] + N_NEXT) and torch.equal(s2[:, 2], s[:, 2])
    assert torch.equal(s2[:, 3], rp.next_steps[idx].to(torch.float64))
    plain.rng.setstate(st)
    out = plain.sample(5, _KeyedStub(), 3)
    assert len(out) == 3 and torch.equal(out[0], s)


def test_next_observation_replay_needs_the_next_observation():
    rp = ObservationReplay(4, (2, 2), device="cpu", rng=random.Random(1), next_obs=True)
    rgb, depth = _obs(2, 0)
    with pytest.raises(ValueError):
        rp.push_batch(rgb, depth, torch.arange(2), torch.ones(2), torch.arange(2), torch.zeros(2))
    assert len(rp) == 0 and rp.position == 0


def test_trainer_bootstraps_with_a_synced_target_network():
    """BatchedTrainer.bellman_targets with stand-ins for the learner: syncs exactly at step_count % target_update == 0 and whenever the
    learner has no target yet (a fresh or a resumed trainer)"""
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer

    synced = []

    class Target:
        def max_target(self, s2, r, gamma):
            return None, (r, gamma)

    learner = types.SimpleNamespace(target=None, step_count=7)

    def sync_target():
        synced.append(learner.step_count)
        learner.target = Target()

    learner.sync_target = sync_target
    tr = types.SimpleNamespace(learner=learner, gamma=0.5, target_update=4)
    for u in range(7, 18):
        learner.step_count = u
        assert BatchedTrainer.bellman_targets(tr, None, u) == (u, 0.5)
    assert synced == [7, 8, 12, 16]
