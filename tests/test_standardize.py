"""Standardised observations (transform_observation(normalize=False)) and normalize.py's channel statistics, on the CPU: the
mean_and_std pickle, a numpy restatement of gq_obs_to_state_standard's arithmetic against the reference's own transform
(tests/golden/standardize.npz, written by tests/golden/make_standardize_golden.py) and the trainer's argument checks.
The device side is tests/test_standardize_gpu.py."""
import json
import os
import pickle

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
THR = np.float32(1.1)  # the agent's depth_threshold (np.round(cam z - TABLE_HEIGHT + 0.01, 3)) as the float32 depth compares with it
# (seed, H, W) of the observations the reference's transform_observation(normalize=False) was run on
STATE_CASES = [(11, 200, 200), (12, 37, 23), (13, 23, 37), (14, 48, 64), (15, 1, 7)]
NORMALIZE_CASE = dict(seed=2024, n=100, H=200, W=200)


def synthetic_obs(seed, H, W):
    """one seeded observation (rgb u8 [H,W,3], depth f32 [H,W] metres) holding 0 and 255 in every channel and depths above, at and
    below float32(1.1); the 200x200 one is piecewise smooth (so that its states compress), the others are noise"""
    rng = np.random.RandomState(seed)
    if H * W >= 10000:
        yy, xx = np.mgrid[0:H, 0:W]
        rgb = np.stack([(xx * 255) // (W - 1), (yy * 255) // (H - 1), ((xx + yy) * 7) % 256], axis=-1).astype(np.uint8)
        depth = (np.float32(0.95) + np.float32(0.002) * ((xx // 8 + yy // 5) % 90).astype(np.float32)).astype(np.float32)
    else:
        rgb = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
        depth = rng.uniform(0.8, 1.3, size=(H, W)).astype(np.float32)
    flat_rgb, flat_d = rgb.reshape(-1, 3), depth.reshape(-1)
    n = flat_d.size
    flat_rgb[0] = 0
    flat_rgb[n - 1] = 255
    flat_d[0] = THR
    if n > 1:
        flat_d[1] = np.nextafter(THR, np.float32(2))
    if n > 2:
        flat_d[2] = np.nextafter(THR, np.float32(0))
    if n > 3:
        flat_d[3] = np.float32(1.5)
    return rgb, depth


def normalize_observations(seed=NORMALIZE_CASE["seed"], n=NORMALIZE_CASE["n"], H=NORMALIZE_CASE["H"], W=NORMALIZE_CASE["W"]):
    """the observations the reference's normalize.py was given (one per env.reset()), as arrays rgb [n,H,W,3] u8, depth [n,H,W] f32:
    rgb channels with different spreads, depth a table plane with objects on it"""
    rng = np.random.RandomState(seed)
    rgb = np.empty((n, H, W, 3), np.uint8)
    depth = np.empty((n, H, W), np.float32)
    for i in range(n):
        rgb[i, ..., 0] = rng.randint(0, 256, size=(H, W))
        rgb[i, ..., 1] = np.clip(rng.normal(120, 50, size=(H, W)), 0, 255).astype(np.uint8)
        rgb[i, ..., 2] = rng.binomial(255, 0.6, size=(H, W))
        d = np.full((H, W), 1.77, np.float32)
        for _ in range(6):
            y, x, s = rng.randint(0, H - 20), rng.randint(0, W - 20), rng.randint(5, 20)
            d[y:y + s, x:x + s] = rng.uniform(1.6, 1.75)
        depth[i] = d + rng.normal(0, 1e-3, size=(H, W)).astype(np.float32)
    return rgb, depth


def standard_state_numpy(rgb, depth, stats32, thr=THR):
    """gq_obs_to_state_standard at noise_std = 0 in numpy float32 (every operation rounded on its own): [4,H,W] f32"""
    m, s = stats32[:4], stats32[4:]
    out = [(rgb[..., c].astype(np.float32) - m[c]) / s[c] for c in range(3)]
    d = (np.minimum(depth, thr) - m[3]) / s[3]
    out.append(d + np.float32(0.0))
    return np.stack(out).astype(np.float32)


def _golden():
    with open(os.path.join(GOLDEN, "standardize.json")) as f:
        meta = json.load(f)
    return meta, np.load(os.path.join(GOLDEN, "standardize.npz"))


def _typed(entry):
    return [np.dtype(t).type(float.fromhex(v)) for v, t in zip(entry["values"], entry["types"])]


def test_load_reads_the_reference_file_values_and_types(tmp_path):
    from mujoco_rl_ur5_b200.obs_stats import load_mean_and_std

    meta, _ = _golden()
    ship = meta["shipped"]
    p = tmp_path / "mean_and_std"
    p.write_bytes(bytes.fromhex(ship["pickle_hex"]))  # the reference's shipped file, byte for byte
    got = load_mean_and_std(str(p))
    assert [type(v).__name__ for v in got] == ship["types"] == ["float64"] * 3 + ["float32"] + ["float64"] * 3 + ["float32"]
    assert [float(v).hex() for v in got] == ship["values"]
    nm = meta["normalize"]
    p2 = tmp_path / "from_normalize_py"
    p2.write_bytes(bytes.fromhex(nm["pickle_hex"]))
    assert [float(v).hex() for v in load_mean_and_std(str(p2))] == nm["values"]


def test_save_load_round_trip_keeps_the_reference_types(tmp_path):
    from mujoco_rl_ur5_b200.obs_stats import load_mean_and_std, save_mean_and_std

    meta, _ = _golden()
    vals = _typed(meta["shipped"])
    p = tmp_path / "ms"
    save_mean_and_std(str(p), [float(v) for v in vals])
    got = load_mean_and_std(str(p))
    assert [type(v) for v in got] == [type(v) for v in vals]
    assert [float(v) for v in got] == [float(v) for v in vals]
    with open(p, "rb") as f:
        assert [float(v) for v in pickle.load(f)] == [float(v) for v in vals]


def test_loader_refuses_other_pickles(tmp_path):
    from mujoco_rl_ur5_b200.obs_stats import load_mean_and_std

    p = tmp_path / "evil"
    p.write_bytes(pickle.dumps(os.getcwd))  # a callable global: refused without being looked up
    with pytest.raises(ValueError, match="numpy scalars only"):
        load_mean_and_std(str(p))
    p.write_bytes(pickle.dumps([1.0] * 7))
    with pytest.raises(ValueError):
        load_mean_and_std(str(p))
    p.write_bytes(b"")
    with pytest.raises(ValueError):
        load_mean_and_std(str(p))


def test_numpy_restatement_equals_the_reference_transform_bit_for_bit():
    from mujoco_rl_ur5_b200.obs_stats import as_float32

    meta, z = _golden()
    stats32 = as_float32(_typed(meta["used"]))
    assert [c["seed"] for c in meta["states"]] == [c[0] for c in STATE_CASES]
    for seed, H, W in STATE_CASES:
        rgb, depth = synthetic_obs(seed, H, W)
        ref = z[f"state_{seed}"]
        assert ref.shape == (1, 4, H, W) and ref.dtype == np.float32
        mine = standard_state_numpy(rgb, depth, stats32)
        assert np.array_equal(mine.view(np.uint32), ref[0].view(np.uint32)), (seed, H, W)


@pytest.mark.parametrize("bad, match", [([1.0] * 7, "8 finite"), ([1, 2, 3, 4, 5, 6, 0.0, 8], "> 0"), ([1, 2, 3, 4, 5, 6, 7, -1], "> 0"),
                                        ([1, 2, 3, float("nan"), 5, 6, 7, 8], "8 finite"), ([1, 2, "x", 4, 5, 6, 7, 8], "8 numbers")])
def test_bad_statistics_are_refused(bad, match):
    from mujoco_rl_ur5_b200.batched_train import resolve_standardize

    with pytest.raises(ValueError, match=match):
        resolve_standardize(bad)


def test_trainer_standardize_argument_checks(tmp_path):
    from mujoco_rl_ur5_b200.batched_train import BatchedTrainer, main, resolve_standardize
    from mujoco_rl_ur5_b200.obs_stats import save_mean_and_std

    with pytest.raises(FileNotFoundError):
        resolve_standardize(str(tmp_path / "missing"))
    with pytest.raises(FileNotFoundError):  # refused before any device work
        BatchedTrainer(4, standardize=str(tmp_path / "missing"))
    with pytest.raises(ValueError, match="8 finite"):
        BatchedTrainer(4, standardize=[1.0, 2.0])
    with pytest.raises(ValueError, match="> 0"):
        BatchedTrainer(4, standardize=[100, 100, 100, 1.5, 50, 0, 50, 0.4])
    with pytest.raises(SystemExit):
        main(["--standardize", str(tmp_path / "missing")])
    vals = [108.5, 120.25, 132.0, 1.53, 67.8, 57.1, 48.9, 0.42]
    p = tmp_path / "ms"
    save_mean_and_std(str(p), vals)
    assert [float(v) for v in resolve_standardize(str(p))] == [float(v) for v in resolve_standardize(vals)]
    ckpt = {"mean_and_std": [float(v) for v in resolve_standardize(vals)]}
    assert [float(v) for v in resolve_standardize(None, ckpt)] == ckpt["mean_and_std"]  # a resume keeps the stored values
    assert [float(v) for v in resolve_standardize(str(p), ckpt)] == ckpt["mean_and_std"]
    assert resolve_standardize(None, {"step": 3}) is None                                 # a min-max checkpoint stays min-max
    other = list(vals)
    other[7] = 0.43
    with pytest.raises(ValueError, match="mean_and_std"):
        resolve_standardize(other, ckpt)
    with pytest.raises(ValueError, match="mean_and_std"):
        BatchedTrainer(4, load=ckpt, standardize=other)


def test_normalize_cli_refuses_bad_arguments():
    from mujoco_rl_ur5_b200.normalize import main

    with pytest.raises(SystemExit):
        main(["--scene", "C"])
    with pytest.raises(SystemExit):
        main(["--envs", "0"])
