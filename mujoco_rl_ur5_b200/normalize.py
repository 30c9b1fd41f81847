"""The reference's normalize.py, batched: the channel statistics of reset observations for transform_observation(normalize=False).

normalize.py (:14-66) resets one environment 100 times, takes np.mean / np.std of every pixel per channel and pickles the eight
values to `mean_and_std`.  Here one BatchedGraspEnv of N environments is reset once (env i seeded seed_base + i, as every batched
reset), gq_obs_channel_stats reduces the N observations on the device, and the same pickle is written (obs_stats.save_mean_and_std).
The statistics belong to the scene and the renderer: compute them for the scene a run trains on.

    python -m mujoco_rl_ur5_b200.normalize --scene A --envs 100 --out mean_and_std
"""
import argparse

from .obs_stats import channel_statistics, save_mean_and_std

NAMES = ("Red", "Green", "Blue", "Depth")


def compute(scene, n_envs, seed_base=20000, device=0):
    """-> the 8 statistics of one batched reset of n_envs environments of `scene`"""
    from .batched_env import BatchedGraspEnv

    env = BatchedGraspEnv(n_envs, scene, device, seed_base=seed_base)
    try:
        obs = env.reset()
        return channel_statistics(obs["rgb"], obs["depth"])
    finally:
        env.close()


def main(argv=None):
    p = argparse.ArgumentParser(prog="python -m mujoco_rl_ur5_b200.normalize", description=__doc__.split("\n")[0])
    p.add_argument("--scene", choices=("A", "A1", "B"), default="A")
    p.add_argument("--envs", type=int, default=100, help="environments reset once (normalize.py takes 100 resets)")
    p.add_argument("--seed-base", type=int, default=20000, help="env i resets with seed seed_base + i")
    p.add_argument("--device", type=int, default=0)
    p.add_argument("--out", default="mean_and_std", help="the pickle to write (the reference's file name by default)")
    a = p.parse_args(argv)
    if a.envs < 1:
        p.error("--envs must be >= 1")
    values = compute(a.scene, a.envs, a.seed_base, a.device)
    print(f"Collected {a.envs} images from the environment.")
    for name, v in zip(NAMES, values[:4]):
        print(f"Calculated mean value of {v} for channel {name}.")
    for name, v in zip(NAMES, values[4:]):
        print(f"Calculated standard deviation of {v} for channel {name}.")
    save_mean_and_std(a.out, values)
    print(f"\nWrote values to file {a.out}.")
    return values


if __name__ == "__main__":
    main()
