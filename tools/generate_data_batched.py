#!/usr/bin/env python
"""Offline-RL data generation with N batched environments — what `Offline RL/generate_data.py:21-101` does with one env:
epsilon-greedy actions from the Q-network, every (state, flat action, reward) written in the reference's file format
(`Data/grasping_data_{k}.pt`, 12 transitions each; mujoco_rl_ur5_b200/offline_data.py) so that the reference's
`Offline RL/train.py` / `grasping_dataset.py` read them unchanged.

  python tools/generate_data_batched.py --envs 256 --episodes 2 --steps 10 --out Data [--weights ckpt.pt] [--eps 0.3] [--branches K]
Needs a GPU (no CPU fallback).  One `add` = N transitions; episodes reset all environments (GraspingEnv.py:409-477).
--branches K > 1: every step also labels K - 1 random table actions (BatchedGreedyAgent.random_table_actions) from the same state with
BatchedGraspEnv.evaluate_actions, so one settled scene and one observation give K labelled transitions per env.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--eps", type=float, default=0.3)
    ap.add_argument("--out", default="Data")
    ap.add_argument("--weights", default=None, help="checkpoint written by the reference agent (key model_state_dict) or a bare state_dict")
    ap.add_argument("--scene", default="A")
    ap.add_argument("--seed", type=int, default=122)  # generate_data.py:16
    ap.add_argument("--branches", type=int, default=1, help="labelled transitions per env and step (1 + K-1 random table actions)")
    args = ap.parse_args()
    import torch

    from mujoco_rl_ur5_b200.batched_agent import BatchedGreedyAgent
    from mujoco_rl_ur5_b200.batched_env import BatchedGraspEnv
    from mujoco_rl_ur5_b200.offline_data import TransitionRecorder

    sd = None
    if args.weights:
        ck = torch.load(args.weights, map_location="cpu", weights_only=False)
        sd = ck.get("model_state_dict", ck)
    env = BatchedGraspEnv(args.envs, args.scene, 0)
    agent = BatchedGreedyAgent(env, sd, seed=args.seed)
    rec = TransitionRecorder(args.out)
    for ep in range(args.episodes):
        obs = env.reset()
        for _ in range(args.steps):
            act, _ = agent.epsilon_greedy(obs, args.eps)
            extra = None
            if args.branches > 1:  # labelled before the step: the extra attempts start from the state the observation shows
                extra = torch.stack([agent.random_table_actions(obs) for _ in range(args.branches - 1)], dim=1)
                extra_reward, _ = env.evaluate_actions(extra)
            nxt, reward, done, info = env.step(act)
            rec.add(obs, act, reward)
            for k in range(args.branches - 1):
                rec.add(obs, extra[:, k], extra_reward[:, k])
            obs = nxt
        print(f"episode {ep + 1}: rewards so far {dict(rec.reward_counter)}, {len(rec.files)} files")
    files = rec.close()
    print(f"wrote {len(files)} files to {args.out}")


if __name__ == "__main__":
    main()
