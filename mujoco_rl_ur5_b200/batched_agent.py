"""BatchedGreedyAgent: the acting half of the reference's Grasp_Agent for N environments at once, entirely on the device.

Reference: Grasping_Agent_multidiscrete.py — `greedy` (:284-299) = transform_observation (:301-368) -> policy_net (:295) ->
flat arg-max -> transform_action (:381-386); `epsilon_greedy` (:232-282) mixes in uniformly random table pixels.
Here: gq_obs_to_state -> wgmma Q-network forward -> gq_argmax, all kernels of libgrasp_qnet.so; the result is an int32
[N,2] tensor (pixel index, rotation index) that BatchedGraspEnv.step accepts without leaving the GPU (BASELINE config 4).
The learner (replay buffer, BCE loss, Adam; :388-446) is a SURVEY 8(f) "next" row and is not part of this class.

standardize=<mean_and_std path or its 8 values> acts on transform_observation(normalize=False) instead (gq_obs_to_state_standard,
obs_stats): channels standardised with normalize.py's statistics and the depth noise N(0, noise_std) in standardised units, which the
reference adds on every such call; the noise is keyed on (seed, global env id, acting call), the call counted by `acting_step`.
"""
import numpy as np

from .qnet import QNetForward, make_torch_qnet


class BatchedGreedyAgent:
    standardize = None  # the min-max transform unless __init__ is given statistics (also for agents assembled field by field)

    def __init__(self, env, state_dict=None, seed=0, chunk=64, standardize=None, noise_std=0.001):
        import torch

        from .batched_train import resolve_standardize

        self.standardize = resolve_standardize(standardize)
        self.noise_std = float(noise_std)
        self.seed = int(seed)
        self.acting_step = 0

        self.torch = torch
        self.env = env
        if state_dict is None:  # random default initialisation, as the reference's agent starts from
            torch.manual_seed(seed)
            state_dict = make_torch_qnet(len(env.rotations)).state_dict()
        self.qnet = QNetForward(state_dict, env.engine.device.index or 0, max_batch=chunk)
        # depth_threshold = camera height - TABLE_HEIGHT + 0.01 (Grasping_Agent_multidiscrete.py:130-135)
        cam_z = float(np.asarray(env.arrays["cam_pos0"]).reshape(-1, 3)[env.cam][2])
        self.depth_threshold = float(np.round(cam_z - env.TABLE_HEIGHT + 0.01, 3))
        self.gen = torch.Generator(device=env.engine.device)
        self.gen.manual_seed(seed)

    def states(self, obs):
        """the state the agent acts on: the deterministic min-max transform, or with `standardize` the standardised one (each call
        draws the next acting step's noise)"""
        if self.standardize is None:
            return self.qnet.obs_to_state(obs, self.depth_threshold)
        t = self.torch
        genv = self.env.env_index_offset + t.arange(obs["depth"].shape[0], dtype=t.int64, device=obs["depth"].device)
        s = self.qnet.obs_to_state_standard(obs, self.standardize, self.depth_threshold, self.noise_std, self.seed, self.acting_step, genv)
        self.acting_step += 1
        return s

    def q_values(self, obs):
        return self.qnet.forward(self.states(obs))

    def greedy(self, obs):
        """[N,2] int32 actions on the device and their Q-values"""
        act, val = self.qnet.greedy(self.q_values(obs))
        return act.to(self.torch.int32), val

    def random_table_actions(self, obs, max_rounds=64):
        """The reference's random action (Grasping_Agent_multidiscrete.py:262-279): draw a flat action uniformly from all
        W*H*n_rot, look the pixel's depth up in the current observation, transform it with pixel_2_world and REJECT it unless the
        point lies on or above the table (z >= TABLE_HEIGHT - 0.01); resample until accepted.  Batched: every round redraws only the
        environments that are still rejected (pixel_2_world is the engine's kernel).  Returns int32 [N,2] on the device."""
        t = self.torch
        env = self.env
        N, W, H, R = env.n_envs, env.IMAGE_WIDTH, env.IMAGE_HEIGHT, len(env.rotations)
        dev = obs["depth"].device
        out = t.zeros((N, 2), dtype=t.int32, device=dev)
        todo = t.ones(N, dtype=t.bool, device=dev)
        ar = t.arange(N, device=dev)
        for _ in range(max_rounds):
            flat = t.randint(0, W * H * R, (N,), generator=self.gen, device=dev)
            a1, a2 = flat % (W * H), flat // (W * H)
            x, y = a1 % W, a1 // W
            d = obs["depth"][ar, y, x].contiguous()
            xyz = env.engine.pixel_2_world(x.to(t.int32).contiguous(), y.to(t.int32).contiguous(), d, env.cam, W, H)
            ok = todo & (xyz[:, 2] >= env.TABLE_HEIGHT - 0.01)
            out[ok, 0] = a1[ok].to(t.int32)
            out[ok, 1] = a2[ok].to(t.int32)
            todo = todo & ~ok
            if not bool(todo.any()):
                break
        if bool(todo.any()):  # an image without a single table pixel: keep the last draw (the reference would loop forever)
            out[todo, 0] = a1[todo].to(t.int32)
            out[todo, 1] = a2[todo].to(t.int32)
        return out

    def epsilon_greedy(self, obs, eps):
        """with probability eps the reference's depth-filtered random action (random_table_actions), else the greedy one"""
        t = self.torch
        act, val = self.greedy(obs)
        rnd = self.random_table_actions(obs)
        pick = t.rand(act.shape[0], generator=self.gen, device=act.device) < eps
        return t.where(pick[:, None], rnd, act), val
